"""-m gpu: operator-level parity of the hand-written sm_90a kernels (through the C ABI) against plain PyTorch
fp32 references of the same op on the same (16-bit rounded) inputs."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, to_padded_nhwc, empty_padded, from_padded_nhwc, border_ok

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}


def _lib():
    return capi.lib()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (1370, 1152, 384), (300, 256, 592), (677, 1024, 4096), (2 * 1370, 3072, 1024)])
def test_linear_bias(M, N, K, dtype):
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    x = (torch.randn(M, K, generator=g)).to(DEV).to(dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV).to(dtype)
    b = torch.randn(N, generator=g).to(DEV)
    out = torch.full((M, N), float("nan"), dtype=dtype, device=DEV)
    capi.check(_lib().moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), None, out.data_ptr(), M, N, K, 0, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t() + b
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_linear_gelu(dtype):
    M, N, K = 1370, 1536, 384
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV).to(dtype)
    b = torch.randn(N, generator=g).to(DEV)
    out = torch.empty(M, N, dtype=dtype, device=DEV)
    capi.check(_lib().moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), None, out.data_ptr(), M, N, K, 1, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.gelu(x.float() @ w.float().t() + b)
    assert rel_l2(out, ref) < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(1370, 384, 1536), (1370, 1024, 1024), (150, 768, 3072)])
def test_linear_residual_layerscale(M, N, K, dtype):
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV).to(dtype)
    b = torch.randn(N, generator=g).to(DEV)
    gamma = torch.randn(N, generator=g).to(DEV)
    res = torch.randn(M, N, generator=g).to(DEV)
    out = res.clone()
    capi.check(_lib().moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), gamma.data_ptr(), out.data_ptr(), M, N, K, 2, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = res + gamma * (x.float() @ w.float().t() + b)
    assert rel_l2(out, ref) < (2e-5 if dtype == torch.float16 else 2e-5) + 1e-4


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K,epi", [(1370, 1152, 384, 0), (300, 3072, 1024, 0), (677, 3072, 768, 1), (2 * 1370, 4096, 1024, 1)])
def test_linear_with_folded_layernorm(M, N, K, epi, dtype):
    """norm -> linear (-> GELU) computed as ONE GEMM on the rounded residual rows (LayerNorm folded into weights + epilogue),
    against LayerNorm + linear in fp32.  The rows get a per-row offset and scale so mean and variance matter."""
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    x = (torch.randn(M, K, generator=g) * (0.5 + 2 * torch.rand(M, 1, generator=g)) + torch.randn(M, 1, generator=g)).to(DEV)
    lg = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    lb = (0.2 * torch.randn(K, generator=g)).to(DEV)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    out = torch.empty(M, N, device=DEV, dtype=dtype)
    capi.check(_lib().moge_op_linear_ln(x.data_ptr(), lg.data_ptr(), lb.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, epi,
                                        dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.linear(F.layer_norm(x, (K,), lg, lb, 1e-6), w, b)
    if epi == 1:
        ref = F.gelu(ref)
    assert rel_l2(out, ref) < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [384, 768, 1024])
def test_layernorm(D, dtype):
    rows = 1371
    g = torch.Generator(device="cpu").manual_seed(D)
    x = (torch.randn(rows, D, generator=g) * 3 + 0.5).to(DEV)
    gm = (1 + 0.1 * torch.randn(D, generator=g)).to(DEV)
    bt = (0.1 * torch.randn(D, generator=g)).to(DEV)
    out = torch.empty(rows, D, dtype=dtype, device=DEV)
    capi.check(_lib().moge_op_layernorm(x.data_ptr(), gm.data_ptr(), bt.data_ptr(), out.data_ptr(), rows, D, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.layer_norm(x, (D,), gm, bt, 1e-6)
    assert rel_l2(out, ref) < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,N,heads", [(1, 118, 6), (2, 257, 6), (1, 1370, 16), (2, 700, 12)])
def test_attention(B, N, heads, dtype):
    D = heads * 64
    g = torch.Generator(device="cpu").manual_seed(N)
    qkv = (torch.randn(B, N, 3 * D, generator=g) * 1.5).to(DEV).to(dtype)
    out = torch.full((B, N, D), float("nan"), dtype=dtype, device=DEV)
    capi.check(_lib().moge_op_attention(qkv.data_ptr(), out.data_ptr(), B, N, D, heads, dt(dtype), stream()))
    torch.cuda.synchronize()
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4).unbind(0)
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, D)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < (3e-3 if dtype == torch.float16 else 1.5e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 18, 26, 64, 64), (2, 24, 40, 256, 256), (1, 37, 37, 128, 128), (1, 48, 36, 64, 32),
                                               (2, 40, 50, 64, 64), (1, 33, 47, 64, 128), (1, 9, 20, 64, 64)])
def test_conv3x3_replicate_skip_relu(B, H, W, Cin, Cout, dtype):
    g = torch.Generator(device="cpu").manual_seed(H * W + Cin)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(DEV)
    b = torch.randn(Cout, generator=g).to(DEV)
    skip = torch.randn(B, Cout, H, W, generator=g).to(DEV).to(dtype)
    xp, sp = to_padded_nhwc(x, dtype), to_padded_nhwc(skip, dtype)
    raw, relu = empty_padded(B, H, W, Cout, dtype, DEV), empty_padded(B, H, W, Cout, dtype, DEV)
    capi.check(_lib().moge_op_conv(xp.data_ptr(), w.data_ptr(), b.data_ptr(), sp.data_ptr(), raw.data_ptr(), relu.data_ptr(),
                                   B, H, W, Cin, Cout, 9, 0, dt(dtype), stream()))
    torch.cuda.synchronize()
    wq = w.to(dtype).float()
    ref = F.conv2d(F.pad(x.float(), (1, 1, 1, 1), mode="replicate"), wq, b) + skip.float()
    assert rel_l2(from_padded_nhwc(raw, H, W), ref) < TOL[dtype]
    assert rel_l2(from_padded_nhwc(relu, H, W), F.relu(ref)) < TOL[dtype]
    assert border_ok(raw, H, W) and border_ok(relu, H, W)


def test_conv3x3_halo_streamed_weights():
    """3x3 convs with C_in >= 128.  Images at least 8 pixels tall (padded height >= 10, one halo box) take the CONVH mode
    (halo boxes + streamed weights); the 6-pixel-tall ones (padded height 8) take the per-tap GEMM mode."""
    for dtype in (torch.float16, torch.bfloat16):
        test_conv3x3_replicate_skip_relu(2, 24, 40, 256, 256, dtype)      # CONVH
        test_conv3x3_replicate_skip_relu(1, 37, 37, 128, 128, dtype)      # CONVH
        test_conv3x3_replicate_skip_relu(1, 21, 50, 192, 128, dtype)      # CONVH
        test_conv3x3_replicate_skip_relu(2, 6, 40, 256, 256, dtype)       # per-tap GEMM
        test_conv3x3_replicate_skip_relu(1, 6, 37, 128, 128, dtype)       # per-tap GEMM
        test_conv3x3_replicate_skip_relu(1, 6, 50, 192, 128, dtype)       # per-tap GEMM


def test_conv3x3_c64_resident_weights():
    """The CONV64 mode (C_in = 64: resident weights, halo boxes) with one and two output-channel tiles, ragged image edges."""
    for dtype in (torch.float16, torch.bfloat16):
        test_conv3x3_replicate_skip_relu(2, 40, 50, 64, 64, dtype)
        test_conv3x3_replicate_skip_relu(1, 33, 47, 64, 128, dtype)


@pytest.mark.parametrize("dtype", [torch.float16])
def test_conv1x1(dtype):
    B, H, W, Cin, Cout = 2, 19, 37, 384, 384
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(dtype)
    w = (torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5).to(DEV)
    b = torch.randn(Cout, generator=g).to(DEV)
    xp = to_padded_nhwc(x, dtype)
    raw = empty_padded(B, H, W, Cout, dtype, DEV)
    capi.check(_lib().moge_op_conv(xp.data_ptr(), w.data_ptr(), b.data_ptr(), None, raw.data_ptr(), None, B, H, W, Cin, Cout, 1, 0, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), w.to(dtype).float(), b)
    assert rel_l2(from_padded_nhwc(raw, H, W), ref) < TOL[dtype]
    assert border_ok(raw, H, W)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 9, 13, 384, 256), (2, 18, 26, 256, 128), (1, 37, 37, 128, 64)])
def test_conv_transpose_k2s2(B, H, W, Cin, Cout, dtype):
    g = torch.Generator(device="cpu").manual_seed(H + W + Cin)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(dtype)
    w = (torch.randn(Cin, Cout, 2, 2, generator=g) / Cin ** 0.5).to(DEV)
    b = torch.randn(Cout, generator=g).to(DEV)
    xp = to_padded_nhwc(x, dtype)
    raw = empty_padded(B, 2 * H, 2 * W, Cout, dtype, DEV)
    capi.check(_lib().moge_op_conv(xp.data_ptr(), w.data_ptr(), b.data_ptr(), None, raw.data_ptr(), None, B, H, W, Cin, Cout, 1, 1, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(x.float(), w.to(dtype).float(), b, stride=2)
    assert rel_l2(from_padded_nhwc(raw, 2 * H, 2 * W), ref) < TOL[dtype]
    assert border_ok(raw, 2 * H, 2 * W)
