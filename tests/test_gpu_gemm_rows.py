"""-m gpu: the four encoder linears of ViT-L at the benchmark's row count (32 images x 1370 tokens = 43840 rows: many tiles per
CTA of the persistent grid and a ragged last wave) through the staged epilogues that the epilogue warpgroup runs -- qkv
(EPI_STORE16) and fc1 (EPI_GELU16) with the LayerNorm fold, proj and fc2 (EPI_RESID, updating a pre-filled fp32 residual in
place) -- against fp32 references, and two identical calls against each other bit for bit."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, check_tiles, TILE_LINEAR

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}      # test_gpu_ops' tolerances for 16-bit outputs
M = 32 * 1370
LINEARS = {"qkv": (3072, 1024, 0), "fc1": (4096, 1024, 1), "proj": (1024, 1024, 2), "fc2": (1024, 4096, 2)}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name", list(LINEARS))
def test_encoder_linear_at_bench_rows(name, dtype):
    N, K, epi = LINEARS[name]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    b = torch.randn(N, generator=g, device=DEV)
    lib = capi.lib()
    if epi == 2:
        x = torch.randn(M, K, generator=g, device=DEV).to(dtype)
        w = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).to(dtype)
        gamma = torch.randn(N, generator=g, device=DEV)
        res = torch.randn(M, N, generator=g, device=DEV)

        def run():
            out = res.clone()
            capi.check(lib.moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), gamma.data_ptr(), out.data_ptr(), M, N, K, 2,
                                          dt(dtype), stream()))
            return out

        gemm = gamma * (x.float() @ w.float().t() + b)
        ref = res + gemm
        tol = 2e-5 + 1e-4
    else:
        # rows with a per-row offset and scale, so that the folded mean and variance matter
        x = torch.randn(M, K, generator=g, device=DEV) * (0.5 + 2 * torch.rand(M, 1, generator=g, device=DEV)) \
            + torch.randn(M, 1, generator=g, device=DEV)
        lg = 1 + 0.3 * torch.randn(K, generator=g, device=DEV)
        lb = 0.2 * torch.randn(K, generator=g, device=DEV)
        w = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5

        def run():
            out = torch.full((M, N), float("nan"), device=DEV, dtype=dtype)
            capi.check(lib.moge_op_linear_ln(x.data_ptr(), lg.data_ptr(), lb.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                             M, N, K, epi, dt(dtype), stream()))
            return out

        ref = F.linear(F.layer_norm(x, (K,), lg, lb, 1e-6), w, b)
        if epi == 1:
            ref = F.gelu(ref)
        tol = TOL[dtype]
    first = run()
    second = run()
    torch.cuda.synchronize()
    assert torch.isfinite(first.float()).all()
    assert rel_l2(first, ref) < tol
    if epi == 2:      # the GEMM's contribution on its own, so that the fp32 residual cannot mask a tile of it
        check_tiles(first - res, gemm, TILE_LINEAR, tol, f"linear {name} {dtype}")
    else:
        check_tiles(first, ref, TILE_LINEAR, tol, f"linear {name} {dtype}")
    assert torch.equal(first, second), "two identical calls differ"
