"""-m gpu: the 128 x 256 row tiles with the direct epilogue, which qkv- and fc1-like linears (EPI_STORE16 / EPI_GELU16, with and
without the LayerNorm fold) take when N is a multiple of 256 and there are at least four such tiles per SM: accuracy against fp32
references, no write past row M, the same bits as the 128 x 128 staged tiles on the same columns, and two identical calls against
each other bit for bit.  The wide tiles run at M = 43840 (the benchmark's rows; last tile 64 rows) and at 64 full row tiles plus
1, 37 or 100 rows (a last tile with a single row, with rows for the first consumer warpgroup only, and for both); the small M
(1, 100, 257, 1370: one or two tiles per SM) take the staged tiles, through the same entry points."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, check_tiles, TILE_LINEAR

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}      # test_gpu_gemm_rows' tolerances for 16-bit outputs
K = 1024
SENTINEL = 1234.0      # exact in fp16 and bf16
PAD = 64               # rows past M that must stay untouched


def make_case(M, N, ln, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = torch.randn(N, generator=g, device=DEV)
    if ln:
        # rows with a per-row offset and scale, so that the folded mean and variance matter
        x = torch.randn(M, K, generator=g, device=DEV) * (0.5 + 2 * torch.rand(M, 1, generator=g, device=DEV)) \
            + torch.randn(M, 1, generator=g, device=DEV)
        lg = 1 + 0.3 * torch.randn(K, generator=g, device=DEV)
        lb = 0.2 * torch.randn(K, generator=g, device=DEV)
        w = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5
        return dict(x=x, lg=lg, lb=lb, w=w, b=b)
    x = torch.randn(M, K, generator=g, device=DEV).to(dtype)
    w = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).to(dtype)
    return dict(x=x, w=w, b=b)


def run(case, M, N, epi, ln, dtype, w=None, b=None):
    """out[:M] = the linear; out[M:M+PAD] prefilled with SENTINEL, out[:M] with NaN"""
    w = case["w"] if w is None else w
    b = case["b"] if b is None else b
    out = torch.full((M + PAD, N), float("nan"), device=DEV, dtype=dtype)
    out[M:] = SENTINEL
    lib = capi.lib()
    if ln:
        capi.check(lib.moge_op_linear_ln(case["x"].data_ptr(), case["lg"].data_ptr(), case["lb"].data_ptr(), w.data_ptr(), b.data_ptr(),
                                         out.data_ptr(), M, N, K, epi, dt(dtype), stream()))
    else:
        capi.check(lib.moge_op_linear(case["x"].data_ptr(), w.data_ptr(), b.data_ptr(), None, out.data_ptr(), M, N, K, epi, dt(dtype),
                                      stream()))
    return out


def reference(case, epi, ln):
    if ln:
        ref = F.linear(F.layer_norm(case["x"], (K,), case["lg"], case["lb"], 1e-6), case["w"], case["b"])
    else:
        ref = case["x"].float() @ case["w"].float().t() + case["b"]
    return F.gelu(ref) if epi == 1 else ref


@pytest.mark.parametrize("M", [43840, 8193, 8229, 8292, 1370, 1, 100, 257])
@pytest.mark.parametrize("N", [3072, 4096, 2304])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("ln", [True, False], ids=["linear_ln", "linear"])
@pytest.mark.parametrize("epi", [0, 1], ids=["store", "gelu"])
def test_wide_tiles_accuracy_and_bounds(epi, ln, dtype, N, M):
    case = make_case(M, N, ln, dtype, seed=M + N + 7 * epi)
    out = run(case, M, N, epi, ln, dtype)
    torch.cuda.synchronize()
    assert bool((out[M:] == SENTINEL).all()), "a row past M was written"
    got = out[:M]
    assert bool(torch.isfinite(got.float()).all()), "a row below M was not written"
    ref = reference(case, epi, ln)
    assert rel_l2(got, ref) < TOL[dtype]
    # every tile, the ragged last row tile (1, 37 or 100 rows past 64 full tiles) included
    check_tiles(got, ref, TILE_LINEAR, TOL[dtype], f"linear wide {dtype}")


@pytest.mark.parametrize("M", [43840, 8229])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("ln", [True, False], ids=["linear_ln", "linear"])
@pytest.mark.parametrize("epi", [0, 1], ids=["store", "gelu"])
def test_wide_tiles_match_narrow_tiles_and_repeat(epi, ln, dtype, M):
    # N = 3072 runs the 128 x 256 tiles; N = 1152 (not a multiple of 256) the 128 x 128 staged ones, on the same first 1152
    # weight rows with the same k-order
    case = make_case(M, 3072, ln, dtype, seed=11 + M + epi)
    wide = run(case, M, 3072, epi, ln, dtype)
    again = run(case, M, 3072, epi, ln, dtype)
    narrow = run(case, M, 1152, epi, ln, dtype, w=case["w"][:1152].contiguous(), b=case["b"][:1152].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(wide, again), "two identical calls differ"
    a, b = wide[:M, :1152], narrow[:M]
    diff = (a.float() - b.float()).abs().max().item()
    assert torch.equal(a, b), f"128 x 256 and 128 x 128 tiles differ: max |diff| {diff:.3e}"
