"""CPU only: the tile-resolved check of gpu_util (worst_tile) catches a single wrong tile that the whole-tensor relative L2 lets
through.  A synthetic fp32 reference and its 16-bit rounding stand in for a kernel's output; one tile of it is then scaled by
1 + 5 tol -- an interior tile, a ragged last row tile one row tall, an edge pixel tile -- at a gemm_rows-like and a ragged
conv-like shape."""
import pytest
import torch

from gpu_util import TILE_C, TILE_LINEAR, rel_l2, tile_conv, tile_errors, worst_tile

TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}      # test_gpu_ops' whole-tensor tolerances for 16-bit outputs
LINEAR_SHAPE = (43 * 64 + 1, 3072)                       # 43 full row tiles and a last one of a single row
CONV_SHAPE = (2, 96, 37, 53)                             # channel tiles of 64 and 32; last tiles 1 row tall and 5 px wide


def _case(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(shape, generator=g) * (0.5 + torch.rand(shape[-1], generator=g)) + torch.randn(shape[-1], generator=g)
    return ref, ref.to(dtype).float()


def _perturb(out, tile, idx, factor):
    bad = out.clone()
    bad[tuple(slice(i * t, (i + 1) * t) for i, t in zip(idx, tile))] *= factor
    return bad


LINEAR_TILES = {"interior": (17, 23), "ragged_last_row": (43, 11)}
CONV_TILES = {"interior": (1, 0, 4, 1), "ragged_last_row": (0, 0, 9, 2), "edge_pixels": (1, 1, 9, 3), "left_edge": (0, 1, 0, 0)}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape,tile,where", [(LINEAR_SHAPE, TILE_LINEAR, w) for w in LINEAR_TILES] +
                         [(CONV_SHAPE, tile_conv(CONV_SHAPE[1]), w) for w in CONV_TILES])
def test_one_wrong_tile_passes_rel_l2_but_not_worst_tile(shape, tile, where, dtype):
    ref, out = _case(shape, dtype, seed=len(shape))
    tol = TOL[dtype]
    # the untouched rounding passes both checks
    assert rel_l2(out, ref) < tol
    err0, _ = worst_tile(out, ref, tile)
    assert err0 < TILE_C * tol, err0
    idx = (LINEAR_TILES if len(shape) == 2 else CONV_TILES)[where]
    bad = _perturb(out, tile, idx, 1 + 5 * tol)
    # the whole-tensor norm dilutes the wrong tile below the tolerance ...
    assert rel_l2(bad, ref) < tol, rel_l2(bad, ref)
    # ... the tile check names it
    err, at = worst_tile(bad, ref, tile)
    assert err > TILE_C * tol, err
    assert at == idx


def test_tile_errors_match_a_direct_loop():
    """the vectorised per-tile error against a loop over the tiles, partial tiles and the floor included"""
    g = torch.Generator().manual_seed(3)
    ref = torch.randn(3, 70, 45, generator=g)
    ref[1, 64:] *= 1e-3                  # a near-zero partial tile: its denominator is the floor
    out = ref + 1e-2 * torch.randn(ref.shape, generator=g)
    tile, floor = (2, 64, 16), 0.25
    e = tile_errors(out, ref, tile, floor)
    assert e.shape == (2, 2, 3)
    g_rms = ref.double().square().mean().sqrt()
    for i in range(2):
        for j in range(2):
            for k in range(3):
                sl = (slice(2 * i, 2 * i + 2), slice(64 * j, 64 * j + 64), slice(16 * k, 16 * k + 16))
                o, r = out[sl].double(), ref[sl].double()
                want = (o - r).square().mean().sqrt() / torch.maximum(r.square().mean().sqrt(), floor * g_rms)
                torch.testing.assert_close(e[i, j, k], want, rtol=1e-12, atol=0)
