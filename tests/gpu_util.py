"""Shared helpers for the -m gpu parity tests (all compute goes through the C ABI via moge_b200.capi)."""
import ctypes as C

import torch
import torch.nn.functional as F

from moge_b200 import capi


def rel_l2(a, b):
    """Whole-tensor relative L2 error of `a` against the reference `b`, in fp64 on `a`'s device (outputs reach 180 M elements)."""
    a, b = a.double(), b.to(a.device).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# Tile-resolved accuracy.  The kernels write their outputs a tile at a time, and a fault (a ragged last row tile, an edge tile
# off the TMA-store path, one consumer warpgroup's query rows) spoils one tile.  A whole-tensor norm dilutes that by the square
# root of the tile count, so the tests also bound the worst tile, with tiles the finest unit a kernel writes as a whole:
TILE_LINEAR = (64, 64)            # (rows, columns): the wide path's TMA box and the staged epilogue's column group (kEpiCols)
TILE_ATTENTION = (1, 64, 64)      # (image, query rows, head) of (B, N, heads * 64): half of a consumer warpgroup's query tile


def tile_conv(c_out):
    """(image, channels, rows, px) of an NCHW map: the direct conv epilogue's store box, on the 8 x 16 pixel tile grid"""
    return (1, min(64, c_out), 4, 16)


# A tile's error is rms(out_t - ref_t) / max(rms(ref_t), TILE_FLOOR * rms(ref)): judged against its own scale, with a floor so
# that a near-zero tile (ReLU / GELU outputs, a one-row ragged tile) cannot blow up.  The bound is TILE_C times the test's
# whole-tensor tolerance.  Worst-tile / whole-tensor ratios of the kernels in the tests, measured on an H100 80GB HBM3:
#   linears            fp16 1.01-1.56, bf16 1.02-1.63   (the largest on one-row last tiles)
#   linear + residual  fp16 1.14-1.30, bf16 1.15-1.24   (the GEMM's contribution out - res)
#   convs              fp16 1.02-1.22, bf16 1.01-1.22
#   attention          fp16 1.05-1.54, bf16 1.03-1.54   (the largest on a one-row last query block)
# TILE_C = 2 clears the largest ratio, so an output that is uniformly at its whole-tensor tolerance still passes, while one tile
# twice the tolerance off fails.  The smallest tile RMS of a reference was 0.44 of its global RMS (0.82 in the convs), so the
# floor did not engage in these tests; it only bounds tiles whose own scale is below a quarter of the map's.
TILE_FLOOR = 0.25
TILE_C = 2.0


def _tile_sums(x, tile):
    """sums of x over the tiles of shape `tile` (partial tiles at the far edges included as they are)"""
    for d, t in enumerate(tile):
        n = -(-x.shape[d] // t)
        pad = n * t - x.shape[d]
        if pad:
            x = torch.cat([x, x.new_zeros(x.shape[:d] + (pad,) + x.shape[d + 1:])], dim=d)
        x = x.reshape(x.shape[:d] + (n, t) + x.shape[d + 1:]).sum(dim=d + 1)
    return x


def tile_errors(out, ref, tile, floor=TILE_FLOOR):
    """the error of every tile (see TILE_FLOOR), in fp64 on `out`'s device, as a tensor indexed by tile"""
    assert out.shape == ref.shape and len(tile) == out.dim(), (out.shape, ref.shape, tile)
    r = ref.to(out.device).double()
    d2 = _tile_sums((out.double() - r).square(), tile)
    r2 = r.square()
    g2 = r2.sum() / max(r.numel(), 1)
    r2 = _tile_sums(r2, tile)
    cnt = torch.ones((), dtype=torch.float64, device=out.device)
    for d, t in enumerate(tile):
        L = out.shape[d]
        c = torch.full((-(-L // t),), float(t), dtype=torch.float64, device=out.device)
        c[-1] = L - t * (c.numel() - 1)
        cnt = cnt.unsqueeze(-1) * c
    den = torch.maximum(r2 / cnt, floor * floor * g2).clamp_min(1e-60)
    return (d2 / cnt / den).sqrt()


def worst_tile(out, ref, tile, floor=TILE_FLOOR):
    """(error, index) of the worst tile of `out` against `ref`: index is the tile's position in the tile grid"""
    e = tile_errors(out, ref, tile, floor)
    i = int(e.argmax())
    idx = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), e.shape))
    return float(e.reshape(-1)[i]), idx


def check_tiles(out, ref, tile, tol, what=""):
    """asserts that the worst tile of `out` is within TILE_C * tol (tol: the test's whole-tensor bound); prints the worst-tile /
    whole-tensor ratio and returns (error, index) of the worst tile"""
    err, idx = worst_tile(out, ref, tile)
    whole = rel_l2(out, ref)
    print(f"tile-check {what} {tuple(out.shape)} tile {tuple(tile)}: whole {whole:.3e} worst {err:.3e} at {idx} "
          f"ratio {err / max(whole, 1e-30):.2f}")
    assert err < TILE_C * tol, \
        f"{what}: tile {idx} of {tuple(tile)} has error {err:.3e} (whole tensor {whole:.3e}, bound {TILE_C * tol:.1e})"
    return err, idx


def stream():
    return capi.current_stream()


def dt(dtype):
    return capi.torch_dtype_code(dtype)


def to_padded_nhwc(x_nchw: torch.Tensor, dtype) -> torch.Tensor:
    """(B,C,H,W) -> (B,Hp,Wp,C) with a replicated 1-pixel border; Hp = max(H+2, 8), Wp = max(W+2, 16)."""
    B, Cc, H, W = x_nchw.shape
    p = F.pad(x_nchw, (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
    Hp, Wp = max(H + 2, 8), max(W + 2, 16)
    out = torch.zeros(B, Hp, Wp, Cc, dtype=dtype, device=x_nchw.device)
    out[:, :H + 2, :W + 2] = p.to(dtype)
    return out.contiguous()


def empty_padded(B, H, W, Cc, dtype, device):
    return torch.full((B, max(H + 2, 8), max(W + 2, 16), Cc), float("nan"), dtype=dtype, device=device)


def from_padded_nhwc(x: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """interior of a padded map -> (B,C,H,W) fp32"""
    return x[:, 1:H + 1, 1:W + 1].permute(0, 3, 1, 2).float()


def border_ok(x: torch.Tensor, H: int, W: int) -> bool:
    """the 1-pixel border must replicate the edge pixels"""
    inner = x[:, 1:H + 1, 1:W + 1].float()
    ref = F.pad(inner.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
    return bool(torch.equal(ref, x[:, :H + 2, :W + 2].float()))
