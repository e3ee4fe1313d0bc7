"""Map colourisation on the GPU: the reference's `moge/utils/vis.py` colourisers (`colorize_depth`, `colorize_depth_affine`,
`colorize_disparity`, `colorize_normal`) on CUDA tensors, with the reference's arguments.

The work runs in moge_b200/csrc/vis.cu: the normalising quantiles are np.nanquantile's exact order statistics, found by a radix
select whose result stays on the device, and a colouring kernel reads them there, so a call never waits on the host.  Results
are bitwise those of the numpy restatement in oracle/vis_port.py (the reference's lines, with matplotlib's "Spectral" map
restated).  Only "Spectral" is provided; any other `cmap` raises.

A (H, W) map is one image, as in the reference.  A (B, H, W) map is a batch: each image is normalised by its own quantiles, so
every image's colours equal those of a call on it alone.  The returns are (..., H, W, 3) uint8 RGB, or BGR with `bgr=True`
(what cv2.imwrite expects); `out` may name a contiguous uint8 CUDA tensor of that shape to write into.  CUDA tensors only; there
is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import capi
from .capi import MogeError

__all__ = ["colorize_depth", "colorize_depth_affine", "colorize_disparity", "colorize_normal", "quantiles", "spectral_table"]

MAX_PIXELS = 1 << 30
SPECTRAL = ((158, 1, 66), (213, 62, 79), (244, 109, 67), (253, 174, 97), (254, 224, 139), (255, 255, 191), (230, 245, 152),
            (171, 221, 164), (102, 194, 165), (50, 136, 189), (94, 79, 162))      # ColorBrewer "Spectral", 8-bit


def spectral_table() -> np.ndarray:
    """The (256, 3) uint8 colour table: matplotlib's LinearSegmentedColormap.from_list over the 11 Spectral colours with
    _create_lookup_table(256, gamma=1) in float64, then trunc(clip(lut, 0, 1) * 255) as the reference converts colours."""
    rgb = np.array(SPECTRAL, dtype=np.float64) / 255
    x = np.linspace(0, 1, len(rgb)) * 255
    xind = 255 * np.linspace(0, 1, 256)
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([rgb[:1], distance[:, None] * (rgb[ind] - rgb[ind - 1]) + rgb[ind - 1], rgb[-1:]])
    return (np.clip(lut, 0.0, 1.0) * 255).astype(np.uint8)


_tables: Dict[torch.device, torch.Tensor] = {}


def _table(device: torch.device) -> torch.Tensor:
    t = _tables.get(device)
    if t is None:
        t = _tables[device] = torch.from_numpy(spectral_table()).to(device)
    return t


def _check_cmap(cmap: str) -> None:
    if cmap != "Spectral":
        raise MogeError(f"colour map {cmap!r} is not provided: only 'Spectral'")


def _maps(what: str, x: torch.Tensor, mask: Optional[torch.Tensor], channels: int = 0) -> Tuple[torch.Tensor, Optional[torch.Tensor], tuple]:
    """(..., H, W[, C]) fp32 map and (..., H, W) mask -> (batch, H, W[, C]) contiguous map, uint8 mask, the leading shape."""
    lead = 3 if channels else 2
    if not isinstance(x, torch.Tensor) or x.dim() < lead or (channels and x.shape[-1] != channels):
        raise MogeError(f"{what}: expected a (..., H, W{', %d' % channels if channels else ''}) tensor")
    if x.dtype != torch.float32:
        raise MogeError(f"{what}: the map must be float32, not {x.dtype}")
    shape = tuple(x.shape[:-1]) if channels else tuple(x.shape)
    if mask is not None and (not isinstance(mask, torch.Tensor) or tuple(mask.shape) != shape):
        raise MogeError(f"{what}: mask {tuple(getattr(mask, 'shape', ()))} does not match the map {shape}")
    capi.require_cuda(what, x, mask)
    H, W = shape[-2:]
    capi.check_pixels(what, H, W, MAX_PIXELS)
    x = x.detach().contiguous().view(-1, H, W, *([channels] if channels else []))
    m = None if mask is None else capi.mask_u8(mask).view(-1, H, W)
    return x, m, shape


def _out(what: str, out: Optional[torch.Tensor], shape: tuple, device) -> torch.Tensor:
    want = shape + (3,)
    if out is None:
        return torch.empty(want, dtype=torch.uint8, device=device)
    if not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or tuple(out.shape) != want or not out.is_contiguous() \
            or out.device != device:
        raise MogeError(f"{what}: out must be a contiguous uint8 tensor of shape {want} on {device}")
    return out


def _quantiles(x: torch.Tensor, kind: int, m: Optional[torch.Tensor], q) -> torch.Tensor:
    B, H, W = x.shape
    L = capi.lib()
    qs = (C.c_float * len(q))(*[float(np.float32(v)) for v in q])
    out = torch.empty(B, len(q), dtype=torch.float32, device=x.device)
    ws = capi.workspace(L.moge_vis_workspace_bytes, B, H, W, device=x.device)
    capi.check(L.moge_vis_quantiles(x.data_ptr(), kind, capi.ptr(m), B, H, W, qs, len(q), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                    capi.current_stream()))
    return out


def quantiles(values: torch.Tensor, q, mask: torch.Tensor = None, depth: bool = False) -> torch.Tensor:
    """np.nanquantile of each image's valid values, linear method, fp32, bitwise: values (..., H, W) fp32, q a sequence of up to 4
    values in [0, 1].  Excluded are NaN values, pixels off `mask` and, with depth=True, the values are 1 / depth where depth > 0
    (the disparities colorize_depth normalises).  Returns (..., len(q)) fp32 on the device, NaN for an image with no valid value."""
    q = list(q)
    if not 1 <= len(q) <= capi.VIS_MAX_QUANTILES:
        raise MogeError(f"quantiles: 1 to {capi.VIS_MAX_QUANTILES} quantiles, not {len(q)}")
    x, m, shape = _maps("quantiles", values, mask)
    with torch.cuda.device(x.device):
        return _quantiles(x, capi.VIS_DEPTH if depth else capi.VIS_VALUE, m, q).view(*shape[:-2], len(q))


def _colorize(what: str, values: torch.Tensor, mask, kind: int, q, invert: bool, cmap: str, bgr: bool, out) -> torch.Tensor:
    _check_cmap(cmap)
    x, m, shape = _maps(what, values, mask)
    B, H, W = x.shape
    with torch.cuda.device(x.device):
        res = _out(what, out, shape, x.device)
        rng = None if q is None else _quantiles(x, kind, m, q)
        capi.check(capi.lib().moge_vis_colorize(x.data_ptr(), kind, int(invert), capi.ptr(m), B, H, W, capi.ptr(rng),
                                                _table(x.device).data_ptr(), int(bool(bgr)), res.data_ptr(), capi.current_stream()))
    return res


def colorize_depth(depth: torch.Tensor, mask: torch.Tensor = None, normalize: bool = True, cmap: str = 'Spectral', *,
                   bgr: bool = False, out: torch.Tensor = None) -> torch.Tensor:
    """The disparity 1 / depth where depth > 0 (and in `mask`), normalised between its 0.001 and 0.99 quantiles, coloured at
    1 - x.  +inf depth is disparity 0 and takes part; depth <= 0, NaN and masked-out pixels are black."""
    return _colorize("colorize_depth", depth, mask, capi.VIS_DEPTH, (0.001, 0.99) if normalize else None, True, cmap, bgr, out)


def colorize_depth_affine(depth: torch.Tensor, mask: torch.Tensor = None, cmap: str = 'Spectral', *, bgr: bool = False,
                          out: torch.Tensor = None) -> torch.Tensor:
    """The depth (in `mask`) normalised between its 0.001 and 0.999 quantiles, coloured at x (not inverted)."""
    return _colorize("colorize_depth_affine", depth, mask, capi.VIS_VALUE, (0.001, 0.999), False, cmap, bgr, out)


def colorize_disparity(disparity: torch.Tensor, mask: torch.Tensor = None, normalize: bool = True, cmap: str = 'Spectral', *,
                       bgr: bool = False, out: torch.Tensor = None) -> torch.Tensor:
    """The disparity (in `mask`) normalised between its 0.001 and 0.999 quantiles, coloured at 1 - x."""
    return _colorize("colorize_disparity", disparity, mask, capi.VIS_VALUE, (0.001, 0.999) if normalize else None, True, cmap, bgr,
                     out)


def colorize_normal(normal: torch.Tensor, mask: torch.Tensor = None, *, bgr: bool = False, out: torch.Tensor = None) -> torch.Tensor:
    """(..., H, W, 3) fp32 normals -> uint8 trunc(clip(n * (0.5, -0.5, -0.5) + 0.5, 0, 1) * 255), computed in fp64; pixels off
    `mask` are the zero normal (127, 127, 127)."""
    x, m, shape = _maps("colorize_normal", normal, mask, channels=3)
    B, H, W = x.shape[:3]
    with torch.cuda.device(x.device):
        res = _out("colorize_normal", out, shape, x.device)
        capi.check(capi.lib().moge_vis_normal(x.data_ptr(), capi.ptr(m), B, H, W, int(bool(bgr)), res.data_ptr(), capi.current_stream()))
    return res
