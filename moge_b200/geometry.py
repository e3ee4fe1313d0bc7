"""Geometry utilities on the GPU: the functions of the reference's `moge/utils/geometry_torch.py` with its signatures, defaults
and return conventions.  `moge.utils.geometry_torch` re-exports them as a drop-in for the reference's module.

Kernel-backed (moge_b200/csrc/geometry.cu and, for `recover_focal_shift`, the engine's focal/shift kernel): CUDA tensors only, no
CPU fallback, fp32 maps, leading dimensions flattened (at most 65535 maps per call).  No kernel uses atomics, so every call gives
the same bits on every run.
  - `refine_depth_with_normal`: a log kernel, a set-up kernel (Laplacian term) and one Jacobi sweep kernel per iteration.  Like
    the reference it clamps the caller's `depth` to at least `eps` IN PLACE.  Within a per-element bound of the fp64
    restatement in oracle/geometry_port.py (the gradient term is computed in fp64 here; the sweeps in fp32 as in the reference).
  - `dilate_with_mask`: one launch per iteration.  `min`, `max` and `median` are bitwise the reference's; `mean` sums the at most
    four neighbours left to right, within 4 fp32 roundings per iteration of the exact mean.
  - `theshold_depth_change` (the reference's spelling): bitwise the reference's.
  - `gaussian_blur_2d`: the reference's fp32 weights, summed in row-major tap order.  Even kernel sizes are rejected (the
    reference's taps are then asymmetric and its output one pixel larger).
  - `recover_focal_shift`: the engine's focal/shift kernel, which restates the reference's SciPy solve on its fixed 64 x 64
    nearest-downsampled grid; other `downsample_size` values raise.

The closed forms (`weighted_mean`, `harmonic_mean`, `geometric_mean`, `normalized_view_plane_uv`, `focal_to_fov`, `fov_to_focal`,
`angle_diff_vec3`, `intrinsics_to_fov`, `point_map_to_depth_legacy`, `view_plane_uv_to_focal`) are torch expressions stated from
their definitions; they run on any device.

Divergences from the reference:
  - `dilate_with_mask` with `min` or `max`: the reference calls `Tensor.min` / `Tensor.max` with a tuple of dims, which torch
    rejects with a TypeError; these filters take the window minimum / maximum over the valid neighbours (NaN propagating, as
    torch.amin / amax), with +inf / -inf where there is none, the reference's fill values;
  - an unknown `filter` raises ValueError (the reference leaves the values unchanged and still grows the mask);
  - kernel-backed functions take fp32 maps only and return no autograd graph.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Literal, Tuple, Union

import torch

from . import capi
from .capi import MogeError
from .configs import uv_spans

__all__ = ["weighted_mean", "harmonic_mean", "geometric_mean", "normalized_view_plane_uv", "gaussian_blur_2d", "focal_to_fov",
           "fov_to_focal", "angle_diff_vec3", "intrinsics_to_fov", "point_map_to_depth_legacy", "view_plane_uv_to_focal",
           "recover_focal_shift", "theshold_depth_change", "dilate_with_mask", "refine_depth_with_normal"]

FOCAL_SHIFT_GRID = (64, 64)        # the focal/shift kernel's downsample grid (height, width)


# ------------------------------------------------------------------------------------------------------------ closed forms
def weighted_mean(x: torch.Tensor, w: torch.Tensor = None, dim: Union[int, torch.Size] = None, keepdim: bool = False,
                  eps: float = 1e-7) -> torch.Tensor:
    """mean(x w) / (mean(w) + eps) over `dim`; the plain mean without `w`."""
    if w is None:
        return x.mean(dim=dim, keepdim=keepdim)
    w = w.to(x.dtype)
    return (x * w).mean(dim=dim, keepdim=keepdim) / w.mean(dim=dim, keepdim=keepdim).add(eps)


def harmonic_mean(x: torch.Tensor, w: torch.Tensor = None, dim: Union[int, torch.Size] = None, keepdim: bool = False,
                  eps: float = 1e-7) -> torch.Tensor:
    """1 / (the (weighted) mean of 1 / (x + eps)), with eps added again before the last reciprocal when weighted."""
    inv = x.add(eps).reciprocal()
    if w is None:
        return inv.mean(dim=dim, keepdim=keepdim).reciprocal()
    return weighted_mean(inv, w.to(x.dtype), dim=dim, keepdim=keepdim, eps=eps).add(eps).reciprocal()


def geometric_mean(x: torch.Tensor, w: torch.Tensor = None, dim: Union[int, torch.Size] = None, keepdim: bool = False,
                   eps: float = 1e-7) -> torch.Tensor:
    """exp of the (weighted) mean of log(x + eps).  Without `w` the reduced dims are dropped whatever `keepdim` says, as in the
    reference."""
    logs = x.add(eps).log()
    if w is None:
        return logs.mean(dim=dim).exp()
    return weighted_mean(logs, w.to(x.dtype), dim=dim, keepdim=keepdim, eps=eps).exp()


def normalized_view_plane_uv(width: int, height: int, aspect_ratio: float = None, dtype: torch.dtype = None,
                             device: torch.device = None) -> torch.Tensor:
    """(height, width, 2) pixel-centre UV on the view plane of unit half diagonal: the corners are at +-(width, height) /
    diagonal times (n - 1) / n, for an aspect ratio of width / height unless given."""
    if aspect_ratio is None:
        aspect_ratio = width / height
    sx, sy = uv_spans(aspect_ratio)
    u = torch.linspace(-sx * (width - 1) / width, sx * (width - 1) / width, width, dtype=dtype, device=device)
    v = torch.linspace(-sy * (height - 1) / height, sy * (height - 1) / height, height, dtype=dtype, device=device)
    return torch.stack(torch.meshgrid(u, v, indexing="xy"), dim=-1)


def focal_to_fov(focal: torch.Tensor):
    """Field of view of a focal length relative to the image extent: 2 atan(1 / (2 focal))."""
    return 2 * torch.atan(0.5 / focal)


def fov_to_focal(fov: torch.Tensor):
    """The inverse of focal_to_fov: 1 / (2 tan(fov / 2))."""
    return 0.5 / torch.tan(fov / 2)


def angle_diff_vec3(v1: torch.Tensor, v2: torch.Tensor, eps: float = 1e-12):
    """Angle between 3-vectors along the last dim: atan2(|v1 x v2| + eps, v1 . v2)."""
    return torch.atan2(torch.cross(v1, v2, dim=-1).norm(dim=-1) + eps, (v1 * v2).sum(dim=-1))


def intrinsics_to_fov(intrinsics: torch.Tensor):
    """(fov_x, fov_y) in radians of normalized intrinsics (..., 3, 3), from their focal lengths fx = K[0, 0], fy = K[1, 1]."""
    return focal_to_fov(intrinsics[..., 0, 0]), focal_to_fov(intrinsics[..., 1, 1])


def point_map_to_depth_legacy(points: torch.Tensor):
    """The least-squares focal and z shift of a point map (..., H, W, 3) on the view-plane UV, u (z + shift) = focal x and
    v (z + shift) = focal y with a 1e-6 ridge: returns (depth = z + shift, fov_x, fov_y, shift)."""
    height, width = points.shape[-3:-1]
    diagonal = math.hypot(height, width)
    uv = normalized_view_plane_uv(width, height, dtype=points.dtype, device=points.device)
    b = (uv * points[..., 2:]).flatten(-3, -1)                                             # (..., H W 2)
    A = torch.stack([points[..., :2], -uv.expand_as(points[..., :2])], dim=-1).flatten(-4, -2)   # (..., H W 2, 2): [x, -u]
    At = A.transpose(-2, -1)
    ridge = 1e-6 * torch.eye(2, dtype=A.dtype, device=A.device)
    focal, shift = (torch.inverse(At @ A + ridge) @ (At @ b[..., None])).squeeze(-1).unbind(-1)
    depth = points[..., 2] + shift[..., None, None]
    fov_x = torch.atan(width / diagonal / focal) * 2
    fov_y = torch.atan(height / diagonal / focal) * 2
    return depth, fov_x, fov_y, shift


def view_plane_uv_to_focal(uv: torch.Tensor):
    """The least-squares focal f of a (H, W, 2) UV map against the view-plane UV n: sum(uv n) / (sum(uv^2) + 1e-12)."""
    n = normalized_view_plane_uv(width=uv.shape[-2], height=uv.shape[-3], device=uv.device, dtype=uv.dtype)
    return (uv * n).sum() / uv.square().sum().add(1e-12)


# ------------------------------------------------------------------------------------------------------------ kernel-backed
def _f32(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise MogeError(f"{what} must be a float32 tensor, not {getattr(t, 'dtype', type(t).__name__)}")
    return t.detach().contiguous()


def _odd_size(what: str, kernel_size: int, lo: int, hi: int) -> int:
    if not isinstance(kernel_size, int) or kernel_size % 2 == 0 or not lo <= kernel_size <= hi:
        raise ValueError(f"{what}: kernel_size must be an odd integer from {lo} to {hi}, not {kernel_size!r}")
    return kernel_size


def _maps(x: torch.Tensor, what: str, lead: int = 2):
    if not isinstance(x, torch.Tensor) or x.dim() < lead:
        raise MogeError(f"{what} must be a tensor of at least {lead} dims")
    return x.shape[-lead], x.shape[-lead + 1]


def recover_focal_shift(points: torch.Tensor, mask: torch.Tensor = None, focal: torch.Tensor = None,
                        downsample_size: Tuple[int, int] = (64, 64)):
    """(focal, shift) of the point map (..., H, W, 3): the focal length relative to the half diagonal and the z shift that make
    it a pinhole camera's (optical centre at the map's centre), solved on the map's nearest downsample to 64 x 64 over the
    valid points of `mask` (..., H, W).  With `focal` (...) given, only the shift is solved and `focal` is returned.  An image
    with fewer than two valid downsampled points gives focal 1 and shift 0.  Both have the shape `points.shape[:-3]` and
    `points.dtype` (the solve runs in fp32 / fp64)."""
    if tuple(downsample_size) != FOCAL_SHIFT_GRID:
        raise ValueError(f"recover_focal_shift: downsample_size {tuple(downsample_size)} is not supported; the focal/shift kernel "
                         f"solves on the {FOCAL_SHIFT_GRID[0]} x {FOCAL_SHIFT_GRID[1]} grid only")
    capi.require_cuda("recover_focal_shift", points, mask, focal)
    if points.dim() < 3 or points.shape[-1] != 3:
        raise MogeError(f"recover_focal_shift: points must be (..., H, W, 3), not {tuple(points.shape)}")
    shape = points.shape
    H, W = shape[-3], shape[-2]
    p = points.detach().reshape(-1, H, W, 3).float().contiguous()
    B = p.shape[0]
    if mask is not None and mask.shape != shape[:-1]:
        raise MogeError(f"recover_focal_shift: mask {tuple(mask.shape)} does not match points {tuple(shape)}")
    m = None if mask is None else capi.mask_u8(mask).reshape(B, H, W)
    f_in = None if focal is None else focal.detach().reshape(-1).float().contiguous()
    if f_in is not None and f_in.numel() != B:
        raise MogeError(f"recover_focal_shift: focal has {f_in.numel()} values for {B} point maps")
    f_out = torch.empty(B, dtype=torch.float32, device=points.device)
    s_out = torch.empty(B, dtype=torch.float32, device=points.device)
    if B:
        capi.check(capi.lib().moge_recover_focal_shift(p.data_ptr(), None, capi.ptr(m), B, H, W, capi.ptr(f_in), f_out.data_ptr(),
                                                       s_out.data_ptr(), capi.current_stream()))
    shift = s_out.to(points.dtype).reshape(shape[:-3])
    if focal is not None:
        return focal.reshape(shape[:-3]), shift
    return f_out.to(points.dtype).reshape(shape[:-3]), shift


def theshold_depth_change(depth: torch.Tensor, mask: torch.Tensor, pooler: Literal['min', 'max'], rtol: float = 0.2,
                          kernel_size: int = 3):
    """Bool map (..., H, W): with pooler 'max', the largest masked-in depth of the kernel_size window (NaN propagating) exceeds
    depth * (1 + rtol); with 'min', the smallest is below depth * (1 - rtol).  kernel_size is odd, at most 15."""
    if pooler not in ("min", "max"):
        raise ValueError(f"Unsupported pooler: {pooler}")
    _odd_size("theshold_depth_change", kernel_size, 1, capi.GEOMETRY_MAX_POOL_KERNEL)
    capi.require_cuda("theshold_depth_change", depth, mask)
    H, W = _maps(depth, "depth")
    if mask.shape != depth.shape:
        raise MogeError(f"theshold_depth_change: mask {tuple(mask.shape)} does not match depth {tuple(depth.shape)}")
    d = _f32(depth, "depth").reshape(-1, H, W)
    out = torch.empty(d.shape, dtype=torch.uint8, device=depth.device)
    if d.shape[0]:
        factor = C.c_float(1 + rtol if pooler == "max" else 1 - rtol)       # the fp32 operand of the reference's product
        capi.check(capi.lib().moge_threshold_depth_change(d.data_ptr(), capi.mask_u8(mask).reshape(-1, H, W).data_ptr(), d.shape[0],
                                                          H, W, int(pooler == "max"), factor, kernel_size, out.data_ptr(),
                                                          capi.current_stream()))
    return out.view(torch.bool).reshape(depth.shape)


def dilate_with_mask(input: torch.Tensor, mask: torch.BoolTensor, filter: Literal['min', 'max', 'mean', 'median'] = 'mean',
                     iterations: int = 1) -> torch.Tensor:
    """`iterations` steps of: invalid pixels of `input` (..., H, W) take the filter of their valid up / left / right / down
    neighbours and become valid in `mask` when they have one; valid pixels keep their value.  'median' takes the lower middle
    value of an even count (torch.nanmedian); 'mean' and 'median' skip NaN values.  Returns (input, mask)."""
    if filter not in capi.DILATE:
        raise ValueError(f"dilate_with_mask: filter must be one of {', '.join(capi.DILATE)}, not {filter!r}")
    capi.require_cuda("dilate_with_mask", input, mask)
    H, W = _maps(input, "input")
    if mask.shape != input.shape:
        raise MogeError(f"dilate_with_mask: mask {tuple(mask.shape)} does not match input {tuple(input.shape)}")
    x = _f32(input, "input").reshape(-1, H, W)
    if iterations <= 0:
        return input, mask
    B = x.shape[0]
    m = capi.mask_u8(mask).reshape(B, H, W)
    if B == 0:
        return x.clone().reshape(input.shape), m.clone().view(torch.bool).reshape(mask.shape)
    bufs = [(torch.empty_like(x), torch.empty_like(m)) for _ in range(min(iterations, 2))]
    for it in range(iterations):
        ox, om = bufs[it % len(bufs)]
        capi.check(capi.lib().moge_dilate_with_mask(x.data_ptr(), m.data_ptr(), B, H, W, capi.DILATE[filter], ox.data_ptr(),
                                                    om.data_ptr(), capi.current_stream()))
        x, m = ox, om
    return x.reshape(input.shape), m.view(torch.bool).reshape(mask.shape)


def gaussian_blur_2d(input: torch.Tensor, kernel_size: int, sigma: float) -> torch.Tensor:
    """Blur of each channel of `input` (B, C, H, W) by the kernel_size x kernel_size Gaussian of `sigma` (pixels) with replicate
    padding: the outer product of the normalised fp32 taps exp(-t^2 / (2 sigma^2)), t = -(k // 2) .. k // 2.  kernel_size is
    odd, at most 31; even sizes raise ValueError."""
    _odd_size("gaussian_blur_2d", kernel_size, 1, capi.GEOMETRY_MAX_BLUR_KERNEL)
    capi.require_cuda("gaussian_blur_2d", input)
    if not isinstance(input, torch.Tensor) or input.dim() != 4:
        raise MogeError("gaussian_blur_2d: input must be (B, C, H, W)")
    x = _f32(input, "input")
    B, Cc, H, W = x.shape
    taps = torch.arange(-kernel_size // 2 + 1, kernel_size // 2 + 1, dtype=torch.float32)     # the weights: host-side, k values
    k1 = torch.exp(-(taps ** 2) / (2 * sigma ** 2))
    k1 = (k1 / k1.sum()).contiguous()
    out = torch.empty_like(x)
    if B * Cc:
        capi.check(capi.lib().moge_gaussian_blur_2d(x.data_ptr(), B * Cc, H, W, C.cast(k1.data_ptr(), C.POINTER(C.c_float)),
                                                    kernel_size, out.data_ptr(), capi.current_stream()))
    return out


def refine_depth_with_normal(depth: torch.Tensor, normal: torch.Tensor, intrinsics: torch.Tensor, iterations: int = 10,
                             damp: float = 1e-3, eps: float = 1e-12, kernel_size: int = 5) -> torch.Tensor:
    """Depth (..., H, W) refined with the normals (..., H, W, 3) and normalized intrinsics (broadcast to (..., 3, 3)): log-depth
    smoothed by `iterations` Jacobi sweeps of a kernel_size x kernel_size bilateral stencil whose right-hand side is the
    Laplacian implied by the normals, at the pixels kernel_size // 2 or more from the border; the border keeps the input depth.
    kernel_size is odd, from 3 to 9.  Like the reference, `depth` itself is clamped to at least `eps` in place."""
    _odd_size("refine_depth_with_normal", kernel_size, 3, capi.GEOMETRY_MAX_REFINE_KERNEL)
    capi.require_cuda("refine_depth_with_normal", depth, normal, intrinsics)
    H, W = _maps(depth, "depth")
    if depth.dtype != torch.float32:
        raise MogeError(f"refine_depth_with_normal: depth must be float32, not {depth.dtype}")
    if normal.shape != (*depth.shape, 3):
        raise MogeError(f"refine_depth_with_normal: normal {tuple(normal.shape)} is not depth's shape + (3,)")
    batch = depth.shape[:-2]
    d = depth.detach()
    d = d if d.is_contiguous() else d.contiguous()
    n = _f32(normal, "normal").reshape(-1, H, W, 3)
    K = _f32(intrinsics, "intrinsics").broadcast_to((*batch, 3, 3)).reshape(-1, 3, 3).contiguous()
    B = n.shape[0]
    out = torch.empty(d.shape, dtype=torch.float32, device=depth.device)
    if B == 0:
        return out
    ws = capi.workspace(capi.lib().moge_geometry_workspace_bytes, B, H, W, device=depth.device)
    capi.check(capi.lib().moge_refine_depth_with_normal(d.data_ptr(), n.data_ptr(), K.data_ptr(), B, H, W, max(int(iterations), 0),
                                                        float(damp), float(eps), kernel_size, out.data_ptr(), ws.data_ptr(),
                                                        ws.numel(), capi.current_stream()))
    if d.data_ptr() != depth.data_ptr():
        depth.detach().copy_(d)                    # the in-place clamp reaches a non-contiguous caller's tensor too
    return out
