"""Panorama inference on the GPU: the reference's `moge/scripts/infer_panorama.py:83-122` without file I/O, and the device side of
its `moge/utils/panorama.py`.

An equirectangular panorama is split into 12 perspective views (one camera per icosahedron vertex, 90 x 90 degrees), the views go
through one `model.infer(views, fov_x=..., apply_mask=False)` call, and the views' log-distances are merged back into a panorama
by a gradient-domain least-squares solve (SciPy's LSMR on a 4-level pyramid at up to 1920 x 960), then resized to the input.

The batch forms (`split_panoramas`, `merge_panoramas`, `finish_panoramas`, `infer_panoramas`) take up to 64 panoramas of one size
with the same cameras; the merge solves every panorama's system of a level in one cooperative launch, so the panoramas share
that launch's grid barriers.  The single-panorama functions run the same code as a batch of one, so each panorama of a batch
gets bitwise what its single call gives it.

The work runs in moge_b200/csrc/panorama.cu: a split kernel that samples the uint8 panorama as cv2.remap does, a per-level
right-hand-side pass that reads log |points| straight from the engine's output, a matrix-free LSMR in one cooperative kernel
per level, and the resizes.  A merge never waits on the host.  The panorama ray table of each merge size is the reference's own
numpy float32 trigonometry (`spherical_uv_to_directions`), computed once per size and kept on the device, so the projections
see bitwise the reference's rays.  CUDA tensors only; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import capi
from .capi import MogeError

__all__ = ["get_panorama_cameras", "spherical_uv_to_directions", "directions_to_spherical_uv", "uv_map", "split_panorama",
           "merge_panorama", "finish_panorama", "infer_panorama", "last_merge_stats", "split_panoramas", "merge_panoramas",
           "finish_panoramas", "infer_panoramas", "SPLIT_RESOLUTION", "MAX_BATCH"]

SPLIT_RESOLUTION = 512                 # infer_panorama.py:90
MERGE_WIDTH, MERGE_HEIGHT = 1920, 960  # infer_panorama.py:117
PYRAMID_SIZE = 256                     # panorama.py:106: a level recurses while max(w, h) > 256
MAX_PIXELS = 1 << 28
MAX_BATCH = 64                         # panoramas per batched call (MOGE_PANORAMA_MAX_BATCH)


# ------------------------------------------------------------------------------------------------------------ host geometry
def _icosahedron_vertices() -> np.ndarray:
    A = (1 + 5 ** 0.5) / 2
    return np.array([[0, 1, A], [0, -1, A], [0, 1, -A], [0, -1, -A], [1, A, 0], [-1, A, 0], [1, -A, 0], [-1, -A, 0],
                     [A, 0, 1], [A, 0, -1], [-A, 0, 1], [-A, 0, -1]], dtype=np.float32)


def _look_at(eye, look_at, up) -> np.ndarray:
    """OpenCV world-to-camera extrinsics: z towards look_at, x = -up x z, y = z x x."""
    eye, look_at, up = np.asarray(eye), np.asarray(look_at), np.asarray(up)
    z = look_at - eye
    x = np.cross(-up, z)
    y = np.cross(z, x)
    x = x / np.linalg.norm(x, axis=-1, keepdims=True)
    y = y / np.linalg.norm(y, axis=-1, keepdims=True)
    z = z / np.linalg.norm(z, axis=-1, keepdims=True)
    R = np.stack([x, y, z], axis=-2)
    E = np.zeros(R.shape[:-2] + (4, 4), dtype=R.dtype)
    E[..., :3, :3] = R
    E[..., :3, 3] = -(R * eye[..., None, :]).sum(axis=-1)
    E[..., 3, 3] = 1
    return E


def get_panorama_cameras():
    """The reference's 12 cameras: (extrinsics (12, 4, 4) float32, [intrinsics (3, 3) float64] * 12), 90 x 90 degrees."""
    vertices = _icosahedron_vertices()
    fx = 0.5 / np.tan(np.deg2rad(90) / 2)
    intrinsics = np.array([[fx, 0, 0.5], [0, fx, 0.5], [0, 0, 1]], dtype=np.float64)
    extrinsics = _look_at([0, 0, 0], vertices, [0, 0, 1]).astype(np.float32)
    return extrinsics, [intrinsics] * len(vertices)


def uv_map(height: int, width: int) -> np.ndarray:
    """Pixel-centre UV grid (height, width, 2) float32."""
    u = np.linspace(0.5 / width, 1 - 0.5 / width, width, dtype=np.float32)
    v = np.linspace(0.5 / height, 1 - 0.5 / height, height, dtype=np.float32)
    u, v = np.meshgrid(u, v, indexing='xy')
    return np.stack([u, v], axis=2)


def spherical_uv_to_directions(uv: np.ndarray) -> np.ndarray:
    """panorama.py:27-30."""
    theta, phi = (1 - uv[..., 0]) * (2 * np.pi), uv[..., 1] * np.pi
    return np.stack([np.sin(phi) * np.cos(theta), np.sin(phi) * np.sin(theta), np.cos(phi)], axis=-1)


def directions_to_spherical_uv(directions: np.ndarray) -> np.ndarray:
    """panorama.py:33-37."""
    directions = directions / np.linalg.norm(directions, axis=-1, keepdims=True)
    u = 1 - np.arctan2(directions[..., 1], directions[..., 0]) / (2 * np.pi) % 1.0
    v = np.arccos(directions[..., 2]) / np.pi
    return np.stack([u, v], axis=-1)


def _cameras(extrinsics, intrinsics) -> Tuple[C.Array, int]:
    extrinsics = np.asarray(extrinsics, dtype=np.float32)
    intrinsics = np.asarray(intrinsics, dtype=np.float64)
    if extrinsics.ndim != 3 or extrinsics.shape[1:] not in ((4, 4), (3, 4)):
        raise MogeError(f"extrinsics must be (N, 4, 4), not {extrinsics.shape}")
    n = extrinsics.shape[0]
    if intrinsics.shape != (n, 3, 3):
        raise MogeError(f"intrinsics must be {n} (3, 3) matrices, not {intrinsics.shape}")
    if not 1 <= n <= capi.PANORAMA_MAX_VIEWS:
        raise MogeError(f"{n} views is outside [1, {capi.PANORAMA_MAX_VIEWS}]")
    cams = (capi.PanoramaCamera * n)()
    for k in range(n):
        cams[k].R[:] = [float(v) for v in extrinsics[k, :3, :3].reshape(-1)]
        cams[k].t[:] = [float(v) for v in extrinsics[k, :3, 3]]
        K = intrinsics[k]
        cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    return cams, n


_default_cams = None
_tables: Dict[tuple, torch.Tensor] = {}


def _default_cameras():
    global _default_cams
    if _default_cams is None:
        _default_cams = get_panorama_cameras()
    return _default_cams


def _table(kind: str, size: Tuple[int, int], device: torch.device) -> torch.Tensor:
    """Device copies of host tables, made once per size: the split grid (uv_map's fp32 coordinates) and the panorama rays."""
    key = (kind, size, device)
    t = _tables.get(key)
    if t is None:
        if kind == "grid":
            arr = uv_map(1, size[0])[0, :, 0]
        else:
            arr = spherical_uv_to_directions(uv_map(*size)).astype(np.float32)
        t = torch.from_numpy(np.ascontiguousarray(arr)).to(device)
        _tables[key] = t
    return t


def _check_size(what: str, h: int, w: int) -> None:
    if h < 2 or w < 2:
        raise MogeError(f"{what}: a {h} x {w} map is outside [2 x 2, 2^28 pixels]")
    capi.check_pixels(what, h, w, MAX_PIXELS)


def _check_batch(what: str, batch: int) -> None:
    if not 1 <= batch <= MAX_BATCH:
        raise MogeError(f"{what}: a batch of {batch} panoramas is outside [1, {MAX_BATCH}]")


def _check_images(what: str, images) -> Tuple[int, int, int]:
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3:
        raise MogeError(f"{what}: images must be a (P, H, W, 3) uint8 tensor")
    P, H, W = images.shape[:3]
    _check_batch(what, P)
    _check_size(what, H, W)
    capi.require_cuda(what, images)
    return P, H, W


# Each stage has one implementation over a batch of P panoramas (_split, _merge, _finish, _infer), called after the public
# function's own argument checks with the name it raises under; a single-panorama function passes a batch of one and drops
# the leading dimension of the results.

# ------------------------------------------------------------------------------------------------------------ split
def _split(what: str, images: torch.Tensor, extrinsics, intrinsics, resolution: int, return_uint8: bool):
    P, H, W = images.shape[:3]
    if not 1 <= int(resolution) <= 8192:
        raise MogeError(f"{what}: resolution {resolution} is outside [1, 8192]")
    res = int(resolution)
    if extrinsics is None:
        extrinsics, intrinsics = _default_cameras()
    cams, n = _cameras(extrinsics, intrinsics)
    dev = images.device
    with torch.cuda.device(dev):
        img = images.contiguous()
        out = torch.empty(P, n, 3, res, res, dtype=torch.float32, device=dev)
        u8 = torch.empty(P, n, res, res, 3, dtype=torch.uint8, device=dev) if return_uint8 else None
        grid = _table("grid", (res, res), dev)
        capi.check(capi.lib().moge_panorama_split(img.data_ptr(), P, H, W, cams, n, grid.data_ptr(), res, out.data_ptr(), capi.ptr(u8),
                                                  capi.current_stream()))
    return out, u8


def split_panorama(image: torch.Tensor, extrinsics=None, intrinsics=None, resolution: int = SPLIT_RESOLUTION,
                   return_uint8: bool = False):
    """split_panorama_image on the device: image (H, W, 3) uint8 RGB CUDA tensor -> views (N, 3, res, res) float32 (value / 255,
    the tensor infer_panorama.py:98 builds), and with return_uint8 also the uint8 views (N, res, res, 3).  Cameras default to
    get_panorama_cameras()."""
    if not isinstance(image, torch.Tensor) or image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
        raise MogeError("split_panorama: image must be a (H, W, 3) uint8 tensor")
    H, W = image.shape[:2]
    _check_size("split_panorama", H, W)
    capi.require_cuda("split_panorama", image)
    out, u8 = _split("split_panorama", image[None], extrinsics, intrinsics, resolution, return_uint8)
    return (out[0], u8[0]) if return_uint8 else out[0]


def split_panoramas(images: torch.Tensor, extrinsics=None, intrinsics=None, resolution: int = SPLIT_RESOLUTION,
                    return_uint8: bool = False):
    """split_panorama of P panoramas of one size in one launch: images (P, H, W, 3) uint8 RGB CUDA tensor -> views
    (P, N, 3, res, res) float32, and with return_uint8 also (P, N, res, res, 3) uint8; each panorama's views are bitwise its
    split_panorama."""
    _check_images("split_panoramas", images)
    out, u8 = _split("split_panoramas", images, extrinsics, intrinsics, resolution, return_uint8)
    return (out, u8) if return_uint8 else out


# ------------------------------------------------------------------------------------------------------------ merge
def _levels(width: int, height: int) -> List[Tuple[int, int]]:
    sizes = [(width, height)]
    while max(sizes[-1]) > PYRAMID_SIZE:
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    return sizes[::-1]


_last: Dict[str, object] = {}


def num_rows(h: int, w: int) -> int:
    """Rows of a level's system: x-gradient h*w, y-gradient (h-1) x (w+1) on the reference's x-wrapped grid (column w repeats
    column 0), Laplacian h*w."""
    return 2 * h * w + (h - 1) * (w + 1)


def _merge(what: str, width: int, height: int, src: torch.Tensor, mask: torch.Tensor, extrinsics, intrinsics, return_levels: bool):
    """The merge of src (P, N, vh, vw[, 3]) and mask (P, N, vh, vw), whose types and shapes the caller has checked."""
    P, n, vh, vw = src.shape[:4]
    _check_batch(what, P)
    capi.require_cuda(what, src, mask)
    _check_size(f"{what} view", vh, vw)
    if extrinsics is None:
        extrinsics, intrinsics = _default_cameras()
    cams, nc = _cameras(extrinsics, intrinsics)
    if nc != n:
        raise MogeError(f"{what}: {n} views but {nc} cameras")
    channels = 1 if src.dim() == 4 else 3
    dev = src.device
    L = capi.lib()
    levels = _levels(width, height)
    with torch.cuda.device(dev):
        st = capi.current_stream()
        s = src.detach().contiguous()
        m = capi.mask_u8(mask)
        ws = capi.workspace(L.moge_panorama_workspace_bytes, P, n, height, width, device=dev)
        stats = torch.zeros(len(levels), P, 2, dtype=torch.int32, device=dev)
        depth, init, out = None, None, []
        for lv, (w, h) in enumerate(levels):
            b = torch.empty(P, num_rows(h, w), dtype=torch.float64, device=dev)
            rm = torch.empty(P, num_rows(h, w), dtype=torch.uint8, device=dev)
            pm = torch.empty(P, h, w, dtype=torch.uint8, device=dev)
            dirs = _table("dirs", (h, w), dev)
            capi.check(L.moge_panorama_rhs(s.data_ptr(), channels, m.data_ptr(), P, n, vh, vw, cams, dirs.data_ptr(), h, w, b.data_ptr(),
                                           rm.data_ptr(), pm.data_ptr(), ws.data_ptr(), ws.numel(), st))
            depth = torch.empty(P, h, w, dtype=torch.float32, device=dev)
            capi.check(L.moge_panorama_lsmr(b.data_ptr(), rm.data_ptr(), P, h, w, capi.ptr(init), depth.data_ptr(), stats[lv].data_ptr(),
                                            ws.data_ptr(), ws.numel(), st))
            if return_levels:
                out.append({"width": w, "height": h, "b": b, "row_mask": rm, "depth": depth})
            if lv + 1 < len(levels):
                W2, H2 = levels[lv + 1]
                init = torch.empty(P, H2, W2, dtype=torch.float32, device=dev)
                capi.check(L.moge_panorama_resize(depth.data_ptr(), P, h, w, H2, W2, init.data_ptr(), st))
    _last.update(levels=levels, stats=stats)
    return depth, pm.view(torch.bool), out


def merge_panorama(width: int, height: int, src: torch.Tensor, mask: torch.Tensor, extrinsics=None, intrinsics=None,
                   return_levels: bool = False):
    """merge_panorama_depth on the device: src (N, vh, vw) distance maps, or (N, vh, vw, 3) point maps whose norms are the
    distances (the engine's `points`), mask (N, vh, vw) bool / uint8.  Returns (depth (height, width) float32, mask (height, width)
    bool).  With return_levels, also per level (coarsest first) a dict of its size, the fp64 right-hand side, the uint8 row mask in
    the reference's row order (see num_rows) and the solver's fp32 depth.  The per-level iteration
    counts and istop values are in last_merge_stats()."""
    width, height = int(width), int(height)
    _check_size("merge_panorama", height, width)
    if not isinstance(src, torch.Tensor) or src.dtype != torch.float32 or src.dim() not in (3, 4) or (src.dim() == 4 and src.shape[3] != 3):
        raise MogeError("merge_panorama: src must be float32 (N, vh, vw) distances or (N, vh, vw, 3) points")
    if not isinstance(mask, torch.Tensor) or tuple(mask.shape) != tuple(src.shape[:3]) or mask.dtype not in (torch.bool, torch.uint8):
        raise MogeError(f"merge_panorama: mask must be bool / uint8 of shape {tuple(src.shape[:3])}")
    depth, pm, levels = _merge("merge_panorama", width, height, src[None], mask[None], extrinsics, intrinsics, return_levels)
    _last["stats"] = _last["stats"][:, 0]
    result = (depth[0], pm[0])
    if return_levels:
        return (*result, [{k: v[0] if isinstance(v, torch.Tensor) else v for k, v in lv.items()} for lv in levels])
    return result


def merge_panoramas(width: int, height: int, src: torch.Tensor, mask: torch.Tensor, extrinsics=None, intrinsics=None,
                    return_levels: bool = False):
    """merge_panorama of P panoramas with the same cameras: src (P, N, vh, vw) distances or (P, N, vh, vw, 3) points, mask
    (P, N, vh, vw).  Returns (depth (P, height, width) float32, mask (P, height, width) bool), each panorama's bitwise its
    merge_panorama, and with return_levels the per-level dicts with a leading P on b, row_mask and depth.  Each level's P
    systems are solved in one cooperative launch; last_merge_stats() then gives one per-level list per panorama."""
    width, height = int(width), int(height)
    _check_size("merge_panoramas", height, width)
    if not isinstance(src, torch.Tensor) or src.dtype != torch.float32 or src.dim() not in (4, 5) or (src.dim() == 5 and src.shape[4] != 3):
        raise MogeError("merge_panoramas: src must be float32 (P, N, vh, vw) distances or (P, N, vh, vw, 3) points")
    if not isinstance(mask, torch.Tensor) or tuple(mask.shape) != tuple(src.shape[:4]) or mask.dtype not in (torch.bool, torch.uint8):
        raise MogeError(f"merge_panoramas: mask must be bool / uint8 of shape {tuple(src.shape[:4])}")
    depth, pm, levels = _merge("merge_panoramas", width, height, src, mask, extrinsics, intrinsics, return_levels)
    return (depth, pm, levels) if return_levels else (depth, pm)


def last_merge_stats() -> list:
    """Per level of the most recent merge_panorama call on this thread's process, coarsest first: width, height, LSMR iterations
    and istop (SciPy's stopping reason).  After merge_panoramas, one such list per panorama.  Reading them copies the counters to
    the host."""
    if not _last:
        return []
    batched = _last["stats"].dim() == 3              # (levels, P, 2) after merge_panoramas, (levels, 2) after merge_panorama
    stats = _last["stats"].cpu().tolist()

    def per_level(rows):
        return [{"width": w, "height": h, "iterations": it, "istop": st} for (w, h), (it, st) in zip(_last["levels"], rows)]
    if batched:
        return [per_level([lv[k] for lv in stats]) for k in range(len(stats[0]))]
    return per_level(stats)


# ------------------------------------------------------------------------------------------------------------ finish
def _finish(what: str, depth: torch.Tensor, mask: torch.Tensor, height: int, width: int):
    P, h, w = depth.shape
    _check_size(what, h, w)
    _check_size(what, height, width)
    dev = depth.device
    with torch.cuda.device(dev):
        d = depth.contiguous()
        m = capi.mask_u8(mask)
        out_d = torch.empty(P, height, width, dtype=torch.float32, device=dev)
        out_m = torch.empty(P, height, width, dtype=torch.uint8, device=dev)
        points = torch.empty(P, height, width, 3, dtype=torch.float32, device=dev)
        capi.check(capi.lib().moge_panorama_finish(d.data_ptr(), m.data_ptr(), P, h, w, height, width, out_d.data_ptr(),
                                                   out_m.data_ptr(), points.data_ptr(), capi.current_stream()))
    return out_d, out_m.view(torch.bool), points


def finish_panorama(depth: torch.Tensor, mask: torch.Tensor, height: int, width: int):
    """infer_panorama.py:119-122: the merged depth and mask resized to (height, width) as cv2.resize does, and the points."""
    capi.require_cuda("finish_panorama", depth, mask)
    if depth.dtype != torch.float32 or depth.dim() != 2 or tuple(mask.shape) != tuple(depth.shape):
        raise MogeError("finish_panorama: depth must be float32 (h, w) and mask (h, w)")
    return tuple(t[0] for t in _finish("finish_panorama", depth[None], mask[None], height, width))


def finish_panoramas(depth: torch.Tensor, mask: torch.Tensor, height: int, width: int):
    """finish_panorama of P merged maps: depth (P, h, w) float32 and mask (P, h, w) -> depth (P, height, width), mask
    (P, height, width) bool and points (P, height, width, 3)."""
    if not isinstance(depth, torch.Tensor) or not isinstance(mask, torch.Tensor) or depth.dtype != torch.float32 or depth.dim() != 3 \
            or tuple(mask.shape) != tuple(depth.shape):
        raise MogeError("finish_panoramas: depth must be float32 (P, h, w) and mask (P, h, w)")
    _check_batch("finish_panoramas", depth.shape[0])
    capi.require_cuda("finish_panoramas", depth, mask)
    return _finish("finish_panoramas", depth, mask, height, width)


# ------------------------------------------------------------------------------------------------------------ end to end
def _fov_x(intrinsics, device) -> torch.Tensor:
    """infer_panorama.py:99-100: the views' horizontal fields of view in degrees, float32."""
    K = np.asarray(intrinsics)
    fov_x = np.rad2deg(2 * np.arctan(0.5 / K[..., 0, 0]))
    return torch.tensor(fov_x, dtype=torch.float32, device=device)


def _infer(what: str, model, images: torch.Tensor, batch_size: Optional[int], return_views: bool) -> Dict[str, torch.Tensor]:
    P, H, W = images.shape[:3]
    extrinsics, intrinsics = _default_cameras()
    views, views_u8 = _split(what, images, extrinsics, intrinsics, SPLIT_RESOLUTION, return_views)
    n = views.shape[1]
    flat = views.view(P * n, *views.shape[2:])
    fov_x = _fov_x(intrinsics, images.device).repeat(P)
    step = len(flat) if batch_size is None else int(batch_size)
    points, masks = [], []
    for lo in range(0, len(flat), step):
        out = model.infer(flat[lo:lo + step], fov_x=fov_x[lo:lo + step], apply_mask=False)
        points.append(out['points'])
        masks.append(out['mask'])
    points = points[0] if len(points) == 1 else torch.cat(points)
    masks = masks[0] if len(masks) == 1 else torch.cat(masks)
    view_points, view_masks = points.reshape(P, n, *points.shape[1:]), masks.reshape(P, n, *masks.shape[1:])
    depth, mask, _ = _merge(what, min(MERGE_WIDTH, W), min(MERGE_HEIGHT, H), view_points, view_masks, extrinsics, intrinsics, False)
    depth, mask, points = _finish(what, depth, mask, H, W)
    out = {'depth': depth, 'mask': mask, 'points': points}
    if return_views:
        out.update(views=views_u8, view_distance=view_points.norm(dim=-1), view_mask=view_masks)
    return out


def infer_panorama(model, image: torch.Tensor, batch_size: Optional[int] = None, return_views: bool = False) -> Dict[str, torch.Tensor]:
    """infer_panorama.py:83-122 without file I/O.  image: (H, W, 3) uint8 RGB CUDA tensor; model: an engine MoGeModel (MoGe-1 as in
    the reference, or MoGe-2) on the same device.  The 12 views go through one `model.infer(views, fov_x=..., apply_mask=False)`
    call, or calls of batch_size views (the reference's --batch_size).  Returns device tensors {'depth' (H, W), 'mask' (H, W) bool,
    'points' (H, W, 3)}.  With return_views, also what the script's --splitted option writes: 'views' (12, 512, 512, 3) uint8 RGB,
    'view_distance' (12, 512, 512) = the views' points.norm(dim=-1), and 'view_mask' (12, 512, 512) bool."""
    if batch_size is not None and int(batch_size) < 1:
        raise MogeError(f"infer_panorama: batch_size {batch_size} must be positive")
    if not isinstance(image, torch.Tensor) or image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
        raise MogeError("infer_panorama: image must be a (H, W, 3) uint8 tensor")
    capi.require_cuda("infer_panorama", image)
    H, W = image.shape[:2]
    _check_size("infer_panorama", H, W)
    out = _infer("infer_panorama", model, image[None], batch_size, return_views)
    _last["stats"] = _last["stats"][:, 0]
    return {k: v[0] for k, v in out.items()}


def infer_panoramas(model, images: torch.Tensor, batch_size: Optional[int] = None, return_views: bool = False) -> Dict[str, torch.Tensor]:
    """infer_panorama of P panoramas of one size: images (P, H, W, 3) uint8 RGB CUDA tensor.  The 12P views go through
    `model.infer(views, fov_x=..., apply_mask=False)` in one call, or in calls of batch_size views that may straddle panoramas;
    the split, the merge and the finish run once for the whole batch.  Returns device tensors {'depth' (P, H, W), 'mask'
    (P, H, W) bool, 'points' (P, H, W, 3)}, and with return_views 'views', 'view_distance' and 'view_mask' with a leading P.
    Each panorama's outputs are bitwise its infer_panorama."""
    if batch_size is not None and int(batch_size) < 1:
        raise MogeError(f"infer_panoramas: batch_size {batch_size} must be positive")
    _check_images("infer_panoramas", images)
    return _infer("infer_panoramas", model, images, batch_size, return_views)
