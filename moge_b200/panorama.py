"""Panorama inference on the GPU: the reference's `moge/scripts/infer_panorama.py:83-122` without file I/O, and the device side of
its `moge/utils/panorama.py`.

An equirectangular panorama is split into 12 perspective views (one camera per icosahedron vertex, 90 x 90 degrees), the views go
through one `model.infer(views, fov_x=..., apply_mask=False)` call, and the views' log-distances are merged back into a panorama
by a gradient-domain least-squares solve (SciPy's LSMR on a 4-level pyramid at up to 1920 x 960), then resized to the input.

The batch forms (`split_panoramas`, `merge_panoramas`, `finish_panoramas`, `infer_panoramas`) take up to 64 panoramas of one size
with the same cameras, and `infer_panoramas_many` takes a list of up to 64 panoramas of any sizes.  Every stage is one launch
over all the panoramas of a call; the merge solves every panorama's system of a pyramid level in one cooperative launch, with
the pyramids of different sizes aligned at their finest level (see _schedule).  The single-panorama and one-size functions run
the same code over a list of one size, so each panorama of a call gets bitwise what its single call gives it.

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
           "finish_panoramas", "infer_panoramas", "infer_panoramas_many", "SPLIT_RESOLUTION", "MAX_BATCH"]

SPLIT_RESOLUTION = 512                 # infer_panorama.py:90
MERGE_WIDTH, MERGE_HEIGHT = 1920, 960  # infer_panorama.py:117
PYRAMID_SIZE = 256                     # panorama.py:106: a level recurses while max(w, h) > 256
MAX_PIXELS = 1 << 28
MAX_BATCH = 64                         # panoramas per call (MOGE_PANORAMA_MAX_BATCH)


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


def _check_list(what: str, images, device) -> List[Tuple[int, int]]:
    """The (H, W) of each panorama of the list `images`, after checking it as infer_panoramas_many takes it: 1 to MAX_BATCH
    (H, W, 3) uint8 CUDA tensors on `device` (None: the first panorama's device).  An error names the offending panorama."""
    if not isinstance(images, (list, tuple)):
        raise MogeError(f"{what}: images must be a list of (H, W, 3) uint8 tensors, not {type(images).__name__}")
    if not 1 <= len(images) <= MAX_BATCH:
        raise MogeError(f"{what}: a list of {len(images)} panoramas is outside [1, {MAX_BATCH}]")
    sizes = []
    for k, image in enumerate(images):
        name = f"{what}: panorama {k}"
        if not isinstance(image, torch.Tensor) or image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
            raise MogeError(f"{name} must be a (H, W, 3) uint8 tensor")
        capi.require_cuda(name, image)
        device = image.device if device is None else device
        if image.device != device:
            raise MogeError(f"{name} is on {image.device}, not on {device}")
        H, W = image.shape[:2]
        _check_size(name, H, W)
        sizes.append((H, W))
    return sizes


# Each stage has one implementation over a list of P panoramas (_split, _merge, _finish, _infer), called after the public
# function's own argument checks with the name it raises under.  The one-size functions pass their batch as a list of one size
# (a single panorama as a list of one) and view the results with a leading dimension, or drop it.

def _ptr(t: torch.Tensor, offset: int = 0) -> int:
    """The device address of element `offset` of the flat contiguous tensor t."""
    return t.data_ptr() + offset * t.element_size()


# ------------------------------------------------------------------------------------------------------------ split
def _split(what: str, images: Sequence[torch.Tensor], extrinsics, intrinsics, resolution: int, return_uint8: bool):
    """The views (P, N, 3, res, res) of the P panoramas `images`, (H_i, W_i, 3) uint8 on one device, in one launch."""
    P = len(images)
    if not 1 <= int(resolution) <= 8192:
        raise MogeError(f"{what}: resolution {resolution} is outside [1, 8192]")
    res = int(resolution)
    if extrinsics is None:
        extrinsics, intrinsics = _default_cameras()
    cams, n = _cameras(extrinsics, intrinsics)
    dev = images[0].device
    with torch.cuda.device(dev):
        imgs = [image.contiguous() for image in images]
        out = torch.empty(P, n, 3, res, res, dtype=torch.float32, device=dev)
        u8 = torch.empty(P, n, res, res, 3, dtype=torch.uint8, device=dev) if return_uint8 else None
        grid = _table("grid", (res, res), dev)
        panos = (capi.PanoramaSplit * P)()
        for k, image in enumerate(imgs):
            panos[k].image, panos[k].H, panos[k].W, panos[k].view0 = image.data_ptr(), image.shape[0], image.shape[1], k * n
        capi.check(capi.lib().moge_panorama_split_groups(panos, P, cams, n, grid.data_ptr(), res, out.data_ptr(), capi.ptr(u8),
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
    out, u8 = _split("split_panorama", [image], extrinsics, intrinsics, resolution, return_uint8)
    return (out[0], u8[0]) if return_uint8 else out[0]


def split_panoramas(images: torch.Tensor, extrinsics=None, intrinsics=None, resolution: int = SPLIT_RESOLUTION,
                    return_uint8: bool = False):
    """split_panorama of P panoramas of one size in one launch: images (P, H, W, 3) uint8 RGB CUDA tensor -> views
    (P, N, 3, res, res) float32, and with return_uint8 also (P, N, res, res, 3) uint8; each panorama's views are bitwise its
    split_panorama."""
    _check_images("split_panoramas", images)
    out, u8 = _split("split_panoramas", list(images.contiguous()), extrinsics, intrinsics, resolution, return_uint8)
    return (out, u8) if return_uint8 else out


# ------------------------------------------------------------------------------------------------------------ merge
def _levels(width: int, height: int) -> List[Tuple[int, int]]:
    sizes = [(width, height)]
    while max(sizes[-1]) > PYRAMID_SIZE:
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    return sizes[::-1]


def _schedule(sizes: Sequence[Tuple[int, int]]) -> Tuple[List[List[Tuple[int, int]]], List[List[Tuple[int, int]]]]:
    """The merge launches of panoramas merged at sizes[i] = (width, height).  Panorama i has the L_i pyramid levels of
    _levels (coarsest first); launch k of K = max L_i solves level k - (K - L_i) of every panorama that has one, so the
    pyramids line up at their finest level and the last launch solves every panorama at its merge size.  Each panorama still
    sees its own levels in order, each started from its own previous level.  Returns (the levels of each panorama, per launch
    the (panorama, level index) pairs in input order)."""
    levels = [_levels(w, h) for w, h in sizes]
    K = max(len(lv) for lv in levels)
    return levels, [[(i, k - (K - len(lv))) for i, lv in enumerate(levels) if k >= K - len(lv)] for k in range(K)]


_last: Dict[str, object] = {}


def num_rows(h: int, w: int) -> int:
    """Rows of a level's system: x-gradient h*w, y-gradient (h-1) x (w+1) on the reference's x-wrapped grid (column w repeats
    column 0), Laplacian h*w."""
    return 2 * h * w + (h - 1) * (w + 1)


def _offsets(counts: Sequence[int]) -> List[int]:
    out, total = [], 0
    for c in counts:
        out.append(total)
        total += c
    return out


def _merge(what: str, sizes: Sequence[Tuple[int, int]], src: torch.Tensor, mask: torch.Tensor, extrinsics, intrinsics,
           return_levels: bool):
    """The merges of src (P, N, vh, vw[, 3]) and mask (P, N, vh, vw), whose types and shapes the caller has checked, panorama i
    at sizes[i] = (width, height).  Returns the final depth and mask of every panorama back to back in flat tensors, in input
    order, and with return_levels per launch of _schedule a dict of its members and its flat b, row_mask and depth."""
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
    levels, launches = _schedule(sizes)
    with torch.cuda.device(dev):
        st = capi.current_stream()
        s = src.detach().contiguous()
        m = capi.mask_u8(mask)
        finest = (capi.PanoramaLevel * P)()
        for i, (w, h) in enumerate(sizes):
            finest[i].h, finest[i].w = h, w
        ws = capi.workspace(L.moge_panorama_workspace_bytes_groups, finest, P, n, device=dev)
        stats = torch.zeros(len(launches), P, 2, dtype=torch.int32, device=dev)
        # the initial guesses of the next launch: the buffer (kept until that launch is queued) and each member's address in it
        init_buf, init_at, out = None, {}, []
        for k, members in enumerate(launches):
            shapes = [levels[i][j] for i, j in members]
            pixels = [w * h for w, h in shapes]
            rows = [num_rows(h, w) for w, h in shapes]
            po, ro = _offsets(pixels), _offsets(rows)
            b = torch.empty(sum(rows), dtype=torch.float64, device=dev)
            rm = torch.empty(sum(rows), dtype=torch.uint8, device=dev)
            pm = torch.empty(sum(pixels), dtype=torch.uint8, device=dev)
            depth = torch.empty(sum(pixels), dtype=torch.float32, device=dev)
            lv = (capi.PanoramaLevel * len(members))()
            for e, ((i, j), (w, h)) in enumerate(zip(members, shapes)):
                lv[e].h, lv[e].w, lv[e].view0 = h, w, i * n
                lv[e].directions = _table("dirs", (h, w), dev).data_ptr()
                lv[e].b, lv[e].row_mask = _ptr(b, ro[e]), _ptr(rm, ro[e])
                lv[e].pano_mask, lv[e].depth = _ptr(pm, po[e]), _ptr(depth, po[e])
                lv[e].init = init_at.get(i)              # None at a panorama's coarsest level
                lv[e].stats = _ptr(stats, (k * P + i) * 2)
            capi.check(L.moge_panorama_rhs_groups(s.data_ptr(), channels, m.data_ptr(), n, vh, vw, cams, lv, len(members),
                                                  ws.data_ptr(), ws.numel(), st))
            capi.check(L.moge_panorama_lsmr_groups(lv, len(members), ws.data_ptr(), ws.numel(), st))
            if return_levels:
                out.append({"members": members, "sizes": shapes, "b": b, "row_mask": rm, "depth": depth})
            if k + 1 < len(launches):
                # every member of this launch is in the next one, one level finer: its initial guess is this depth, upsampled
                nxt = [levels[i][j + 1] for i, j in members]
                npix = [w * h for w, h in nxt]
                io = _offsets(npix)
                init_buf = torch.empty(sum(npix), dtype=torch.float32, device=dev)
                init_at = {i: _ptr(init_buf, io[e]) for e, (i, _) in enumerate(members)}
                maps = (capi.PanoramaResize * len(members))()
                for e, ((i, _), (w, h), (W2, H2)) in enumerate(zip(members, shapes, nxt)):
                    maps[e].src, maps[e].h, maps[e].w = _ptr(depth, po[e]), h, w
                    maps[e].dst, maps[e].H, maps[e].W = init_at[i], H2, W2
                capi.check(L.moge_panorama_resize_groups(maps, len(members), st))
    _last.update(levels=levels, stats=stats, single=False)
    return depth, pm.view(torch.bool), out


def _one_size_levels(levels: list, P: int) -> list:
    """The per-launch records of a one-size merge as merge_panoramas returns them: per level its size and b, row_mask and
    depth with a leading P."""
    return [{"width": lv["sizes"][0][0], "height": lv["sizes"][0][1], "b": lv["b"].view(P, -1), "row_mask": lv["row_mask"].view(P, -1),
             "depth": lv["depth"].view(P, lv["sizes"][0][1], lv["sizes"][0][0])} for lv in levels]


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
    depth, pm, levels = _merge("merge_panorama", [(width, height)], src[None], mask[None], extrinsics, intrinsics, return_levels)
    _last["single"] = True
    result = (depth.view(height, width), pm.view(height, width))
    if return_levels:
        return (*result, [{k: v[0] if isinstance(v, torch.Tensor) else v for k, v in lv.items()} for lv in _one_size_levels(levels, 1)])
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
    P = src.shape[0]
    depth, pm, levels = _merge("merge_panoramas", [(width, height)] * P, src, mask, extrinsics, intrinsics, return_levels)
    result = (depth.view(P, height, width), pm.view(P, height, width))
    return (*result, _one_size_levels(levels, P)) if return_levels else result


def last_merge_stats() -> list:
    """Per level of the most recent merge on this process, coarsest first: width, height, LSMR iterations and istop (SciPy's
    stopping reason).  After merge_panoramas, infer_panoramas or infer_panoramas_many, one such list per panorama, each with
    that panorama's own levels.  Reading them copies the counters to the host."""
    if not _last:
        return []
    stats = _last["stats"].cpu().tolist()            # (launches, P, 2)
    K = len(stats)
    per = [[{"width": w, "height": h, "iterations": stats[K - len(lv) + j][i][0], "istop": stats[K - len(lv) + j][i][1]}
            for j, (w, h) in enumerate(lv)] for i, lv in enumerate(_last["levels"])]
    return per[0] if _last["single"] else per


# ------------------------------------------------------------------------------------------------------------ finish
def _finish(what: str, depth: Sequence[torch.Tensor], mask: Sequence[torch.Tensor], sizes: Sequence[Tuple[int, int]], stacked: bool):
    """The merged depth[i] and mask[i] (h_i, w_i) resized to sizes[i] = (H_i, W_i), and the points, in one launch.  With stacked
    (every size equal) the outputs are (P, H, W[, 3]) tensors, otherwise lists of per-panorama tensors."""
    P = len(depth)
    for d, (H, W) in zip(depth, sizes):
        _check_size(what, *d.shape)
        _check_size(what, H, W)
    dev = depth[0].device
    with torch.cuda.device(dev):
        ds = [d.contiguous() for d in depth]
        ms = [capi.mask_u8(m) for m in mask]
        if stacked:
            H, W = sizes[0]
            out_d = torch.empty(P, H, W, dtype=torch.float32, device=dev)
            out_m = torch.empty(P, H, W, dtype=torch.uint8, device=dev)
            points = torch.empty(P, H, W, 3, dtype=torch.float32, device=dev)
        else:
            out_d = [torch.empty(H, W, dtype=torch.float32, device=dev) for H, W in sizes]
            out_m = [torch.empty(H, W, dtype=torch.uint8, device=dev) for H, W in sizes]
            points = [torch.empty(H, W, 3, dtype=torch.float32, device=dev) for H, W in sizes]
        maps = (capi.PanoramaFinish * P)()
        for k, (H, W) in enumerate(sizes):
            f = maps[k]
            f.depth, f.mask, (f.h, f.w), f.H, f.W = ds[k].data_ptr(), ms[k].data_ptr(), ds[k].shape, H, W
            f.depth_out, f.mask_out, f.points = out_d[k].data_ptr(), out_m[k].data_ptr(), points[k].data_ptr()
        capi.check(capi.lib().moge_panorama_finish_groups(maps, P, capi.current_stream()))
    if stacked:
        return out_d, out_m.view(torch.bool), points
    return out_d, [m.view(torch.bool) for m in out_m], points


def finish_panorama(depth: torch.Tensor, mask: torch.Tensor, height: int, width: int):
    """infer_panorama.py:119-122: the merged depth and mask resized to (height, width) as cv2.resize does, and the points."""
    capi.require_cuda("finish_panorama", depth, mask)
    if depth.dtype != torch.float32 or depth.dim() != 2 or tuple(mask.shape) != tuple(depth.shape):
        raise MogeError("finish_panorama: depth must be float32 (h, w) and mask (h, w)")
    return tuple(t[0] for t in _finish("finish_panorama", [depth], [mask], [(int(height), int(width))], True))


def finish_panoramas(depth: torch.Tensor, mask: torch.Tensor, height: int, width: int):
    """finish_panorama of P merged maps: depth (P, h, w) float32 and mask (P, h, w) -> depth (P, height, width), mask
    (P, height, width) bool and points (P, height, width, 3)."""
    if not isinstance(depth, torch.Tensor) or not isinstance(mask, torch.Tensor) or depth.dtype != torch.float32 or depth.dim() != 3 \
            or tuple(mask.shape) != tuple(depth.shape):
        raise MogeError("finish_panoramas: depth must be float32 (P, h, w) and mask (P, h, w)")
    _check_batch("finish_panoramas", depth.shape[0])
    capi.require_cuda("finish_panoramas", depth, mask)
    P = depth.shape[0]
    return _finish("finish_panoramas", list(depth), list(mask), [(int(height), int(width))] * P, True)


# ------------------------------------------------------------------------------------------------------------ end to end
def _fov_x(intrinsics, device) -> torch.Tensor:
    """infer_panorama.py:99-100: the views' horizontal fields of view in degrees, float32."""
    K = np.asarray(intrinsics)
    fov_x = np.rad2deg(2 * np.arctan(0.5 / K[..., 0, 0]))
    return torch.tensor(fov_x, dtype=torch.float32, device=device)


def _infer(what: str, model, images: Sequence[torch.Tensor], batch_size: Optional[int], return_views: bool, stacked: bool):
    """The panoramas `images` ((H_i, W_i, 3) uint8 on one device) end to end: one split launch, the 12P views through
    model.infer in one call or calls of batch_size views, the merge launches of _schedule and one finish launch.  With stacked
    (every size equal) one dict of (P, ...) tensors, otherwise one dict per panorama."""
    P = len(images)
    shapes = [tuple(image.shape[:2]) for image in images]
    extrinsics, intrinsics = _default_cameras()
    views, views_u8 = _split(what, images, extrinsics, intrinsics, SPLIT_RESOLUTION, return_views)
    n = views.shape[1]
    flat = views.view(P * n, *views.shape[2:])
    fov_x = _fov_x(intrinsics, images[0].device).repeat(P)
    step = len(flat) if batch_size is None else int(batch_size)
    points, masks = [], []
    for lo in range(0, len(flat), step):
        out = model.infer(flat[lo:lo + step], fov_x=fov_x[lo:lo + step], apply_mask=False)
        points.append(out['points'])
        masks.append(out['mask'])
    points = points[0] if len(points) == 1 else torch.cat(points)
    masks = masks[0] if len(masks) == 1 else torch.cat(masks)
    view_points, view_masks = points.reshape(P, n, *points.shape[1:]), masks.reshape(P, n, *masks.shape[1:])
    sizes = [(min(MERGE_WIDTH, W), min(MERGE_HEIGHT, H)) for H, W in shapes]
    depth, mask, _ = _merge(what, sizes, view_points, view_masks, extrinsics, intrinsics, False)
    pixels = [w * h for w, h in sizes]
    depth = [d.view(h, w) for d, (w, h) in zip(depth.split(pixels), sizes)]
    mask = [m.view(h, w) for m, (w, h) in zip(mask.split(pixels), sizes)]
    depth, mask, points = _finish(what, depth, mask, shapes, stacked)
    if stacked:
        out = {'depth': depth, 'mask': mask, 'points': points}
        if return_views:
            out.update(views=views_u8, view_distance=view_points.norm(dim=-1), view_mask=view_masks)
        return out
    outs = [{'depth': depth[k], 'mask': mask[k], 'points': points[k]} for k in range(P)]
    if return_views:
        view_distance = view_points.norm(dim=-1)
        for k, out in enumerate(outs):
            out.update(views=views_u8[k], view_distance=view_distance[k], view_mask=view_masks[k])
    return outs


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
    out = _infer("infer_panorama", model, [image], batch_size, return_views, True)
    _last["single"] = True
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
    return _infer("infer_panoramas", model, list(images.contiguous()), batch_size, return_views, True)


def infer_panoramas_many(model, images: Sequence[torch.Tensor], batch_size: Optional[int] = None,
                         return_views: bool = False) -> List[Dict[str, torch.Tensor]]:
    """infer_panorama of a list of 1 to 64 panoramas of any sizes: images[i] is a (H_i, W_i, 3) uint8 RGB CUDA tensor on the
    model's device.  One split launch covers every panorama; the 12P views go through `model.infer(views, fov_x=...,
    apply_mask=False)` in one call, or in calls of batch_size views that may straddle panoramas; each merge level is one
    cooperative launch over every panorama that has it (the pyramids of different sizes line up at their finest level, see
    _schedule); one finish launch writes every output.  Returns one dict per panorama, in input order, with the keys and shapes
    of infer_panorama's; each is bitwise that panorama's infer_panorama.  last_merge_stats() then gives one per-level list per
    panorama, each with its own levels.  Larger collections go in several calls: an 8K panorama's outputs alone take 0.5 GB.
    Every argument is checked before any device work; an error names the offending panorama's index."""
    what = "infer_panoramas_many"
    if batch_size is not None and int(batch_size) < 1:
        raise MogeError(f"{what}: batch_size {batch_size} must be positive")
    device = getattr(model, "device", None)
    device = device if isinstance(device, torch.device) and device.type == "cuda" else None
    _check_list(what, images, device)
    return _infer(what, model, list(images), batch_size, return_views, False)
