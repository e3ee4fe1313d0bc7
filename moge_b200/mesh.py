"""Mesh export on the GPU: utils3d's `depth_map_edge` and `build_mesh_from_map` as the reference's CLI calls them
(moge/scripts/infer.py:124-150), and that whole step after `infer()` as `mesh_from_output`.

The work runs in moge_b200/csrc/mesh.cu: an edge / cleaned-mask kernel, a count pass with a per-image scan of tile counts, and
emit passes for the vertex rows and the faces.  A mesh call copies one small buffer of per-image totals to pinned host memory
and waits for it (the only synchronisation of a call, for the whole batch), allocates exact-size outputs as views of one
allocation and launches the emit passes.  Results are bitwise those of the numpy restatement in oracle/utils3d_mesh.py.

The panorama script's export (moge/scripts/infer_panorama.py:136-150) adds utils3d's `point_map_to_normal_map` and
`normal_map_edge` and is `mesh_from_panorama`: a normal-map kernel and a normal-edge kernel whose fused form writes the cleaned
mask, then the same count and emit passes.  The normals are bitwise those of oracle/utils3d_normals.py; the normal edges may
differ only where an angle is within a few ulp of the threshold (acosf against numpy's arccos).

CUDA tensors only; there is no CPU fallback.  Divergences from utils3d: faces are int32 (utils3d returns intp), and attribute
maps must be fp32 (uint8 colours go through `mesh_from_output` / `mesh_from_panorama`).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import capi
from .capi import MogeError

__all__ = ["depth_map_edge", "build_mesh_from_map", "build_mesh_from_map_batch", "mesh_from_output", "point_map_to_normal_map",
           "normal_map_edge", "mesh_from_panorama"]

MAX_PIXELS = 1 << 30           # per image: vertex ids and triangle counts stay below 2^31
KERNEL_SIZES = (3, 5, 7)
GL_FLIP = (1.0, -1.0, -1.0)    # OpenGL conventions (infer.py:148-150): x right, y up, z backward
UV_FLIP, UV_OFFSET = (1.0, -1.0), (0.0, 1.0)


def _f32(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise MogeError(f"{what} must be float32, not {t.dtype}")
    return t.detach().contiguous()


def _tol(v) -> Optional[C.c_float]:
    return None if v is None else C.c_float(float(v))       # compared as fp32, as numpy compares a Python float with fp32


def _edge(depth: torch.Tensor, mask: Optional[torch.Tensor], keep: Optional[torch.Tensor], atol, rtol, kernel_size: int) -> torch.Tensor:
    B, H, W = depth.shape
    out = torch.empty(B, H, W, dtype=torch.uint8, device=depth.device)
    a, r = _tol(atol), _tol(rtol)
    capi.check(capi.lib().moge_depth_edge(depth.data_ptr(), capi.ptr(mask), capi.ptr(keep), B, H, W, int(kernel_size),
                                          None if a is None else C.byref(a), None if r is None else C.byref(r), out.data_ptr(),
                                          capi.current_stream()))
    return out


def depth_map_edge(depth: torch.Tensor, atol: float = None, rtol: float = None, kernel_size: int = 3,
                   mask: torch.Tensor = None) -> torch.Tensor:
    """utils3d's depth_map_edge on a (..., H, W) fp32 depth: True where max(d) + max(-d) over the kernel_size window exceeds atol,
    or exceeds rtol times d (each test only when its tolerance is given).  With `mask`, the window sees only masked-in pixels.
    kernel_size is 3, 5 or 7."""
    if kernel_size not in KERNEL_SIZES:
        raise MogeError(f"depth_map_edge: kernel_size {kernel_size} is not one of 3, 5, 7")
    if not isinstance(depth, torch.Tensor) or depth.dim() < 2:
        raise MogeError("depth_map_edge: depth must be a (..., H, W) tensor")
    if mask is not None and mask.shape != depth.shape:
        raise MogeError(f"depth_map_edge: mask {tuple(mask.shape)} does not match depth {tuple(depth.shape)}")
    H, W = depth.shape[-2:]
    capi.check_pixels("depth_map_edge", H, W, MAX_PIXELS)
    capi.require_cuda("moge_b200.mesh", depth, mask)
    d = _f32(depth, "depth").reshape(-1, H, W)
    m = None if mask is None else capi.mask_u8(mask).reshape(-1, H, W)
    if d.shape[0] == 0:
        return torch.zeros(depth.shape, dtype=torch.bool, device=depth.device)
    return _edge(d, m, None, atol, rtol, kernel_size).view(torch.bool).reshape(depth.shape)


# ------------------------------------------------------------------------------------------------------------ mesh core
class _Map:
    """One attribute map of a build: a (B, H, W, C) / (B, C, H, W) source, or None for the generated UV."""

    def __init__(self, src: Optional[torch.Tensor], kind: int, channels: int, layout: int = capi.MESH_HWC,
                 sign: Sequence[float] = (), offset: Sequence[float] = (), squeeze: bool = False):
        self.src, self.kind, self.channels, self.layout = src, kind, channels, layout
        self.sign = list(sign) + [1.0] * (capi.MESH_MAX_CHANNELS - len(sign))
        self.offset = list(offset) + [0.0] * (capi.MESH_MAX_CHANNELS - len(offset))
        self.squeeze = squeeze        # a (H, W) map: rows come back as (N,)


def _count(mask: Optional[torch.Tensor], B: int, H: int, W: int, dev):
    """Count pass and the one device-to-host copy: returns (workspace, device totals, pinned host totals, event)."""
    L = capi.lib()
    ws = capi.workspace(L.moge_mesh_workspace_bytes, B, H, W, device=dev)
    totals = torch.empty(B, 4, dtype=torch.int64, device=dev)
    capi.check(L.moge_mesh_count(capi.ptr(mask), B, H, W, totals.data_ptr(), ws.data_ptr(), ws.numel(), capi.current_stream()))
    host = torch.empty(B, 4, dtype=torch.int64, pin_memory=True)
    host.copy_(totals, non_blocking=True)
    event = torch.cuda.Event()
    event.record()
    return ws, totals, host, event


def _emit(mask: Optional[torch.Tensor], B: int, H: int, W: int, maps: List[_Map], tri: bool, ws: torch.Tensor, totals: torch.Tensor,
          faces: torch.Tensor, rows: List[torch.Tensor]) -> None:
    """Launch the emit passes into exact-size outputs: faces and one (total vertices, C) fp32 buffer per map."""
    descs = (capi.MeshMap * max(1, len(maps)))()
    for k, m in enumerate(maps):
        descs[k].src = None if m.src is None else m.src.data_ptr()
        descs[k].kind, descs[k].channels, descs[k].layout = m.kind, m.channels, m.layout
        for c in range(capi.MESH_MAX_CHANNELS):
            descs[k].sign[c], descs[k].offset[c] = m.sign[c], m.offset[c]
        descs[k].dst = rows[k].data_ptr()
    capi.check(capi.lib().moge_mesh_build(capi.ptr(mask), B, H, W, int(bool(tri)), descs, len(maps), totals.data_ptr(),
                                          faces.data_ptr(), ws.data_ptr(), ws.numel(), capi.current_stream()))


def _build(mask: Optional[torch.Tensor], B: int, H: int, W: int, maps: List[_Map], tri: bool, counted) -> List[Tuple[torch.Tensor, ...]]:
    """Emit pass after _count: one allocation for every image's faces and rows, returned as per-image (faces, *rows) views."""
    ws, totals, host, event = counted
    dev = ws.device
    event.synchronize()
    t = host.numpy()
    nv, nq = t[:, 0].astype(np.int64), t[:, 1].astype(np.int64)
    per = 3 if tri else 4
    nf = nq * (2 if tri else 1)
    V, F = int(nv.sum()), int(nf.sum())
    words = F * per + sum(V * m.channels for m in maps)
    buf = torch.empty(max(words, 1), dtype=torch.int32, device=dev)
    faces = buf[:F * per].view(F, per)
    rows, at = [], F * per
    for m in maps:
        rows.append(buf[at:at + V * m.channels].view(torch.float32).view(V, m.channels))
        at += V * m.channels
    if V:                  # no vertex anywhere: no face either, and nothing to write
        _emit(mask, B, H, W, maps, tri, ws, totals, faces, rows)
    out = []
    v0 = np.concatenate([[0], np.cumsum(nv)])
    f0 = np.concatenate([[0], np.cumsum(nf)])
    for b in range(B):
        item = [faces[f0[b]:f0[b + 1]]]
        for m, r in zip(maps, rows):
            x = r[v0[b]:v0[b + 1]]
            item.append(x[:, 0] if m.squeeze else x)
        out.append(tuple(item))
    return out


def _mesh(mask: Optional[torch.Tensor], B: int, H: int, W: int, maps: List[_Map], tri: bool, dev):
    return _build(mask, B, H, W, maps, tri, _count(mask, B, H, W, dev))


def _map_args(maps, lead: int, what: str):
    """Validate the shapes of (lead..., H, W[, C]) maps; returns (H, W, [_Map]) with the sources still to be checked by _sources."""
    if not maps:
        raise MogeError(f"{what}: at least one map is needed")
    for m in maps:
        if not isinstance(m, torch.Tensor) or m.dim() not in (lead + 2, lead + 3):
            raise MogeError(f"{what}: maps must be {'(B, ' if lead else '('}H, W[, C]) tensors")
    shape = maps[0].shape[:lead + 2]
    for m in maps:
        if m.shape[:lead + 2] != shape:
            raise MogeError(f"{what}: map shapes {tuple(m.shape)} and {tuple(maps[0].shape)} do not match")
        if m.dim() == lead + 3 and not 1 <= m.shape[-1] <= capi.MESH_MAX_CHANNELS:
            raise MogeError(f"{what}: maps have 1 to {capi.MESH_MAX_CHANNELS} channels, not {m.shape[-1]}")
    if len(maps) > capi.MESH_MAX_MAPS:
        raise MogeError(f"{what}: at most {capi.MESH_MAX_MAPS} maps")
    H, W = shape[lead], shape[lead + 1]
    capi.check_pixels(what, H, W, MAX_PIXELS)
    out = []
    for m in maps:
        out.append(_Map(m, capi.MESH_F32, 1 if m.dim() == lead + 2 else m.shape[-1], squeeze=m.dim() == lead + 2))
    return H, W, out


def _sources(ms: List[_Map], mask: Optional[torch.Tensor], what: str) -> None:
    """After every shape check: the maps and the mask are CUDA tensors, the maps fp32 and contiguous."""
    capi.require_cuda("moge_b200.mesh", mask, *[m.src for m in ms])
    for m in ms:
        m.src = _f32(m.src, f"{what}: every map")


def build_mesh_from_map(*maps: torch.Tensor, mask: torch.Tensor = None, tri: bool = False) -> Tuple[torch.Tensor, ...]:
    """utils3d's build_mesh_from_map on one image: maps (H, W[, C]) fp32.  Returns (faces int32 (F, 3 or 4), *rows), the rows of
    each map at the kept vertices.  A quad is kept when its four corners are in `mask` (every quad without one)."""
    H, W, ms = _map_args(maps, 0, "build_mesh_from_map")
    if mask is not None and tuple(mask.shape) != (H, W):
        raise MogeError(f"build_mesh_from_map: mask {tuple(mask.shape)} does not match the maps {(H, W)}")
    _sources(ms, mask, "build_mesh_from_map")
    m = None if mask is None else capi.mask_u8(mask)[None]
    return _mesh(m, 1, H, W, ms, tri, maps[0].device)[0]


def build_mesh_from_map_batch(*maps: torch.Tensor, mask: torch.Tensor = None, tri: bool = False) -> List[Tuple[torch.Tensor, ...]]:
    """build_mesh_from_map over a same-shape stack: maps (B, H, W[, C]), mask (B, H, W).  One host synchronisation for the batch;
    returns B tuples, all views of one allocation, each bitwise equal to the single-image call."""
    H, W, ms = _map_args(maps, 1, "build_mesh_from_map_batch")
    B = maps[0].shape[0]
    if mask is not None and tuple(mask.shape) != (B, H, W):
        raise MogeError(f"build_mesh_from_map_batch: mask {tuple(mask.shape)} does not match the maps {(B, H, W)}")
    _sources(ms, mask, "build_mesh_from_map_batch")
    if B == 0:
        return []
    return _mesh(capi.mask_u8(mask), B, H, W, ms, tri, maps[0].device)


# ------------------------------------------------------------------------------------------------------------ after infer()
def _output_maps(points: torch.Tensor, colour: _Map, normal: Optional[torch.Tensor]) -> List[_Map]:
    """infer.py's attribute maps in OpenGL conventions: points, colours, the generated UV and the normals if any."""
    maps = [_Map(_f32(points, "points"), capi.MESH_F32, 3, sign=GL_FLIP), colour,
            _Map(None, capi.MESH_UV, 2, sign=UV_FLIP, offset=UV_OFFSET)]
    if normal is not None:
        maps.append(_Map(_f32(normal, "normal"), capi.MESH_F32, 3, sign=GL_FLIP))
    return maps


def mesh_from_output(output: Dict[str, torch.Tensor], image: torch.Tensor, threshold: float = 0.04, remove_edge: bool = True):
    """infer.py:126-150 in one call: from infer()'s output (points, depth, mask and, with a normal head, normal; batched or not)
    and the input image, either uint8 (H, W, 3) / (B, H, W, 3) or the float32 (3, H, W) / (B, 3, H, W) tensor given to infer()
    (uint8 colours are c / 255 in fp32, float colours are taken as they are).  The mask is cleaned at depth edges
    (mask & ~depth_map_edge(depth, rtol=threshold)) unless remove_edge is False.

    Returns, per image, a dict of `faces` (int32 triangles), `vertices`, `vertex_colors`, `vertex_uvs`, `vertex_normals` (only
    with normals) and `mask_cleaned`, already in OpenGL conventions; a list for a batched output, one dict otherwise."""
    points, depth, mask = output["points"], output["depth"], output["mask"]
    normal = output.get("normal")
    batched = depth.dim() == 3
    if not batched:
        points, depth, mask = points[None], depth[None], mask[None]
        normal = None if normal is None else normal[None]
        image = image[None] if isinstance(image, torch.Tensor) else image
    if depth.dim() != 3:
        raise MogeError("mesh_from_output: depth must be (H, W) or (B, H, W)")
    B, H, W = depth.shape
    for name, t, want in (("points", points, (B, H, W, 3)), ("mask", mask, (B, H, W)), ("normal", normal, (B, H, W, 3))):
        if t is not None and tuple(t.shape) != want:
            raise MogeError(f"mesh_from_output: {name} has shape {tuple(t.shape)}, expected {want}")
    if not isinstance(image, torch.Tensor):
        raise MogeError("mesh_from_output: image must be a CUDA tensor")
    if image.dtype == torch.uint8 and tuple(image.shape) == (B, H, W, 3):
        colour = _Map(image.contiguous(), capi.MESH_U8_UNIT, 3, capi.MESH_HWC)
    elif image.dtype == torch.float32 and tuple(image.shape) == (B, 3, H, W):
        colour = _Map(image.detach().contiguous(), capi.MESH_F32, 3, capi.MESH_CHW)
    else:
        raise MogeError(f"mesh_from_output: image must be uint8 (H, W, 3) or float32 (3, H, W) matching the maps, not "
                        f"{image.dtype} {tuple(image.shape[1:])}")
    capi.check_pixels("mesh_from_output", H, W, MAX_PIXELS)
    capi.require_cuda("moge_b200.mesh", points, depth, mask, normal, image)
    d = _f32(depth, "depth")
    m = capi.mask_u8(mask)
    cleaned = _edge(d, None, m, None, threshold, 3) if remove_edge else m.clone()
    maps = _output_maps(points, colour, normal)
    results = []
    for b, (faces, vertices, colours, uvs, *rest) in enumerate(_mesh(cleaned, B, H, W, maps, True, d.device)):
        r = {"faces": faces, "vertices": vertices, "vertex_colors": colours, "vertex_uvs": uvs}
        if normal is not None:
            r["vertex_normals"] = rest[0]
        r["mask_cleaned"] = cleaned[b].view(torch.bool)
        results.append(r)
    return results if batched else results[0]


# ------------------------------------------------------------------------------------------------------------ normals
def _normal_map(points: torch.Tensor, mask: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(B, H, W, 3) fp32 points, (B, H, W) uint8 mask or None -> (normals, uint8 normal mask)."""
    B, H, W = points.shape[:3]
    normal = torch.empty(B, H, W, 3, dtype=torch.float32, device=points.device)
    nmask = torch.empty(B, H, W, dtype=torch.uint8, device=points.device)
    capi.check(capi.lib().moge_normal_map(points.data_ptr(), capi.ptr(mask), B, H, W, normal.data_ptr(), nmask.data_ptr(),
                                          capi.current_stream()))
    return normal, nmask


def _normal_edge(normals: torch.Tensor, mask: Optional[torch.Tensor], and_edge: Optional[torch.Tensor], keep: Optional[torch.Tensor],
                 tol: float, kernel_size: int, angle: Optional[torch.Tensor] = None) -> torch.Tensor:
    B, H, W = normals.shape[:3]
    out = torch.empty(B, H, W, dtype=torch.uint8, device=normals.device)
    capi.check(capi.lib().moge_normal_edge(normals.data_ptr(), capi.ptr(mask), capi.ptr(and_edge), capi.ptr(keep), B, H, W,
                                           int(kernel_size), float(np.deg2rad(tol)), out.data_ptr(), capi.ptr(angle),
                                           capi.current_stream()))
    return out


def _check_normal_args(what: str, points: torch.Tensor, mask: Optional[torch.Tensor]) -> Tuple[int, int]:
    if not isinstance(points, torch.Tensor) or points.dim() < 3 or points.shape[-1] != 3:
        raise MogeError(f"{what}: expected a (..., H, W, 3) tensor")
    if mask is not None and (not isinstance(mask, torch.Tensor) or tuple(mask.shape) != tuple(points.shape[:-1])):
        raise MogeError(f"{what}: mask {tuple(getattr(mask, 'shape', ()))} does not match the map {tuple(points.shape[:-1])}")
    H, W = points.shape[-3:-1]
    capi.check_pixels(what, H, W, MAX_PIXELS)
    capi.require_cuda("moge_b200.mesh", points, mask)
    return H, W


def point_map_to_normal_map(points: torch.Tensor, mask: torch.Tensor = None, edge_threshold: float = None):
    """utils3d's point_map_to_normal_map on a (..., H, W, 3) fp32 point map: per pixel the normalised sum of the four normalised
    cross products up x left, left x down, down x right, right x up of the neighbour differences (no wrap at the borders).  With
    `mask` (..., H, W), a product counts when its two neighbours and the centre are in the mask, and (normals, normal_mask bool)
    is returned, normals 0 off normal_mask; without, every product counts, border ones against zero points, and only the normals
    are returned.  Bitwise the restatement in oracle/utils3d_normals.py.  edge_threshold is not supported."""
    if edge_threshold is not None:
        raise MogeError("point_map_to_normal_map: edge_threshold is not supported")
    H, W = _check_normal_args("point_map_to_normal_map", points, mask)
    p = _f32(points, "points").reshape(-1, H, W, 3)
    m = None if mask is None else capi.mask_u8(mask).reshape(-1, H, W)
    if p.shape[0] == 0:
        normal, nmask = torch.zeros_like(p), torch.zeros(p.shape[:3], dtype=torch.uint8, device=p.device)
    else:
        normal, nmask = _normal_map(p, m)
    normal = normal.reshape(points.shape)
    if mask is None:
        return normal
    return normal, nmask.view(torch.bool).reshape(mask.shape)


def normal_map_edge(normals: torch.Tensor, tol: float, kernel_size: int = 3, mask: torch.Tensor = None) -> torch.Tensor:
    """utils3d's normal_map_edge on (..., H, W, 3) fp32 normals: True where the largest angle between a normal and those of its
    kernel_size window (edge-padded; with `mask`, only the window's masked-in pixels), max-pooled over the same window, exceeds
    `tol` degrees.  A dot product beyond [-1, 1] gives a NaN angle, which the pooling spreads and which is never an edge.
    kernel_size is 3, 5 or 7."""
    if kernel_size not in KERNEL_SIZES:
        raise MogeError(f"normal_map_edge: kernel_size {kernel_size} is not one of 3, 5, 7")
    H, W = _check_normal_args("normal_map_edge", normals, mask)
    n = _f32(normals, "normals").reshape(-1, H, W, 3)
    m = None if mask is None else capi.mask_u8(mask).reshape(-1, H, W)
    if n.shape[0] == 0:
        return torch.zeros(normals.shape[:-1], dtype=torch.bool, device=normals.device)
    return _normal_edge(n, m, None, None, tol, kernel_size).view(torch.bool).reshape(normals.shape[:-1])


# ------------------------------------------------------------------------------------------------------------ after infer_panorama()
PANORAMA_NORMAL_TOL = 5.0       # infer_panorama.py:142: normal_map_edge(normals, tol=5, ...)


def mesh_from_panorama(output: Dict[str, torch.Tensor], image: torch.Tensor, threshold: float = 0.03) -> Dict[str, torch.Tensor]:
    """infer_panorama.py:136-144 in one call: from infer_panorama()'s output (points (H, W, 3), depth (H, W), mask (H, W)) and the
    (H, W, 3) uint8 panorama.  The mask is cleaned where a depth edge (rtol=threshold; inf: none) and a 5-degree normal edge
    coincide, mask & ~(depth_map_edge(depth, rtol=threshold) & normal_map_edge(normals, tol=5, mask=normals_mask)) with
    (normals, normals_mask) = point_map_to_normal_map(points, mask), and the mesh is built with colours image / 255 and the
    pixel-centre UVs.  No OpenGL flips, as the panorama script applies none.

    Returns a dict of `faces` (int32 triangles), `vertices`, `vertex_colors`, `vertex_uvs` and `mask_cleaned`, ready for
    save_glb(path, vertices, faces, vertex_uvs, image) and save_ply(path, vertices, faces, vertex_colors).  One host wait."""
    points, depth, mask = output["points"], output["depth"], output["mask"]
    if not isinstance(depth, torch.Tensor) or depth.dim() != 2:
        raise MogeError("mesh_from_panorama: depth must be a (H, W) tensor")
    H, W = depth.shape
    for name, t, want in (("points", points, (H, W, 3)), ("mask", mask, (H, W)), ("image", image, (H, W, 3))):
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != want:
            raise MogeError(f"mesh_from_panorama: {name} has shape {tuple(getattr(t, 'shape', ()))}, expected {want}")
    if image.dtype != torch.uint8:
        raise MogeError(f"mesh_from_panorama: image must be uint8, not {image.dtype}")
    capi.check_pixels("mesh_from_panorama", H, W, MAX_PIXELS)
    capi.require_cuda("moge_b200.mesh", points, depth, mask, image)
    d = _f32(depth, "depth")[None]
    p = _f32(points, "points")[None]
    m = capi.mask_u8(mask)[None]
    depth_edge = _edge(d, None, None, None, threshold, 3)
    normals, nmask = _normal_map(p, m)
    cleaned = _normal_edge(normals, nmask, depth_edge, m, PANORAMA_NORMAL_TOL, 3)
    maps = [_Map(p, capi.MESH_F32, 3), _Map(image.contiguous(), capi.MESH_U8_UNIT, 3), _Map(None, capi.MESH_UV, 2)]
    faces, vertices, colours, uvs = _mesh(cleaned, 1, H, W, maps, True, d.device)[0]
    return {"faces": faces, "vertices": vertices, "vertex_colors": colours, "vertex_uvs": uvs, "mask_cleaned": cleaned[0].view(torch.bool)}
