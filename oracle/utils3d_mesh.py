"""The two utils3d functions that the reference's mesh export calls (moge/scripts/infer.py:126-144, moge/scripts/app.py), and that
step itself, restated in numpy from utils3d's published semantics.  TEST INFRASTRUCTURE ONLY, and the host comparator of
tools/bench_mesh.py.

utils3d (pinned by the reference at 3fab839f) is not vendored, so no reference run pins these: parity at this boundary is
"unpinned" (DESIGN.md §2).  The quad corner order and the triangulation below are a restatement, not checked against the pinned
version.  The kernels of moge_b200/csrc/mesh.cu match this module bit for bit.

depth_map_edge(depth, atol=None, rtol=None, kernel_size=3, mask=None), depth (..., H, W) fp32:
  - diff = maxpool(depth) + maxpool(-depth) over the kernel_size x kernel_size window centred on the pixel, padded with -inf so
    that only in-image pixels count.  With `mask`, both pools see only the window's masked-in pixels (the others are -inf), so
    a window with none gives -inf.  np.max propagates NaN.
  - edge = (diff > atol) | (diff / depth > rtol), each term only when its tolerance is given; all False when neither is.
  - fp32 arithmetic with IEEE division.  The tolerance is compared as fp32: numpy casts a Python-float threshold to the array's
    fp32 (an fp32 array holding fp32(0.04) is not > the Python float fp32(0.04) - 1e-12, which would hold in fp64).
  - Infinities are part of the contract: infer(apply_mask=True) sets depth to +inf off the mask.  A finite pixel next to an inf
    one gets inf / d = inf and is an edge; an inf pixel gets inf / inf = NaN, not an edge; a window of only infs gets
    inf + (-inf) = NaN, not an edge.
  - kernel_size is odd, 3 to 7.

build_mesh_from_map(*maps, mask=None, tri=False), maps (H, W[, C]):
  - quads in row-major order of their top-left pixel, corners [(i, j), (i + 1, j), (i + 1, j + 1), (i, j + 1)]; a quad is kept
    when its four corners are in the mask (every quad without a mask);
  - a vertex is kept when a kept quad references it; kept vertices are numbered in row-major pixel order (np.unique's
    compaction);
  - tri=True: each quad [a, b, c, d] becomes [a, b, c], [a, c, d], interleaved per quad;
  - each map's rows are gathered at the kept vertices;
  - a map with fewer than two rows or columns has no faces: (0, 3) / (0, 4) faces and (0, C) attributes.
  Faces come back as int32 (utils3d returns intp; the engine returns int32, DESIGN.md §1d).

mesh_from_output: infer.py:126-150 on one image's maps: the cleaned mask, the mesh with colours uint8 / 255 (an fp32 division),
the pixel-centre UV map ((j + 0.5) / W, (i + 0.5) / H) in fp32 and the normals, then the OpenGL flips, which infer.py computes in
float64 (the integer lists promote): they are exact sign flips and 1 - v, so the fp32 cast of the result is the reference's value.
"""
import numpy as np


def _max_pool(x: np.ndarray, k: int) -> np.ndarray:
    r = k // 2
    pad = [(0, 0)] * (x.ndim - 2) + [(r, r), (r, r)]
    xp = np.pad(x, pad, mode="constant", constant_values=-np.inf)
    win = np.lib.stride_tricks.sliding_window_view(xp, (k, k), axis=(-2, -1))
    return win.max(axis=(-2, -1))


def depth_map_edge(depth: np.ndarray, atol=None, rtol=None, kernel_size: int = 3, mask: np.ndarray = None) -> np.ndarray:
    if kernel_size not in (3, 5, 7):
        raise ValueError(f"kernel_size {kernel_size} is not one of 3, 5, 7")
    depth = np.asarray(depth, dtype=np.float32)
    edge = np.zeros(depth.shape, dtype=bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        if mask is None:
            diff = _max_pool(depth, kernel_size) + _max_pool(-depth, kernel_size)
        else:
            ninf = np.float32(-np.inf)
            diff = _max_pool(np.where(mask, depth, ninf), kernel_size) + _max_pool(np.where(mask, -depth, ninf), kernel_size)
        if atol is not None:
            edge |= diff > atol
        if rtol is not None:
            edge |= diff / depth > rtol
    return edge


def build_mesh_from_map(*maps: np.ndarray, mask: np.ndarray = None, tri: bool = False):
    """Returns (faces int32, *attributes)."""
    H, W = maps[0].shape[:2]
    per = 3 if tri else 4
    if H < 2 or W < 2:
        return (np.zeros((0, per), dtype=np.int32), *[m.reshape(H * W, *m.shape[2:])[:0] for m in maps])
    idx = np.arange(H * W).reshape(H, W)
    quads = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], axis=-1).reshape(-1, 4)
    if mask is not None:
        m = np.asarray(mask, dtype=bool)
        kept = m[:-1, :-1] & m[1:, :-1] & m[1:, 1:] & m[:-1, 1:]
        quads = quads[kept.reshape(-1)]
    faces = np.stack([quads[:, [0, 1, 2]], quads[:, [0, 2, 3]]], axis=1).reshape(-1, 3) if tri else quads
    used, inverse = np.unique(faces, return_inverse=True)
    faces = inverse.reshape(faces.shape).astype(np.int32)
    return (faces, *[m.reshape(H * W, *m.shape[2:])[used] for m in maps])


def uv_map(height: int, width: int) -> np.ndarray:
    """(H, W, 2) fp32: ((j + 0.5) / W, (i + 0.5) / H)."""
    u = (np.arange(width, dtype=np.float32) + np.float32(0.5)) / np.float32(width)
    v = (np.arange(height, dtype=np.float32) + np.float32(0.5)) / np.float32(height)
    uu, vv = np.meshgrid(u, v, indexing="xy")
    return np.stack([uu, vv], axis=-1)


def mesh_from_output(points, depth, mask, image, normal=None, threshold: float = 0.04, remove_edge: bool = True):
    """infer.py:126-150 for one image: points (H, W, 3), depth (H, W), mask (H, W) bool, image (H, W, 3) uint8, normal (H, W, 3)
    or None.  Returns a dict of faces, vertices, vertex_colors, vertex_uvs, [vertex_normals,] mask_cleaned, all fp32 / int32."""
    height, width = depth.shape
    mask_cleaned = mask & ~depth_map_edge(depth, rtol=threshold) if remove_edge else mask.copy()
    maps = [points, image.astype(np.float32) / 255, uv_map(height, width)] + ([normal] if normal is not None else [])
    faces, vertices, vertex_colors, vertex_uvs, *rest = build_mesh_from_map(*maps, mask=mask_cleaned, tri=True)
    vertices, vertex_uvs = vertices * [1, -1, -1], vertex_uvs * [1, -1] + [0, 1]
    out = {"faces": faces, "vertices": vertices.astype(np.float32), "vertex_colors": vertex_colors,
           "vertex_uvs": vertex_uvs.astype(np.float32)}
    if normal is not None:
        out["vertex_normals"] = (rest[0] * [1, -1, -1]).astype(np.float32)
    out["mask_cleaned"] = mask_cleaned
    return out
