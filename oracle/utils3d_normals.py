"""The two utils3d functions that the reference's panorama mesh export adds to the single-image one (moge/scripts/
infer_panorama.py:136-150, and the cleaning step of moge/scripts/infer_baseline.py:120-127), and the panorama step itself,
restated in numpy from utils3d's published semantics.  TEST INFRASTRUCTURE ONLY, and the host comparator of
tools/bench_panorama_mesh.py.

utils3d (pinned by the reference at 3fab839f) is not vendored, so no reference run pins these: parity at this boundary is
"unpinned" (DESIGN.md §2), as for oracle/utils3d_mesh.py, whose depth_map_edge and build_mesh_from_map this module reuses.  The
kernels of moge_b200/csrc/mesh.cu follow the rules below operation by operation.  Every operation is fp32 with one IEEE rounding
(numpy does not contract a * b - c into an FMA), and under NEP 50 a Python-float constant such as 1e-12 is an fp32 operand.

normalise(n) = n / (|n| + 1e-12), |n| = sqrt((x0 * x0 + x1 * x1) + x2 * x2) summed left to right (np.linalg.norm's order for
three contiguous values).

point_map_to_normal_map(point, mask=None), point (..., H, W, 3) fp32, images independent:
  - points are padded with zeros and the mask with False by one pixel; up / left / down / right = neighbour - centre;
  - the four products up x left, left x down, down x right, right x up, each np.cross component a1 * b2 - a2 * b1 with both
    products rounded before the subtraction, each normalised;
  - valid[k] = both neighbours of product k in the padded mask, and the centre in the mask.  Without a mask every product is
    valid, so a border pixel's products use differences to the zero padding (utils3d's behaviour, kept);
  - normal = normalise(((n0 * v0 + n1 * v1) + n2 * v2) + n3 * v3) with v = 0.0 / 1.0: a multiply, not a select, so a NaN or
    inf in an invalid product still poisons the sum;
  - with a mask: (normal, normal_mask), normal_mask = any valid[k], normals +0.0 off it; without: normal only;
  - no wrap at the panorama seam.  utils3d's edge_threshold argument is not restated (no caller we serve passes it).

normal_map_edge(normals, tol, kernel_size=3, mask=None), normals (..., H, W, 3):
  - the normals are normalised as above;
  - for each pixel and each offset of the kernel_size x kernel_size window over the edge-padded (clamped) normals:
    dot = (c0 * w0 + c1 * w1) + c2 * w2, angle = arccos(dot) in fp32.  A dot product above 1 or below -1 (a unit normal with
    itself can reach 1 + 1 ulp) gives NaN, which is part of the contract;
  - with a mask, an angle whose window pixel is off the edge-padded mask becomes 0 (the centre's own mask is not consulted);
  - the window max (NaN propagates), then a kernel_size max pool padded with -inf (NaN propagates);
  - edge = angle > np.deg2rad(tol): np.deg2rad returns an fp64 scalar, so under NEP 50 the fp32 angle is compared in fp64
    (fp32(deg2rad(5)) is not > deg2rad(5)).  A NaN angle is never an edge;
  - kernel_size is 3, 5 or 7.
  utils3d builds the (..., H, W, 3, k, k) window product at once; the loop over window offsets below computes the same values
  with the same roundings and takes the same maximum, in a fraction of the memory.

mesh_from_panorama(points, depth, mask, image, threshold=0.03): infer_panorama.py:137-144 on the panorama maps:
  keep = mask & ~(depth_map_edge(depth, rtol=threshold) & normal_map_edge(normals, tol=5, mask=normals_mask)) with
  (normals, normals_mask) = point_map_to_normal_map(points, mask), then build_mesh_from_map(points, image / 255 (fp32),
  uv_map(H, W), mask=keep, tri=True).  No OpenGL flips and no vertex normals: the panorama script applies neither.
"""
import numpy as np

from .utils3d_mesh import _max_pool, build_mesh_from_map, depth_map_edge
from .utils3d_panorama import uv_map

KERNEL_SIZES = (3, 5, 7)


def _normalize(n: np.ndarray) -> np.ndarray:
    return n / (np.linalg.norm(n, axis=-1, keepdims=True) + 1e-12)


def point_map_to_normal_map(point: np.ndarray, mask: np.ndarray = None, edge_threshold=None):
    if edge_threshold is not None:
        raise NotImplementedError("point_map_to_normal_map: edge_threshold is not restated")
    point = np.asarray(point, dtype=np.float32)
    lead, (H, W) = point.shape[:-3], point.shape[-3:-1]
    pts = np.zeros(lead + (H + 2, W + 2, 3), dtype=np.float32)
    pts[..., 1:-1, 1:-1, :] = point
    centre = pts[..., 1:-1, 1:-1, :]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        up = pts[..., :-2, 1:-1, :] - centre
        left = pts[..., 1:-1, :-2, :] - centre
        down = pts[..., 2:, 1:-1, :] - centre
        right = pts[..., 1:-1, 2:, :] - centre
        normal = _normalize(np.stack([np.cross(up, left), np.cross(left, down), np.cross(down, right), np.cross(right, up)]))
        if mask is None:
            valid = np.ones((4,) + lead + (H, W), dtype=bool)
        else:
            m = np.zeros(lead + (H + 2, W + 2), dtype=bool)
            m[..., 1:-1, 1:-1] = mask
            mu, ml, md, mr = m[..., :-2, 1:-1], m[..., 1:-1, :-2], m[..., 2:, 1:-1], m[..., 1:-1, 2:]
            valid = np.stack([mu & ml, ml & md, md & mr, mr & mu]) & m[None, ..., 1:-1, 1:-1]
        normal = _normalize((normal * valid[..., None]).sum(axis=0))
    if mask is None:
        return normal
    normal_mask = valid.any(axis=0)
    return np.where(normal_mask[..., None], normal, 0), normal_mask


def normal_angle_map(normals: np.ndarray, kernel_size: int = 3, mask: np.ndarray = None) -> np.ndarray:
    """normal_map_edge before the threshold: the pooled fp32 angle map (NaN where it propagated)."""
    if kernel_size not in KERNEL_SIZES:
        raise ValueError(f"kernel_size {kernel_size} is not one of 3, 5, 7")
    normals = np.asarray(normals, dtype=np.float32)
    H, W = normals.shape[-3:-1]
    r = kernel_size // 2
    lead = [(0, 0)] * (normals.ndim - 3)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        normals = _normalize(normals)
        padded = np.pad(normals, lead + [(r, r), (r, r), (0, 0)], mode="edge")
        mpad = None if mask is None else np.pad(np.asarray(mask, dtype=bool), lead + [(r, r), (r, r)], mode="edge")
        angle = None
        for di in range(kernel_size):
            for dj in range(kernel_size):
                a = np.arccos((normals * padded[..., di:di + H, dj:dj + W, :]).sum(axis=-1))
                if mpad is not None:
                    a = np.where(mpad[..., di:di + H, dj:dj + W], a, 0)
                angle = a if angle is None else np.maximum(angle, a)
    return _max_pool(angle, kernel_size)


def normal_map_edge(normals: np.ndarray, tol: float, kernel_size: int = 3, mask: np.ndarray = None) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        return normal_angle_map(normals, kernel_size, mask) > np.deg2rad(tol)


def mesh_from_panorama(points, depth, mask, image, threshold: float = 0.03):
    """infer_panorama.py:137-144: points (H, W, 3), depth (H, W), mask (H, W) bool, image (H, W, 3) uint8.  Returns a dict of
    faces (int32 triangles), vertices, vertex_colors, vertex_uvs and mask_cleaned."""
    height, width = depth.shape
    normals, normals_mask = point_map_to_normal_map(points, mask)
    edge = depth_map_edge(depth, rtol=threshold) & normal_map_edge(normals, tol=5, mask=normals_mask)
    mask_cleaned = mask & ~edge
    faces, vertices, vertex_colors, vertex_uvs = build_mesh_from_map(points, image.astype(np.float32) / 255, uv_map(height, width),
                                                                     mask=mask_cleaned, tri=True)
    return {"faces": faces, "vertices": vertices, "vertex_colors": vertex_colors, "vertex_uvs": vertex_uvs,
            "mask_cleaned": mask_cleaned}
