"""The `utils3d.np` functions that the reference's panorama module and script call (moge/utils/panorama.py,
moge/scripts/infer_panorama.py), restated from utils3d's published semantics.  TEST INFRASTRUCTURE ONLY.

`install()` adds them to the utils3d stand-in (oracle/utils3d_shim) as the submodule `utils3d.np`, so that the UNMODIFIED reference
module imports and runs against it.  No reference test pins them, so parity at this boundary is "unpinned" (DESIGN.md §2).  Two
choices are ours and are written out so the kernels can follow them operation by operation:
- products with a pinhole intrinsics matrix [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] are written as (u - cx) / fx and (fx x + cx z) / z
  (utils3d multiplies by the matrix and its inverse);
- a rigid extrinsics [R | t] is inverted as R^T (p - t) (utils3d calls np.linalg.inv).
Matrix-vector products are left-to-right sums of elementwise products in the operands' dtype: no BLAS, so every rounding is fixed.
"""
import itertools
import os
import sys
import types

import numpy as np

SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "utils3d_shim")


def create_icosahedron_mesh():
    """Vertices (12, 3) float32 of the icosahedron with vertices (0, ±1, ±A), (±1, ±A, 0), (±A, 0, ±1), A the golden ratio, and its
    20 faces (int32) wound outward."""
    A = (1 + 5 ** 0.5) / 2
    vertices = np.array([[0, 1, A], [0, -1, A], [0, 1, -A], [0, -1, -A], [1, A, 0], [-1, A, 0], [1, -A, 0], [-1, -A, 0],
                         [A, 0, 1], [A, 0, -1], [-A, 0, 1], [-A, 0, -1]], dtype=np.float32)
    v = vertices.astype(np.float64)
    faces = []
    for a, b, c in itertools.combinations(range(12), 3):
        if all(abs(np.linalg.norm(v[p] - v[q]) - 2) < 1e-6 for p, q in ((a, b), (b, c), (a, c))):
            if np.dot(np.cross(v[b] - v[a], v[c] - v[a]), v[a] + v[b] + v[c]) < 0:
                b, c = c, b
            faces.append([a, b, c])
    return vertices, np.array(faces, dtype=np.int32)


def intrinsics_from_fov(fov_x=None, fov_y=None):
    """Normalised pinhole intrinsics (principal point (0.5, 0.5)) for horizontal and vertical fields of view in radians."""
    fx = 0.5 / np.tan(fov_x / 2)
    fy = 0.5 / np.tan(fov_y / 2)
    return np.array([[fx, 0, 0.5], [0, fy, 0.5], [0, 0, 1]], dtype=np.float64)


def intrinsics_to_fov(intrinsics):
    """(fov_x, fov_y) in radians of normalised intrinsics (..., 3, 3)."""
    intrinsics = np.asarray(intrinsics)
    return 2 * np.arctan(0.5 / intrinsics[..., 0, 0]), 2 * np.arctan(0.5 / intrinsics[..., 1, 1])


def extrinsics_look_at(eye, look_at, up):
    """OpenCV world-to-camera extrinsics (..., 4, 4): z towards look_at, x = -up × z, y = z × x."""
    eye, look_at, up = np.asarray(eye), np.asarray(look_at), np.asarray(up)
    z = look_at - eye
    x = np.cross(-up, z)
    y = np.cross(z, x)
    x = x / np.linalg.norm(x, axis=-1, keepdims=True)
    y = y / np.linalg.norm(y, axis=-1, keepdims=True)
    z = z / np.linalg.norm(z, axis=-1, keepdims=True)
    R = np.stack([x, y, z], axis=-2)
    t = -(R * eye[..., None, :]).sum(axis=-1)
    E = np.zeros(R.shape[:-2] + (4, 4), dtype=R.dtype)
    E[..., :3, :3] = R
    E[..., :3, 3] = t
    E[..., 3, 3] = 1
    return E


def uv_map(*size, top=0., left=0., bottom=1., right=1., dtype=np.float32):
    """Pixel-centre UV grid (H, W, 2); called as uv_map((H, W)) or uv_map(H, W)."""
    if len(size) == 1 and isinstance(size[0], (tuple, list)):
        size = size[0]
    height, width = size
    u = np.linspace(left + 0.5 / width, right - 0.5 / width, width, dtype=dtype)
    v = np.linspace(top + 0.5 / height, bottom - 0.5 / height, height, dtype=dtype)
    u, v = np.meshgrid(u, v, indexing='xy')
    return np.stack([u, v], axis=2)


def uv_to_pixel(uv, size):
    """UV -> pixel coordinates of an (H, W) image: uv * (W, H) - 0.5."""
    return uv * np.array([size[1], size[0]]) - 0.5


def _mv(M, p):
    return np.stack([M[r, 0] * p[..., 0] + M[r, 1] * p[..., 1] + M[r, 2] * p[..., 2] for r in range(3)], axis=-1)


def unproject_cv(uv, depth, intrinsics=None, extrinsics=None):
    """Pixel UV and depth -> points (camera frame, or world frame with extrinsics)."""
    K = np.asarray(intrinsics)
    x = (uv[..., 0] - K[0, 2]) / K[0, 0] * depth
    y = (uv[..., 1] - K[1, 2]) / K[1, 1] * depth
    points = np.stack([x, y, depth * np.ones_like(x)], axis=-1)
    if extrinsics is not None:
        E = np.asarray(extrinsics)
        points = _mv(E[:3, :3].T, points - E[:3, 3])
    return points


def project_cv(points, intrinsics=None, extrinsics=None):
    """Points -> (UV, depth) of a pinhole camera."""
    if extrinsics is not None:
        E = np.asarray(extrinsics)
        points = _mv(E[:3, :3], points) + E[:3, 3]
    K = np.asarray(intrinsics)
    x, y, z = points[..., 0], points[..., 1], points[..., 2]
    uv = np.stack([(K[0, 0] * x + K[0, 2] * z) / z, (K[1, 1] * y + K[1, 2] * z) / z], axis=-1)
    return uv, z


FUNCTIONS = (create_icosahedron_mesh, intrinsics_from_fov, intrinsics_to_fov, extrinsics_look_at, uv_map, uv_to_pixel, unproject_cv,
             project_cv)


def install():
    """Put the shim on sys.path and add these functions to it as `utils3d.np`; returns that module."""
    if SHIM not in sys.path:
        sys.path.append(SHIM)
    import utils3d
    mod = getattr(utils3d, "np", None)
    if mod is None:
        mod = types.ModuleType("utils3d.np")
        utils3d.np = mod
        sys.modules["utils3d.np"] = mod
    for f in FUNCTIONS:
        setattr(mod, f.__name__, f)
    return mod
