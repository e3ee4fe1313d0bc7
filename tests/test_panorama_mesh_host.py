"""Panorama mesh export on the CPU side: the numpy restatement of utils3d's point_map_to_normal_map / normal_map_edge on hand-built
maps (oracle/utils3d_normals.py), the UV agreement that lets the mesh kernel generate the panorama's UVs, and argument validation
(every check fails before any launch, so none needs a GPU)."""
import ctypes as C

import numpy as np
import pytest
import torch

from moge_b200 import capi
from moge_b200 import mesh as M
from moge_b200 import panorama as P
from moge_b200.capi import MogeError
from moge_b200.synthetic import synthetic_panorama_scene
from oracle import utils3d_mesh as OM
from oracle import utils3d_normals as O


def _plane(H, W, a=0.3, b=-0.7, c=2.0):
    i, j = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    return np.stack([j, i, np.float32(a) * j + np.float32(b) * i + np.float32(c)], -1).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------ point_map_to_normal_map
def test_tilted_plane_normals():
    p = _plane(9, 11)
    want = np.array([-0.3, 0.7, 1.0]) / np.linalg.norm([-0.3, 0.7, 1.0])
    n, nm = O.point_map_to_normal_map(p, np.ones((9, 11), bool))
    assert nm.all() and n.dtype == np.float32
    sign = np.sign(n.reshape(-1, 3) @ want)
    assert (sign == sign[0]).all()                              # one orientation everywhere
    np.testing.assert_allclose(n.reshape(-1, 3) * sign[0], np.broadcast_to(want, (99, 3)), atol=1e-6)
    mask = np.ones((9, 11), bool)
    mask[4, 5] = False
    n, nm = O.point_map_to_normal_map(p, mask)
    assert not nm[4, 5] and (n[4, 5] == 0).all() and nm.sum() == 98
    np.testing.assert_allclose(n[nm] * sign[0], np.broadcast_to(want, (98, 3)), atol=1e-6)


def test_unmasked_border_uses_the_zero_padding():
    p = _plane(6, 7)
    unmasked = O.point_map_to_normal_map(p)
    # the same as a map with a ring of in-mask zero points around it
    padded = np.zeros((8, 9, 3), np.float32)
    padded[1:-1, 1:-1] = p
    ring, _ = O.point_map_to_normal_map(padded, np.ones((8, 9), bool))
    assert unmasked.tobytes() == np.ascontiguousarray(ring[1:-1, 1:-1]).tobytes()
    masked, _ = O.point_map_to_normal_map(p, np.ones((6, 7), bool))
    assert np.array_equal(unmasked[1:-1, 1:-1], masked[1:-1, 1:-1])
    border = np.ones((6, 7), bool)
    border[1:-1, 1:-1] = False
    assert (np.abs(unmasked - masked).max(-1) > 1e-3)[border].all()


def test_nan_neighbour_poisons_an_invalid_product():
    p = _plane(5, 5)
    p[1, 2] = np.nan
    mask = np.ones((5, 5), bool)
    mask[1, 2] = False                      # (2, 2)'s products with its up neighbour are invalid, but multiplied by 0
    n, nm = O.point_map_to_normal_map(p, mask)
    assert nm[2, 2] and np.isnan(n[2, 2]).all()
    assert not np.isnan(n[3, 3]).any()
    p[1, 2] = np.inf
    n, nm = O.point_map_to_normal_map(p, mask)
    assert nm[2, 2] and np.isnan(n[2, 2]).all()


def test_no_wrap_at_the_seam_and_edge_threshold_is_rejected():
    p = _plane(4, 6)
    n, _ = O.point_map_to_normal_map(p, np.ones((4, 6), bool))
    rolled, _ = O.point_map_to_normal_map(np.roll(p, 1, axis=1), np.ones((4, 6), bool))
    assert not np.array_equal(rolled[:, 1], n[:, 0])          # column 0 has no left neighbour, not column W - 1
    with pytest.raises(NotImplementedError):
        O.point_map_to_normal_map(p, edge_threshold=0.1)


def test_numpy_reduction_orders():
    """The orders the kernels follow: np.linalg.norm and the channel sum of three fp32 values go left to right, the sum over the
    four products too."""
    x = np.random.default_rng(0).normal(size=(4, 20000, 3)).astype(np.float32) * np.float32(1e3)
    assert np.array_equal(np.linalg.norm(x, axis=-1), np.sqrt((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2]))
    assert np.array_equal((x[0] * x[1]).sum(-1), (x[0, :, 0] * x[1, :, 0] + x[0, :, 1] * x[1, :, 1]) + x[0, :, 2] * x[1, :, 2])
    assert np.array_equal(x.sum(0), ((x[0] + x[1]) + x[2]) + x[3])
    c = np.cross(x[0], x[1])
    assert np.array_equal(c[:, 0], x[0, :, 1] * x[1, :, 2] - x[0, :, 2] * x[1, :, 1])
    assert (np.float32(1) + 1e-12).dtype == np.float32 and np.float32(1e-12).view(np.uint32) == 0x2B8CBCCC


# ------------------------------------------------------------------------------------------------------------ normal_map_edge
def _nan_normal():
    """A unit fp32 normal whose normalised dot product with itself exceeds 1 (arccos: NaN)."""
    x = np.random.default_rng(1).normal(size=(20000, 3)).astype(np.float32)
    x = x / (np.linalg.norm(x, axis=-1, keepdims=True) + 1e-12)
    x = x / (np.linalg.norm(x, axis=-1, keepdims=True) + 1e-12)
    dots = (x * x).sum(-1)
    return x[np.argmax(dots > 1)] if (dots > 1).any() else None


def test_nan_angle_is_never_an_edge_and_the_pool_spreads_it():
    n = _nan_normal()
    assert n is not None and abs(n[2]) < 0.95
    normals = np.zeros((9, 9, 3), np.float32)
    normals[..., 2] = 1
    normals[4, 4] = n                                           # far from (0, 0, 1): an edge wherever the NaN does not reach
    angle = O.normal_angle_map(normals, 3)
    assert np.isnan(angle[3:6, 3:6]).all() and np.isnan(angle).sum() == 9
    edge = O.normal_map_edge(normals, tol=5)
    want = np.zeros((9, 9), bool)
    want[2:7, 2:7] = True
    want[3:6, 3:6] = False
    assert np.array_equal(edge, want)
    mask = np.ones((9, 9), bool)
    mask[4, 4] = False               # its angles in the others' windows are 0 and there is no NaN, but its own centre is not masked
    assert not np.isnan(O.normal_angle_map(normals, 3, mask)).any()
    want[:] = False
    want[3:6, 3:6] = True
    assert np.array_equal(O.normal_map_edge(normals, tol=5, mask=mask), want)


def test_crease_and_kernel_sizes():
    normals = np.zeros((5, 12, 3), np.float32)
    normals[:, :6, 2] = 1
    normals[:, 6:, 0] = 1                                       # a 90-degree crease between columns 5 and 6
    for k, width in ((3, 4), (5, 8), (7, 12)):
        edge = O.normal_map_edge(normals, tol=5, kernel_size=k)
        cols = np.flatnonzero(edge[2])
        assert len(cols) == min(width, 12) and (edge == edge[2]).all()
    with pytest.raises(ValueError):
        O.normal_map_edge(normals, tol=5, kernel_size=4)


def test_threshold_is_compared_in_fp64(monkeypatch):
    tol = next(t for t in np.arange(1, 90, 0.25) if np.float32(np.deg2rad(t)) > np.deg2rad(t))
    a = np.full((2, 2), np.float32(np.deg2rad(tol)))
    monkeypatch.setattr(O, "normal_angle_map", lambda n, k, m: a)
    assert O.normal_map_edge(np.zeros((2, 2, 3), np.float32), tol).all()        # fp32 rounded up: above the fp64 threshold
    assert not (a > np.float32(np.deg2rad(tol))).any()                          # an fp32 comparison would say no
    assert not np.float32(np.deg2rad(5)) > np.deg2rad(5)


def test_mesh_from_panorama_restatement():
    points, depth, mask, image = synthetic_panorama_scene(64, 128, 0)
    out = O.mesh_from_panorama(points, depth, mask, image)
    normals, nm = O.point_map_to_normal_map(points, mask)
    keep = mask & ~(OM.depth_map_edge(depth, rtol=0.03) & O.normal_map_edge(normals, 5, mask=nm))
    assert np.array_equal(out["mask_cleaned"], keep) and (mask & ~keep).any()
    faces, v, c, uv = OM.build_mesh_from_map(points, image.astype(np.float32) / 255, OM.uv_map(64, 128), mask=keep, tri=True)
    for got, want in zip((out["faces"], out["vertices"], out["vertex_colors"], out["vertex_uvs"]), (faces, v, c, uv)):
        assert got.dtype == want.dtype and got.tobytes() == want.tobytes()
    assert np.array_equal(O.mesh_from_panorama(points, depth, mask, image, threshold=np.inf)["mask_cleaned"], mask)


# ------------------------------------------------------------------------------------------------------------ UVs
def test_kernel_uvs_equal_the_panorama_uv_map():
    """The mesh kernel's UV (c + 0.5) / n in fp32 (oracle/utils3d_mesh.uv_map) is bitwise the panorama's np.linspace uv_map at every
    width and height up to 16384 (4096 x 16384 is beyond the largest panorama the reference script is run on)."""
    for n in range(1, 16385):
        a = P.uv_map(1, n)[0, :, 0]
        b = (np.arange(n, dtype=np.float32) + np.float32(0.5)) / np.float32(n)
        assert a.tobytes() == b.tobytes(), n
    assert np.array_equal(P.uv_map(37, 53), OM.uv_map(37, 53))


# ------------------------------------------------------------------------------------------------------------ validation
def test_cpu_tensors_are_rejected():
    with pytest.raises(MogeError, match="CUDA"):
        M.point_map_to_normal_map(torch.ones(8, 8, 3))
    with pytest.raises(MogeError, match="CUDA"):
        M.point_map_to_normal_map(torch.ones(2, 8, 8, 3), torch.ones(2, 8, 8, dtype=torch.bool))
    with pytest.raises(MogeError, match="CUDA"):
        M.normal_map_edge(torch.ones(8, 8, 3), tol=5)
    out = {"points": torch.ones(8, 8, 3), "depth": torch.ones(8, 8), "mask": torch.ones(8, 8, dtype=torch.bool)}
    with pytest.raises(MogeError, match="CUDA"):
        M.mesh_from_panorama(out, torch.zeros(8, 8, 3, dtype=torch.uint8))


def test_bad_arguments_are_rejected():
    with pytest.raises(MogeError, match="kernel_size"):
        M.normal_map_edge(torch.ones(8, 8, 3), tol=5, kernel_size=4)
    with pytest.raises(MogeError, match="edge_threshold"):
        M.point_map_to_normal_map(torch.ones(8, 8, 3), edge_threshold=0.1)
    with pytest.raises(MogeError, match=r"\(\.\.\., H, W, 3\)"):
        M.point_map_to_normal_map(torch.ones(8, 8, 4))
    with pytest.raises(MogeError, match="does not match"):
        M.normal_map_edge(torch.ones(8, 8, 3), tol=5, mask=torch.ones(8, 9, dtype=torch.bool))
    with pytest.raises(MogeError, match="too large"):
        M.point_map_to_normal_map(torch.ones(1, 1, 3).expand(40000, 30000, 3))
    out = {"points": torch.ones(8, 8, 3), "depth": torch.ones(8, 8), "mask": torch.ones(8, 8, dtype=torch.bool)}
    with pytest.raises(MogeError, match="image"):
        M.mesh_from_panorama(out, torch.zeros(8, 9, 3, dtype=torch.uint8))
    with pytest.raises(MogeError, match="uint8"):
        M.mesh_from_panorama(out, torch.zeros(8, 8, 3))
    with pytest.raises(MogeError, match="points"):
        M.mesh_from_panorama(dict(out, points=torch.ones(8, 8, 4)), torch.zeros(8, 8, 3, dtype=torch.uint8))
    with pytest.raises(MogeError, match="depth"):
        M.mesh_from_panorama(dict(out, depth=torch.ones(1, 8, 8)), torch.zeros(8, 8, 3, dtype=torch.uint8))


def test_abi_rejects_bad_arguments_before_launch():
    L = capi.lib()
    assert L.moge_normal_map(None, None, 1, 8, 8, 8, None, None) != 0 and b"null" in L.moge_last_error()
    assert L.moge_normal_map(8, None, 1, 8, 8, None, None, None) != 0 and b"null" in L.moge_last_error()
    assert L.moge_normal_map(8, None, 0, 8, 8, 8, None, None) != 0 and b"batch" in L.moge_last_error()
    assert L.moge_normal_map(8, None, 1, 40000, 30000, 8, None, None) != 0 and b"too large" in L.moge_last_error()
    assert L.moge_normal_map(8, None, 1, 0, 8, 8, None, None) != 0 and b"size" in L.moge_last_error()
    tol = float(np.deg2rad(5))
    assert L.moge_normal_edge(None, None, None, None, 1, 8, 8, 3, tol, 8, None, None) != 0 and b"null" in L.moge_last_error()
    assert L.moge_normal_edge(8, None, None, None, 1, 8, 8, 3, tol, None, None, None) != 0 and b"null" in L.moge_last_error()
    for k in (1, 2, 4, 9):
        assert L.moge_normal_edge(8, None, None, None, 1, 8, 8, k, tol, 8, None, None) != 0 and b"kernel_size" in L.moge_last_error()
    assert L.moge_normal_edge(8, None, None, None, 1, 40000, 30000, 3, tol, 8, None, None) != 0 and b"too large" in L.moge_last_error()
    assert L.moge_normal_edge(8, None, None, None, 1, 65535 * 32 + 1, 1, 3, tol, 8, None, None) != 0 and b"rows" in L.moge_last_error()
    assert L.moge_normal_edge(8, None, None, None, 70000, 8, 8, 3, tol, 8, None, None) != 0 and b"batch" in L.moge_last_error()
