"""Mesh export on the CPU side: the numpy restatement of utils3d's depth_map_edge / build_mesh_from_map on hand-built maps, the
fp32 tolerance comparison, the PLY and GLB writers read back, and argument validation (every check fails before any launch, so
none needs a GPU)."""
import ctypes as C
import json
import struct

import cv2
import numpy as np
import pytest
import torch

from moge_b200 import capi
from moge_b200 import mesh as M
from moge_b200.capi import MogeError
from moge_b200.export import save_glb, save_ply
from oracle import utils3d_mesh as O

T, F = True, False


# ------------------------------------------------------------------------------------------------------------ depth_map_edge
def test_step_edge():
    d = np.array([[1, 1, 2]] * 3, dtype=np.float32)
    # diff per column: 0, 1, 1; diff / d: 0, 1, 0.5
    assert np.array_equal(O.depth_map_edge(d, rtol=0.04), np.array([[F, T, T]] * 3))
    assert np.array_equal(O.depth_map_edge(d, atol=0.75), np.array([[F, T, T]] * 3))
    assert not O.depth_map_edge(d, atol=1.0).any()                 # 1 > 1 is false
    assert np.array_equal(O.depth_map_edge(d, atol=1.0, rtol=0.6), np.array([[F, T, F]] * 3))
    assert not O.depth_map_edge(d).any()                           # no tolerance: no edge


def test_inf_holes():
    d = np.ones((3, 5), dtype=np.float32)
    d[1, 1] = np.inf
    want = np.zeros((3, 5), dtype=bool)
    want[:, :3] = True            # finite neighbours of the inf pixel: inf / d = inf
    want[1, 1] = False            # the inf pixel itself: inf / inf = NaN
    assert np.array_equal(O.depth_map_edge(d, rtol=0.04), want)
    assert np.array_equal(O.depth_map_edge(d, atol=0.5), want | (np.arange(5) < 3)[None] & (d == np.inf))
    all_inf = np.full((3, 3), np.inf, dtype=np.float32)           # inf + (-inf) = NaN: no edge
    assert not O.depth_map_edge(all_inf, rtol=0.04, atol=0.0).any()


def test_masked_empty_window():
    d = np.array([[1, 2, 3], [4, 5, 6], [7, 8, -1]], dtype=np.float32)
    mask = np.zeros((3, 3), dtype=bool)
    mask[0, 0] = True
    # windows holding (0, 0) see only it: diff = 0; the others see nothing: diff = -inf, and -inf / -1 = inf at (2, 2)
    want = np.zeros((3, 3), dtype=bool)
    want[2, 2] = True
    assert np.array_equal(O.depth_map_edge(d, rtol=0.04, mask=mask), want)
    assert not O.depth_map_edge(d, atol=0.5, mask=mask).any()


def test_kernel_size_five():
    d = np.ones((1, 9), dtype=np.float32)
    d[0, 8] = 2
    assert np.array_equal(O.depth_map_edge(d, rtol=0.04, kernel_size=5)[0], np.arange(9) >= 6)
    assert np.array_equal(O.depth_map_edge(d, rtol=0.04, kernel_size=7)[0], np.arange(9) >= 5)


def test_tolerance_is_compared_in_fp32():
    d = np.array([[1.0, 1.5]], dtype=np.float32)                  # diff = 0.5 at both pixels
    atol = 0.5 - 1e-12
    assert atol < 0.5 and np.float32(atol) == np.float32(0.5)
    assert not O.depth_map_edge(d, atol=atol).any()               # in fp64 0.5 > atol would hold
    assert not (np.array([np.float32(0.04)]) > float(np.float32(0.04)) - 1e-12).any()
    assert M._tol(atol).value == 0.5 and M._tol(0.04).value == float(np.float32(0.04))


# ------------------------------------------------------------------------------------------------------------ build_mesh_from_map
def test_grid_with_one_masked_pixel():
    x = np.arange(6, dtype=np.float32).reshape(2, 3)
    rgb = np.arange(18, dtype=np.float32).reshape(2, 3, 3)
    mask = np.ones((2, 3), dtype=bool)
    mask[0, 2] = False
    faces, a, c = O.build_mesh_from_map(x, rgb, mask=mask)
    assert faces.dtype == np.int32 and np.array_equal(faces, [[0, 2, 3, 1]])
    assert np.array_equal(a, [0, 1, 3, 4]) and np.array_equal(c, rgb.reshape(6, 3)[[0, 1, 3, 4]])
    faces, a = O.build_mesh_from_map(x, mask=mask, tri=True)
    assert np.array_equal(faces, [[0, 2, 3], [0, 3, 1]])
    faces, a = O.build_mesh_from_map(x)
    assert np.array_equal(faces, [[0, 3, 4, 1], [1, 4, 5, 2]]) and np.array_equal(a, x.reshape(-1))
    faces, _ = O.build_mesh_from_map(x, tri=True)
    assert np.array_equal(faces, [[0, 3, 4], [0, 4, 1], [1, 4, 5], [1, 5, 2]])


def test_isolated_pixel_is_dropped():
    x = np.arange(12, dtype=np.float32).reshape(3, 4, 1)
    mask = np.zeros((3, 4), dtype=bool)
    mask[:2, :2] = True
    mask[2, 3] = True
    faces, a = O.build_mesh_from_map(x, mask=mask)
    assert np.array_equal(faces, [[0, 2, 3, 1]]) and np.array_equal(a[:, 0], [0, 1, 4, 5])
    only = np.zeros((3, 3), dtype=bool)
    only[1, 1] = True
    faces, a = O.build_mesh_from_map(x[:, :3], mask=only, tri=True)
    assert faces.shape == (0, 3) and a.shape == (0, 1)


@pytest.mark.parametrize("shape", [(1, 7), (6, 1), (1, 1)])
def test_thin_maps_have_no_faces(shape):
    x = np.ones((*shape, 3), dtype=np.float32)
    for tri, per in ((False, 4), (True, 3)):
        faces, a = O.build_mesh_from_map(x, tri=tri)
        assert faces.shape == (0, per) and faces.dtype == np.int32 and a.shape == (0, 3)


def test_mesh_from_output_conventions():
    H, W = 3, 4
    points = np.random.default_rng(0).normal(size=(H, W, 3)).astype(np.float32)
    depth = np.ones((H, W), dtype=np.float32)
    image = np.arange(H * W * 3, dtype=np.uint8).reshape(H, W, 3)
    out = O.mesh_from_output(points, depth, np.ones((H, W), dtype=bool), image)
    assert out["faces"].shape == (2 * (H - 1) * (W - 1), 3) and out["mask_cleaned"].all()
    assert np.array_equal(out["vertices"], points.reshape(-1, 3) * np.float32([1, -1, -1]))
    assert np.array_equal(out["vertex_colors"], image.reshape(-1, 3).astype(np.float32) / np.float32(255))
    uv = O.uv_map(H, W).reshape(-1, 2)
    assert np.array_equal(out["vertex_uvs"][:, 0], uv[:, 0]) and np.array_equal(out["vertex_uvs"][:, 1], (1 - uv[:, 1].astype(np.float64)).astype(np.float32))
    assert O.uv_map(H, W)[2, 1].tolist() == [np.float32(1.5) / np.float32(W), np.float32(2.5) / np.float32(H)]


# ------------------------------------------------------------------------------------------------------------ writers
def _mesh_arrays(n=50, f=40, seed=0):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3)).astype(np.float32)
    faces = rng.integers(0, n, size=(f, 3)).astype(np.int32)
    colours = rng.random((n, 3)).astype(np.float32)
    colours[0] = [-0.2, 1.3, 0.2 / 255]
    normals = rng.normal(size=(n, 3)).astype(np.float32)
    uvs = rng.random((n, 2)).astype(np.float32)
    return v, faces, colours, normals, uvs


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    return header, data[end:]


def test_ply_round_trip(tmp_path):
    v, faces, colours, normals, _ = _mesh_arrays()
    p = tmp_path / "m.ply"
    save_ply(p, v, faces, colours, normals)
    header, body = _read_ply(p)
    assert header[:3] == ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    assert header[3:9] == [f"property float {c}" for c in ("x", "y", "z", "nx", "ny", "nz")]
    assert header[9:12] == [f"property uchar {c}" for c in ("red", "green", "blue")]
    assert header[12:] == [f"element face {len(faces)}", "property list uchar int vertex_indices", "end_header"]
    rec = np.frombuffer(body, dtype=[("p", "<f4", 3), ("n", "<f4", 3), ("c", "u1", 3)], count=len(v))
    assert rec["p"].tobytes() == v.tobytes() and rec["n"].tobytes() == normals.tobytes()
    assert np.array_equal(rec["c"], np.clip(np.round(colours.astype(np.float64) * 255), 0, 255).astype(np.uint8))
    assert rec["c"][0].tolist() == [0, 255, 0]
    frec = np.frombuffer(body[rec.nbytes:], dtype=[("k", "u1"), ("i", "<i4", 3)])
    assert len(frec) == len(faces) and (frec["k"] == 3).all() and frec["i"].tobytes() == faces.tobytes()


def test_ply_point_cloud(tmp_path):
    """infer.py writes the point cloud with (0, 3) faces and no normals"""
    v, _, colours, _, _ = _mesh_arrays()
    p = tmp_path / "pc.ply"
    save_ply(p, torch.from_numpy(v), np.zeros((0, 3), dtype=np.int32), torch.from_numpy(colours), None)
    header, body = _read_ply(p)
    assert "element face 0" in header and "property float nx" not in header
    assert len(body) == len(v) * 15


@pytest.mark.parametrize("with_normals", [False, True])
def test_glb_round_trip(tmp_path, with_normals):
    v, faces, _, normals, uvs = _mesh_arrays()
    tex = np.random.default_rng(1).integers(0, 256, size=(13, 21, 3)).astype(np.uint8)
    p = tmp_path / "m.glb"
    save_glb(p, v, faces, uvs, tex, normals if with_normals else None)
    data = open(p, "rb").read()
    magic, version, total = struct.unpack_from("<III", data)
    assert (magic, version, total) == (0x46546C67, 2, len(data)) and total % 4 == 0
    jlen, jtype = struct.unpack_from("<II", data, 12)
    assert jtype == 0x4E4F534A and jlen % 4 == 0
    gltf = json.loads(data[20:20 + jlen])
    blen, btype = struct.unpack_from("<II", data, 20 + jlen)
    assert btype == 0x004E4942 and blen % 4 == 0 and 28 + jlen + blen == len(data)
    binary = data[28 + jlen:]
    assert gltf["buffers"] == [{"byteLength": blen}]
    prim = gltf["meshes"][0]["primitives"][0]
    assert prim["mode"] == 4 and set(prim["attributes"]) == ({"POSITION", "TEXCOORD_0"} | ({"NORMAL"} if with_normals else set()))
    mat = gltf["materials"][prim["material"]]["pbrMetallicRoughness"]
    assert mat["metallicFactor"] == 0.5 and mat["roughnessFactor"] == 1.0

    def view_bytes(i):
        bv = gltf["bufferViews"][i]
        assert bv["byteOffset"] % 4 == 0
        return binary[bv["byteOffset"]:bv["byteOffset"] + bv["byteLength"]]

    def accessor(name, want):
        acc = gltf["accessors"][prim["attributes"][name] if name != "indices" else prim["indices"]]
        assert acc["count"] == want.shape[0]
        assert view_bytes(acc["bufferView"]) == want.tobytes()
        return acc

    pos = accessor("POSITION", v)
    assert pos["componentType"] == 5126 and pos["type"] == "VEC3"
    assert pos["min"] == v.min(0).tolist() and pos["max"] == v.max(0).tolist()
    assert accessor("TEXCOORD_0", uvs)["type"] == "VEC2"
    if with_normals:
        accessor("NORMAL", normals)
    idx = accessor("indices", faces.astype(np.uint32).reshape(-1))
    assert idx["componentType"] == 5125 and idx["type"] == "SCALAR"
    img = gltf["images"][gltf["textures"][mat["baseColorTexture"]["index"]]["source"]]
    assert img["mimeType"] == "image/png"
    png = np.frombuffer(view_bytes(img["bufferView"]), dtype=np.uint8)
    assert np.array_equal(cv2.cvtColor(cv2.imdecode(png, cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB), tex)


def test_glb_rejects_quads_and_empty_meshes(tmp_path):
    v, faces, _, _, uvs = _mesh_arrays()
    tex = np.zeros((2, 2, 3), dtype=np.uint8)
    with pytest.raises(ValueError, match="triangles"):
        save_glb(tmp_path / "q.glb", v, np.zeros((3, 4), dtype=np.int32), uvs, tex)
    with pytest.raises(ValueError, match="empty"):
        save_glb(tmp_path / "e.glb", v[:0], faces[:0], uvs[:0], tex)


# ------------------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("k", [1, 2, 4, 6, 9])
def test_bad_kernel_size_is_rejected_first(k):
    with pytest.raises(MogeError, match="kernel_size"):
        M.depth_map_edge(torch.ones(8, 8), rtol=0.04, kernel_size=k)      # a CPU tensor: the size check comes first


def test_cpu_tensors_are_rejected():
    with pytest.raises(MogeError, match="CUDA"):
        M.depth_map_edge(torch.ones(8, 8), rtol=0.04)
    with pytest.raises(MogeError, match="CUDA"):
        M.build_mesh_from_map(torch.ones(8, 8, 3), mask=torch.ones(8, 8, dtype=torch.bool))
    with pytest.raises(MogeError, match="CUDA"):
        M.build_mesh_from_map_batch(torch.ones(2, 8, 8, 3))
    out = {"points": torch.ones(8, 8, 3), "depth": torch.ones(8, 8), "mask": torch.ones(8, 8, dtype=torch.bool)}
    with pytest.raises(MogeError, match="CUDA"):
        M.mesh_from_output(out, torch.zeros(8, 8, 3, dtype=torch.uint8))


def test_mismatched_shapes_are_rejected():
    with pytest.raises(MogeError, match="do not match"):
        M.build_mesh_from_map(torch.ones(8, 8, 3), torch.ones(8, 9))
    with pytest.raises(MogeError, match="does not match"):
        M.build_mesh_from_map(torch.ones(8, 8, 3), mask=torch.ones(8, 9, dtype=torch.bool))
    with pytest.raises(MogeError, match="does not match"):
        M.depth_map_edge(torch.ones(8, 8), rtol=0.1, mask=torch.ones(8, 9, dtype=torch.bool))
    with pytest.raises(MogeError, match="channels"):
        M.build_mesh_from_map(torch.ones(8, 8, 5))
    out = {"points": torch.ones(8, 8, 3), "depth": torch.ones(8, 8), "mask": torch.ones(8, 8, dtype=torch.bool)}
    with pytest.raises(MogeError, match="image"):
        M.mesh_from_output(out, torch.zeros(8, 9, 3, dtype=torch.uint8))
    with pytest.raises(MogeError, match="points"):
        M.mesh_from_output(dict(out, points=torch.ones(8, 8, 4)), torch.zeros(8, 8, 3, dtype=torch.uint8))


def test_over_large_maps_are_rejected():
    big = torch.ones(1, 1).expand(40000, 30000)                   # 1.2e9 pixels, no memory behind it
    with pytest.raises(MogeError, match="too large"):
        M.depth_map_edge(big, rtol=0.04)
    with pytest.raises(MogeError, match="too large"):
        M.build_mesh_from_map(big)


def test_abi_rejects_bad_arguments_before_launch():
    L = capi.lib()
    n = C.c_size_t()
    assert L.moge_mesh_workspace_bytes(1, 40000, 30000, C.byref(n)) != 0 and b"too large" in L.moge_last_error()
    assert L.moge_mesh_workspace_bytes(0, 8, 8, C.byref(n)) != 0
    assert L.moge_mesh_workspace_bytes(2, 37, 53, C.byref(n)) == 0 and n.value > 2 * 37 * 53 * 4
    r = C.c_float(0.04)
    assert L.moge_depth_edge(8, None, None, 1, 8, 8, 4, None, C.byref(r), 8, None) != 0 and b"kernel_size" in L.moge_last_error()
    assert L.moge_depth_edge(8, None, None, 1, 8, 8, 9, None, C.byref(r), 8, None) != 0
    assert L.moge_mesh_count(None, 1, 8, 8, 8, 256, 16, None) != 0 and b"workspace" in L.moge_last_error()
    maps = (capi.MeshMap * 1)()
    maps[0].kind, maps[0].channels, maps[0].dst = capi.MESH_UV, 3, 8
    assert L.moge_mesh_build(None, 1, 8, 8, 1, maps, 1, 8, 8, 256, 1 << 20, None) != 0 and b"UV" in L.moge_last_error()
    maps[0].kind, maps[0].channels, maps[0].src = capi.MESH_F32, 5, 8
    assert L.moge_mesh_build(None, 1, 8, 8, 1, maps, 1, 8, 8, 256, 1 << 20, None) != 0 and b"channels" in L.moge_last_error()
    assert L.moge_mesh_build(None, 1, 8, 8, 1, maps, 9, 8, 8, 256, 1 << 20, None) != 0 and b"maps" in L.moge_last_error()
