"""Mesh and point-cloud writers with the signatures the reference's CLI calls (moge/scripts/infer.py:152-156): `save_ply` and
`save_glb`, in numpy, without trimesh.  Arguments may be numpy arrays or tensors (tensors are copied to the host).

The byte layout is this module's own: trimesh is not a dependency, so the files are not compared with what trimesh writes.
"""
from __future__ import annotations

import json
import struct

import numpy as np

__all__ = ["save_ply", "save_glb"]

_GLB_MAGIC, _GLB_VERSION = 0x46546C67, 2
_CHUNK_JSON, _CHUNK_BIN = 0x4E4F534A, 0x004E4942
_FLOAT, _UINT = 5126, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963


def _np(x, dtype=None):
    if x is None:
        return None
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    return x.astype(dtype, copy=False) if dtype is not None else x


def _colours_u8(c: np.ndarray) -> np.ndarray:
    if c.dtype == np.uint8:
        return c
    return np.clip(np.round(c.astype(np.float64) * 255), 0, 255).astype(np.uint8)


def save_ply(path, vertices, faces, vertex_colors=None, vertex_normals=None) -> None:
    """Binary little-endian PLY: vertex x, y, z (float), then nx, ny, nz (float) with normals, then red, green, blue (uchar) with
    colours (floats are written as uint8 of round(c * 255), clipped to [0, 255]); faces as uchar-counted int lists."""
    v = _np(vertices, np.float32).reshape(-1, 3)
    f = _np(faces, np.int32)
    f = f.reshape(-1, f.shape[-1] if f.ndim == 2 else 3)
    n = _np(vertex_normals, np.float32)
    c = _np(vertex_colors)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if n is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if c is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    rec = np.empty(len(v), dtype=fields)
    rec["x"], rec["y"], rec["z"] = v[:, 0], v[:, 1], v[:, 2]
    if n is not None:
        n = n.reshape(-1, 3)
        rec["nx"], rec["ny"], rec["nz"] = n[:, 0], n[:, 1], n[:, 2]
    if c is not None:
        c = _colours_u8(c).reshape(-1, 3)
        rec["red"], rec["green"], rec["blue"] = c[:, 0], c[:, 1], c[:, 2]
    types = {"<f4": "float", "u1": "uchar"}
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    header += [f"property {types[t]} {name}" for name, t in fields]
    header += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    frec = np.empty(len(f), dtype=[("n", "u1"), ("v", "<i4", (f.shape[1],))])
    frec["n"], frec["v"] = f.shape[1], f
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(rec.tobytes())
        fh.write(frec.tobytes())


def _png(texture: np.ndarray) -> bytes:
    try:
        import cv2
        ok, data = cv2.imencode(".png", cv2.cvtColor(texture, cv2.COLOR_RGB2BGR))
        if not ok:
            raise ValueError("PNG encoding failed")
        return data.tobytes()
    except ImportError:
        import io
        from PIL import Image
        out = io.BytesIO()
        Image.fromarray(texture).save(out, format="PNG")
        return out.getvalue()


def _pad4(b: bytes, fill: bytes) -> bytes:
    return b + fill * (-len(b) % 4)


def save_glb(path, vertices, faces, vertex_uvs, texture, vertex_normals=None) -> None:
    """glTF 2.0 binary with one TRIANGLES primitive: POSITION (with min / max), optional NORMAL, TEXCOORD_0, uint32 indices and a
    PBR material (metallicFactor 0.5, roughnessFactor 1.0, as the reference's CLI writes) whose base colour is `texture`
    (H, W, 3 uint8 RGB, or floats in [0, 1]) embedded as PNG.  Chunks and buffer views are 4-byte aligned."""
    v = np.ascontiguousarray(_np(vertices, np.float32).reshape(-1, 3))
    f = _np(faces)
    if f.ndim != 2 or f.shape[1] != 3:
        raise ValueError(f"save_glb writes triangles: faces must be (F, 3), not {f.shape}")
    idx = np.ascontiguousarray(f.astype(np.uint32))
    uv = np.ascontiguousarray(_np(vertex_uvs, np.float32).reshape(-1, 2))
    n = None if vertex_normals is None else np.ascontiguousarray(_np(vertex_normals, np.float32).reshape(-1, 3))
    if len(v) == 0 or len(idx) == 0:
        raise ValueError("save_glb: a glTF accessor needs at least one element; the mesh is empty")
    if len(uv) != len(v) or (n is not None and len(n) != len(v)):
        raise ValueError("save_glb: vertices, uvs and normals must have the same count")
    tex = _colours_u8(_np(texture))
    blobs, views, accessors = [], [], []

    def add_view(data: bytes, target=None):
        offset = sum(len(b) for b in blobs)
        view = {"buffer": 0, "byteOffset": offset, "byteLength": len(data)}
        if target is not None:
            view["target"] = target
        views.append(view)
        blobs.append(_pad4(data, b"\0"))
        return len(views) - 1

    def add_accessor(arr: np.ndarray, ctype: int, kind: str, target: int, bounds: bool = False):
        acc = {"bufferView": add_view(arr.tobytes(), target), "componentType": ctype, "count": int(arr.shape[0]), "type": kind}
        if bounds:
            acc["min"], acc["max"] = arr.min(axis=0).tolist(), arr.max(axis=0).tolist()
        accessors.append(acc)
        return len(accessors) - 1

    attributes = {"POSITION": add_accessor(v, _FLOAT, "VEC3", _ARRAY_BUFFER, bounds=True)}
    if n is not None:
        attributes["NORMAL"] = add_accessor(n, _FLOAT, "VEC3", _ARRAY_BUFFER)
    attributes["TEXCOORD_0"] = add_accessor(uv, _FLOAT, "VEC2", _ARRAY_BUFFER)
    indices = add_accessor(idx.reshape(-1), _UINT, "SCALAR", _ELEMENT_ARRAY_BUFFER)
    image_view = add_view(_png(np.ascontiguousarray(tex)))
    binary = b"".join(blobs)
    gltf = {
        "asset": {"version": "2.0", "generator": "moge_b200.export"},
        "scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0}],
        "meshes": [{"primitives": [{"attributes": attributes, "indices": indices, "material": 0, "mode": 4}]}],
        "materials": [{"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "metallicFactor": 0.5, "roughnessFactor": 1.0}}],
        "textures": [{"sampler": 0, "source": 0}],
        "samplers": [{}],
        "images": [{"bufferView": image_view, "mimeType": "image/png"}],
        "accessors": accessors, "bufferViews": views, "buffers": [{"byteLength": len(binary)}],
    }
    js = _pad4(json.dumps(gltf, separators=(",", ":")).encode("utf-8"), b" ")
    total = 12 + 8 + len(js) + 8 + len(binary)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<III", _GLB_MAGIC, _GLB_VERSION, total))
        fh.write(struct.pack("<II", len(js), _CHUNK_JSON))
        fh.write(js)
        fh.write(struct.pack("<II", len(binary), _CHUNK_BIN))
        fh.write(binary)
