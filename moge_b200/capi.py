"""ctypes binding of libmoge_b200.so (the C ABI declared in include/moge_b200.h).

The library is built in-tree by `__graft_entry__.build()` / moge_b200/csrc/build.sh into moge_b200/_lib/.  There is
no CPU fallback: if the shared object is missing or no sm_90 (H100) device is present the compute calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libmoge_b200.so")

MOGE_MAX_LEVELS, MOGE_MAX_TAPS, MOGE_MAX_MLP = 8, 8, 8
F32, F16, BF16, U8 = 0, 1, 2, 3
ALIGN_PLAIN, ANCHOR_DEPTH, ANCHOR_POINTS_Z, ANCHOR_POINTS_XYZ = 0, 1, 2, 3
ALIGN_MAX_POINTS = 4096          # points per anchored problem (elements per plain problem: 3x)
REMAP = {"linear": 0, "sinh": 1, "exp": 2, "sinh_exp": 3}
RESAMPLE = {"conv_transpose": 0, "bilinear": 1}

METRICS_MAX_SEGMENTS, METRICS_MAX_VARIANTS, METRICS_F1_THRESHOLDS, METRICS_F1_COUNTS, METRICS_OUT_SEGMENTS = 256, 8, 10, 90, 17
(MV_DEPTH, MV_DEPTH_SCALE, MV_DEPTH_AFFINE, MV_DISPARITY, MV_DISPARITY_FROM_DEPTH, MV_POINTS_SHIFT, MV_POINTS_SCALE,
 MV_POINTS_AFFINE) = range(8)
MESH_MAX_MAPS, MESH_MAX_CHANNELS = 8, 4
MESH_F32, MESH_U8_UNIT, MESH_UV = 0, 1, 2
MESH_HWC, MESH_CHW = 0, 1
PANORAMA_MAX_VIEWS = 20
PANORAMA_MAX_BATCH = 64
LOSS_SUMS = 4
LOSS_MASK_L2, LOSS_MASK_BCE, LOSS_EDGE, LOSS_NORMAL = range(4)
LOSS_LOCAL_PARAMS = 8
VIS_MAX_QUANTILES = 4
VIS_DEPTH, VIS_VALUE = 0, 1
GEOMETRY_MAX_REFINE_KERNEL, GEOMETRY_MAX_POOL_KERNEL, GEOMETRY_MAX_BLUR_KERNEL = 9, 15, 31
DILATE = {"mean": 0, "min": 1, "max": 2, "median": 3}
DINO_FFN = {"mlp": 0, "swiglu": 1, "swiglufused": 1, "identity": 2}
DINO_NORM, DINO_CHANNEL_MAJOR = 1, 2
DINO_MAX_GROUPS = 64


class StackConfig(C.Structure):
    _fields_ = [
        ("present", C.c_int), ("num_levels", C.c_int),
        ("dim_in", C.c_int * MOGE_MAX_LEVELS), ("dim_res_blocks", C.c_int * MOGE_MAX_LEVELS),
        ("num_res_blocks", C.c_int * MOGE_MAX_LEVELS), ("dim_out", C.c_int * MOGE_MAX_LEVELS),
        ("resamplers", C.c_int * MOGE_MAX_LEVELS),
    ]


class Config(C.Structure):
    _fields_ = [
        ("embed_dim", C.c_int), ("depth", C.c_int), ("num_heads", C.c_int),
        ("num_taps", C.c_int), ("taps", C.c_int * MOGE_MAX_TAPS), ("dim_out", C.c_int),
        ("neck", StackConfig), ("points_head", StackConfig), ("normal_head", StackConfig), ("mask_head", StackConfig),
        ("scale_head_layers", C.c_int), ("scale_head_dims", C.c_int * MOGE_MAX_MLP),
        ("remap_output", C.c_int), ("compute_dtype", C.c_int),
    ]


class V1Config(C.Structure):
    """moge_v1_config_t: MoGe-1 (moge/model/v1.py)."""
    _fields_ = [
        ("embed_dim", C.c_int), ("depth", C.c_int), ("num_heads", C.c_int),
        ("num_taps", C.c_int), ("taps", C.c_int * MOGE_MAX_TAPS), ("dim_proj", C.c_int),
        ("num_levels", C.c_int), ("dim_upsample", C.c_int * MOGE_MAX_LEVELS), ("hidden_mult", C.c_int),
        ("num_res_blocks", C.c_int), ("hidden_norm", C.c_int), ("last_res_blocks", C.c_int),
        ("last_conv_channels", C.c_int), ("last_conv_size", C.c_int), ("remap_output", C.c_int), ("compute_dtype", C.c_int),
    ]


class Group(C.Structure):
    """moge_group_t: one shape group of a mixed-shape forward call."""
    _fields_ = [
        ("image", C.c_void_p), ("image_dtype", C.c_int),
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("h", C.c_int), ("w", C.c_int),
        ("points", C.c_void_p), ("normal", C.c_void_p), ("mask_prob", C.c_void_p), ("metric_scale", C.c_void_p),
    ]


class V1Group(C.Structure):
    """moge_v1_group_t: one shape group of a mixed-shape MoGe-1 forward call."""
    _fields_ = [
        ("image", C.c_void_p), ("image_dtype", C.c_int),
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("rh", C.c_int), ("rw", C.c_int),
        ("points", C.c_void_p), ("mask", C.c_void_p),
    ]


class DinoConfig(C.Structure):
    """moge_dino_config_t: the DINOv2 backbone on its own (moge/model/dinov2)."""
    _fields_ = [
        ("embed_dim", C.c_int), ("depth", C.c_int), ("num_heads", C.c_int), ("patch_size", C.c_int),
        ("num_register_tokens", C.c_int), ("interpolate_offset", C.c_float), ("interpolate_antialias", C.c_int),
        ("ffn_layer", C.c_int), ("compute_dtype", C.c_int),
    ]


class DinoGroup(C.Structure):
    """moge_dino_group_t: one shape group of a mixed-shape backbone call."""
    _fields_ = [
        ("x", C.c_void_p), ("x_dtype", C.c_int), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("out_tokens", C.c_void_p), ("out_cls", C.c_void_p), ("out_prenorm", C.c_void_p),
    ]


class MetricVariant(C.Structure):
    """moge_metric_variant_t: a prediction map and its per-image (batch, 4) params on the device."""
    _fields_ = [("kind", C.c_int), ("src", C.c_void_p), ("params", C.c_void_p)]


class MeshMap(C.Structure):
    """moge_mesh_map_t: one attribute map of a mesh build (source, kind, channels, layout, per-channel sign / offset, destination)."""
    _fields_ = [("src", C.c_void_p), ("kind", C.c_int), ("channels", C.c_int), ("layout", C.c_int),
                ("sign", C.c_float * MESH_MAX_CHANNELS), ("offset", C.c_float * MESH_MAX_CHANNELS), ("dst", C.c_void_p)]


class PanoramaCamera(C.Structure):
    """moge_panorama_camera_t: fp32 extrinsics [R | t] (R row-major) and fp64 normalised pinhole intrinsics."""
    _fields_ = [("R", C.c_float * 9), ("t", C.c_float * 3), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double),
                ("cy", C.c_double)]


class PanoramaSplit(C.Structure):
    """moge_panorama_split_t: one panorama of a mixed-size split."""
    _fields_ = [("image", C.c_void_p), ("H", C.c_int), ("W", C.c_int), ("view0", C.c_int)]


class PanoramaLevel(C.Structure):
    """moge_panorama_level_t: one panorama's merge level in a mixed-size rhs / lsmr call."""
    _fields_ = [("h", C.c_int), ("w", C.c_int), ("view0", C.c_int), ("directions", C.c_void_p), ("b", C.c_void_p),
                ("row_mask", C.c_void_p), ("pano_mask", C.c_void_p), ("init", C.c_void_p), ("depth", C.c_void_p),
                ("stats", C.c_void_p)]


class PanoramaResize(C.Structure):
    """moge_panorama_resize_t: one map of a mixed-size resize."""
    _fields_ = [("src", C.c_void_p), ("h", C.c_int), ("w", C.c_int), ("H", C.c_int), ("W", C.c_int), ("dst", C.c_void_p)]


class PanoramaFinish(C.Structure):
    """moge_panorama_finish_t: one panorama of a mixed-size finish."""
    _fields_ = [("depth", C.c_void_p), ("mask", C.c_void_p), ("h", C.c_int), ("w", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("depth_out", C.c_void_p), ("mask_out", C.c_void_p), ("points", C.c_void_p)]


vp, ci, i64, sz = C.c_void_p, C.c_int, C.c_int64, C.c_size_t
fp, pc = C.POINTER(C.c_float), C.POINTER(PanoramaCamera)

# Every entry point of include/moge_b200.h: name -> argtypes for those returning an int status, (restype, argtypes) otherwise.
SIGNATURES = {
    "moge_last_error": (C.c_char_p, None),
    "moge_version": (C.c_char_p, None),
    "moge_engine_create": [C.POINTER(Config), ci, C.POINTER(vp)],
    "moge_engine_destroy": (None, [vp]),
    "moge_engine_set_weight": [vp, C.c_char_p, vp, C.POINTER(i64), ci, ci, vp],
    "moge_engine_finalize": [vp, vp],
    "moge_engine_workspace_bytes_groups": [vp, C.POINTER(Group), ci, C.POINTER(sz)],
    "moge_engine_forward_groups": [vp, C.POINTER(Group), ci, vp, sz, vp],
    "moge_engine_num_ops": [vp, C.POINTER(ci)],
    "moge_attention_work_list": [C.POINTER(ci), ci, ci, ci, C.POINTER(ci), ci, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)],
    "moge_engine_op_info": [vp, ci, C.c_char_p, ci, C.POINTER(C.c_double), C.POINTER(C.c_double)],
    "moge_engine_profile": [vp, fp, ci, vp],
    "moge_recover_focal_shift": [vp, vp, vp, ci, ci, ci, vp, vp, vp, vp],
    "moge_postprocess": [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp],
    "moge_peer_alloc": [sz, C.POINTER(vp), C.c_char_p],
    "moge_peer_free": [vp],
    "moge_peer_open": [C.c_char_p, C.POINTER(vp)],
    "moge_peer_close": [vp],
    "moge_peer_copy": [vp, vp, sz, vp],
    "moge_peer_flag_set": [vp, ci, vp],
    "moge_peer_flag_wait": [vp, ci, vp],
    "moge_op_linear": [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "moge_op_linear_ln": [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "moge_op_attention": [vp, vp, ci, ci, ci, ci, ci, vp],
    "moge_op_layernorm": [vp, vp, vp, vp, ci, ci, ci, vp],
    "moge_op_conv": [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp],
    "moge_op_preprocess": [vp, ci, ci, ci, ci, ci, ci, vp, ci, vp],
    "moge_op_pos_table": [vp, vp, vp, ci, ci, ci, vp, vp, vp],
    "moge_op_patch_embed": [vp, ci, ci, ci, ci, ci, ci, vp, vp, vp, vp, ci, vp, vp, vp, C.POINTER(ci), ci, vp],
    "moge_op_linear_resid_ln": [vp, vp, vp, vp, vp, vp, vp, C.POINTER(ci), ci, ci, ci, ci, vp],
    "moge_op_ln_rstd": [vp, ci, ci, ci, vp, vp],
    "moge_op_linear_ln_rows": [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "moge_op_layernorm_taps": [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp],
    "moge_align_workspace_bytes": [ci, ci, i64, ci, C.POINTER(sz)],
    "moge_align": [vp, vp, vp, vp, ci, i64, ci, vp, vp, vp, vp, sz, vp],
    "moge_align_anchored": [vp, vp, vp, ci, C.c_float, i64, ci, vp, vp, vp, vp, sz, vp],
    "moge_align_affine_lstsq": [vp, vp, vp, i64, i64, vp, vp, vp],
    "moge_engine_create_v1": [C.POINTER(V1Config), ci, C.POINTER(vp)],
    "moge_v1_workspace_bytes_groups": [vp, C.POINTER(V1Group), ci, C.POINTER(sz)],
    "moge_v1_forward_groups": [vp, C.POINTER(V1Group), ci, vp, sz, vp],
    "moge_v1_postprocess": [vp, vp, C.c_float, vp, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp],
    "moge_op_resize_bicubic_aa": [vp, ci, ci, ci, ci, ci, ci, ci, vp, vp],
    "moge_op_groupnorm_relu": [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp],
    "moge_op_conv_transpose_uv": [vp, vp, vp, vp, ci, ci, ci, ci, ci, C.c_float, C.c_float, ci, vp],
    "moge_bicubic_aa_weights": [ci, ci, ci, C.POINTER(ci), fp, ci],
    "moge_metrics_workspace_bytes": [i64, ci, ci, ci, C.POINTER(sz)],
    "moge_metrics_resize": [vp, i64, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp],
    "moge_metrics_stats": [vp, vp, vp, vp, ci, vp, vp, vp, ci, i64, ci, ci, vp, vp, vp, sz, vp],
    "moge_metrics_eval": [vp, vp, vp, C.POINTER(MetricVariant), ci, vp, vp, vp, vp, ci, vp, vp, i64, ci, ci, vp, i64, vp, sz,
                          vp],
    "moge_metrics_boundary": [vp, vp, C.POINTER(MetricVariant), fp, i64, ci, ci, vp, i64, vp],
    "moge_mesh_workspace_bytes": [i64, ci, ci, C.POINTER(sz)],
    "moge_depth_edge": [vp, vp, vp, i64, ci, ci, ci, fp, fp, vp, vp],
    "moge_mesh_count": [vp, i64, ci, ci, vp, vp, sz, vp],
    "moge_mesh_build": [vp, i64, ci, ci, ci, C.POINTER(MeshMap), ci, vp, vp, vp, sz, vp],
    "moge_normal_map": [vp, vp, i64, ci, ci, vp, vp, vp],
    "moge_normal_edge": [vp, vp, vp, vp, i64, ci, ci, ci, C.c_double, vp, vp, vp],
    "moge_panorama_split_groups": [C.POINTER(PanoramaSplit), ci, pc, ci, vp, ci, vp, vp, vp],
    "moge_panorama_workspace_bytes_groups": [C.POINTER(PanoramaLevel), ci, ci, C.POINTER(sz)],
    "moge_panorama_rhs_groups": [vp, ci, vp, ci, ci, ci, pc, C.POINTER(PanoramaLevel), ci, vp, sz, vp],
    "moge_panorama_lsmr_groups": [C.POINTER(PanoramaLevel), ci, vp, sz, vp],
    "moge_panorama_resize_groups": [C.POINTER(PanoramaResize), ci, vp],
    "moge_panorama_finish_groups": [C.POINTER(PanoramaFinish), ci, vp],
    "moge_loss_workspace_bytes": [i64, ci, ci, C.POINTER(sz)],
    "moge_loss_mask": [ci, vp, vp, vp, i64, ci, ci, vp, vp, vp, vp, sz, vp],
    "moge_loss_stencil": [ci, vp, vp, i64, ci, ci, vp, vp, vp, vp, sz, vp],
    "moge_loss_normal_map": [vp, vp, i64, ci, ci, vp, vp, vp, vp, sz, vp],
    "moge_loss_global": [vp, vp, vp, C.c_float, ci, i64, ci, ci, vp, vp, vp, sz, vp],
    "moge_loss_anchor_weight": [vp, vp, vp, vp, vp, i64, ci, ci, ci, vp, vp],
    "moge_loss_patch_mask": [vp, vp, vp, vp, C.c_float, i64, ci, ci, i64, ci, vp, vp, vp, vp],
    "moge_loss_local": [vp, vp, vp, vp, vp, C.c_float, ci, i64, ci, ci, i64, ci, vp, vp, vp, sz, vp],
    "moge_vis_workspace_bytes": [i64, ci, ci, C.POINTER(sz)],
    "moge_vis_quantiles": [vp, ci, vp, i64, ci, ci, fp, ci, vp, vp, sz, vp],
    "moge_vis_colorize": [vp, ci, ci, vp, i64, ci, ci, vp, vp, ci, vp, vp],
    "moge_vis_normal": [vp, vp, i64, ci, ci, ci, vp, vp],
    "moge_geometry_workspace_bytes": [i64, ci, ci, C.POINTER(sz)],
    "moge_refine_depth_with_normal": [vp, vp, vp, i64, ci, ci, ci, C.c_float, C.c_float, ci, vp, vp, sz, vp],
    "moge_dilate_with_mask": [vp, vp, i64, ci, ci, ci, vp, vp, vp],
    "moge_threshold_depth_change": [vp, vp, i64, ci, ci, ci, C.c_float, ci, vp, vp],
    "moge_gaussian_blur_2d": [vp, i64, ci, ci, fp, ci, vp, vp],
    "moge_dino_create": [C.POINTER(DinoConfig), ci, C.POINTER(vp)],
    "moge_dino_workspace_bytes_groups": [vp, C.POINTER(DinoGroup), ci, C.POINTER(ci), ci, ci, C.POINTER(sz)],
    "moge_dino_forward_groups": [vp, C.POINTER(DinoGroup), ci, C.POINTER(ci), ci, ci, vp, sz, vp],
}
EXPORTS = list(SIGNATURES)


class MogeError(RuntimeError):
    pass


_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """Load the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MogeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(moge_b200 has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    for name, sig in SIGNATURES.items():
        f = getattr(L, name)
        f.restype, f.argtypes = sig if isinstance(sig, tuple) else (C.c_int, sig)
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != 0:
        raise MogeError(lib().moge_last_error().decode("utf-8", "replace"))


def torch_dtype_code(dtype) -> int:
    import torch
    try:
        return {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16, torch.uint8: U8, torch.bool: U8}[dtype]
    except KeyError:
        raise MogeError(f"unsupported tensor dtype {dtype}")


def ptr(t) -> Optional[int]:
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    require_cuda("moge_b200", t)
    if not t.is_contiguous():
        raise MogeError("tensor must be contiguous")
    return t.data_ptr()


def require_cuda(what: str, *tensors) -> None:
    """Raise MogeError, naming `what`, unless every argument that is not None is a CUDA tensor."""
    import torch
    for t in tensors:
        if t is not None and not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise MogeError(f"{what} operates on CUDA tensors only (no CPU fallback)")


def mask_u8(m):
    """The contiguous uint8 view of the detached mask `m` as bool (None -> None), as the kernels take masks."""
    import torch
    return None if m is None else m.detach().to(torch.bool).contiguous().view(torch.uint8)


def check_pixels(what: str, H: int, W: int, limit: int) -> None:
    """Raise MogeError, naming `what`, when a H x W map has more than `limit` (a power of two) pixels."""
    if H * W > limit:
        raise MogeError(f"{what}: a {H} x {W} map is too large: at most 2^{limit.bit_length() - 1} pixels per image")


def workspace(query, *args, device):
    """The uint8 workspace tensor of an op-library call: `query` is its `moge_*_workspace_bytes` entry point, called with `args`.
    At least 256 bytes, so that its pointer is never null."""
    import torch
    nbytes = C.c_size_t()
    check(query(*args, C.byref(nbytes)))
    return torch.empty(max(nbytes.value, 256), dtype=torch.uint8, device=device)


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def _fill_stack(sc: StackConfig, cfg: Optional[dict]) -> None:
    if cfg is None:
        sc.present = 0
        return
    widths = list(cfg["dim_res_blocks"])
    n = len(widths)
    if n > MOGE_MAX_LEVELS:
        raise MogeError("too many decoder levels")

    def per_level(v, count, default=None):
        if isinstance(v, (list, tuple)):
            return list(v)
        return [v if v is not None else default] * count

    if cfg.get("res_block_in_norm", "layer_norm") != "none" or cfg.get("res_block_hidden_norm", "group_norm") != "none":
        raise MogeError("only norm-free residual blocks (MoGe-2 configs) are supported")
    if cfg.get("activation", "relu") != "relu" or cfg.get("dim_times_res_block_hidden", 1) != 1:
        raise MogeError("only ReLU residual blocks with hidden width == width are supported")
    sc.present, sc.num_levels = 1, n
    dim_in, dim_out = per_level(cfg["dim_in"], n), per_level(cfg["dim_out"], n)
    nres = per_level(cfg.get("num_res_blocks", 1), n)
    res = per_level(cfg["resamplers"], n - 1)
    for l in range(n):
        sc.dim_in[l] = int(dim_in[l] or 0)
        sc.dim_out[l] = int(dim_out[l] or 0)
        sc.dim_res_blocks[l] = int(widths[l])
        sc.num_res_blocks[l] = int(nres[l])
    for l in range(n - 1):
        if res[l] not in RESAMPLE:
            raise MogeError(f"resampler {res[l]!r} is not supported (MoGe-2 uses conv_transpose / bilinear)")
        sc.resamplers[l] = RESAMPLE[res[l]]


def make_config(model_config: dict, compute_dtype: int) -> Config:
    """`model_config` (the dict stored in a reference checkpoint, v2.py:99-104) -> C struct."""
    from .configs import backbone_dims
    c = Config()
    enc = model_config["encoder"]
    D, depth, heads = backbone_dims(enc["backbone"])
    c.embed_dim, c.depth, c.num_heads = D, depth, heads
    taps = enc["intermediate_layers"]
    if isinstance(taps, int):
        taps = list(range(depth - taps, depth))
    if len(taps) > MOGE_MAX_TAPS:
        raise MogeError("too many intermediate layers")
    c.num_taps = len(taps)
    for i, t in enumerate(taps):
        c.taps[i] = int(t)
    c.dim_out = int(enc["dim_out"])
    _fill_stack(c.neck, model_config["neck"])
    _fill_stack(c.points_head, model_config.get("points_head"))
    _fill_stack(c.normal_head, model_config.get("normal_head"))
    _fill_stack(c.mask_head, model_config.get("mask_head"))
    sh = model_config.get("scale_head")
    if sh is not None:
        dims = list(sh["dims"])
        if len(dims) - 1 > MOGE_MAX_MLP - 1:
            raise MogeError("scale head too deep")
        c.scale_head_layers = len(dims) - 1
        for i, d in enumerate(dims):
            c.scale_head_dims[i] = int(d)
    remap = model_config.get("remap_output", "linear")
    if remap not in REMAP:
        raise ValueError(f"Invalid remap output type: {remap}")       # same error as v2.py:135
    c.remap_output = REMAP[remap]
    c.compute_dtype = compute_dtype
    return c


V1_NORMS = {"group_norm": 0, "layer_norm": 1}


def make_v1_config(model_config: dict, compute_dtype: int) -> V1Config:
    """MoGe-1 kwargs (v1.py:149-163, defaults as there) -> C struct.  The engine validates what it covers (moge_engine_create_v1)."""
    from .configs import backbone_dims
    c = V1Config()
    D, depth, heads = backbone_dims(model_config.get("encoder", "dinov2_vitb14"))
    c.embed_dim, c.depth, c.num_heads = D, depth, heads
    taps = model_config.get("intermediate_layers", 4)
    if isinstance(taps, int):                     # get_intermediate_layers(n=int): the last n blocks
        taps = list(range(depth - taps, depth))
    if not 0 < len(taps) <= MOGE_MAX_TAPS:
        raise MogeError(f"{len(taps)} intermediate layers out of range")
    c.num_taps = len(taps)
    for i, t in enumerate(taps):
        c.taps[i] = int(t)
    c.dim_proj = int(model_config.get("dim_proj", 512))
    ups = list(model_config.get("dim_upsample", [256, 128, 128]))
    if not 0 < len(ups) <= MOGE_MAX_LEVELS:
        raise MogeError(f"{len(ups)} upsampling levels out of range")
    c.num_levels = len(ups)
    for i, d in enumerate(ups):
        c.dim_upsample[i] = int(d)
    c.hidden_mult = int(model_config.get("dim_times_res_block_hidden", 1))
    c.num_res_blocks = int(model_config.get("num_res_blocks", 1))
    norm = model_config.get("res_block_norm", "group_norm")
    if norm not in V1_NORMS:
        raise ValueError(f"Unsupported res_block_norm: {norm}")
    c.hidden_norm = V1_NORMS[norm]
    c.last_res_blocks = int(model_config.get("last_res_blocks", 0))
    c.last_conv_channels = int(model_config.get("last_conv_channels", 32))
    c.last_conv_size = int(model_config.get("last_conv_size", 1))
    remap = model_config.get("remap_output", "linear")
    if remap not in REMAP:
        raise ValueError(f"Invalid remap output type: {remap}")       # same error as v1.py:266
    c.remap_output = REMAP[remap]
    c.compute_dtype = compute_dtype
    return c
