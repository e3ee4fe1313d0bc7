"""ctypes binding of libmoge_b200.so (the C ABI declared in include/moge_b200.h).

The library is built in-tree by `__graft_entry__.build()` / moge_b200/csrc/build.sh into moge_b200/_lib/.  There is
no CPU fallback: if the shared object is missing or no sm_90 (H100) device is present the compute calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# MOGE_B200_LIB selects an A/B variant build (moge_b200/csrc/build.sh with MG_VARIANT=...); default: the product library
LIB_PATH = os.environ.get("MOGE_B200_LIB") or os.path.join(_HERE, "_lib", "libmoge_b200.so")

MOGE_MAX_LEVELS, MOGE_MAX_TAPS, MOGE_MAX_MLP = 8, 8, 8
F32, F16, BF16, U8 = 0, 1, 2, 3
REMAP = {"linear": 0, "sinh": 1, "exp": 2, "sinh_exp": 3}
RESAMPLE = {"conv_transpose": 0, "bilinear": 1}

EXPORTS = [
    "moge_last_error", "moge_version", "moge_engine_create", "moge_engine_destroy", "moge_engine_set_weight",
    "moge_engine_finalize", "moge_engine_workspace_bytes", "moge_engine_forward", "moge_engine_workspace_bytes_groups",
    "moge_engine_forward_groups", "moge_engine_num_ops", "moge_engine_op_info", "moge_engine_profile", "moge_attention_work_list", "moge_recover_focal_shift",
    "moge_postprocess", "moge_peer_alloc", "moge_peer_free", "moge_peer_open", "moge_peer_close", "moge_peer_copy", "moge_peer_flag_set",
    "moge_peer_flag_wait", "moge_op_linear", "moge_op_linear_ln", "moge_op_attention", "moge_op_layernorm", "moge_op_conv",
]


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


class Group(C.Structure):
    """moge_group_t: one shape group of a mixed-shape forward call."""
    _fields_ = [
        ("image", C.c_void_p), ("image_dtype", C.c_int),
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("h", C.c_int), ("w", C.c_int),
        ("points", C.c_void_p), ("normal", C.c_void_p), ("mask_prob", C.c_void_p), ("metric_scale", C.c_void_p),
    ]


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
    vp, ci, cf = C.c_void_p, C.c_int, C.c_void_p
    L.moge_last_error.restype = C.c_char_p
    L.moge_version.restype = C.c_char_p
    L.moge_engine_create.argtypes = [C.POINTER(Config), ci, C.POINTER(vp)]
    L.moge_engine_destroy.argtypes = [vp]
    L.moge_engine_destroy.restype = None
    L.moge_engine_set_weight.argtypes = [vp, C.c_char_p, vp, C.POINTER(C.c_int64), ci, ci, vp]
    L.moge_engine_finalize.argtypes = [vp, vp]
    L.moge_engine_workspace_bytes.argtypes = [vp, ci, ci, ci, ci, ci, C.POINTER(C.c_size_t)]
    L.moge_engine_forward.argtypes = [vp, vp, ci, ci, ci, ci, ci, ci, vp, C.c_size_t, cf, cf, cf, cf, vp]
    L.moge_engine_workspace_bytes_groups.argtypes = [vp, C.POINTER(Group), ci, C.POINTER(C.c_size_t)]
    L.moge_engine_forward_groups.argtypes = [vp, C.POINTER(Group), ci, vp, C.c_size_t, vp]
    L.moge_engine_num_ops.argtypes = [vp, C.POINTER(ci)]
    L.moge_attention_work_list.argtypes = [C.POINTER(ci), ci, ci, ci, C.POINTER(ci), ci, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)]
    L.moge_engine_op_info.argtypes = [vp, ci, C.c_char_p, ci, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.moge_engine_profile.argtypes = [vp, C.POINTER(C.c_float), ci, vp]
    L.moge_recover_focal_shift.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, vp, vp]
    L.moge_postprocess.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp]
    L.moge_peer_alloc.argtypes = [C.c_size_t, C.POINTER(vp), C.c_char_p]
    L.moge_peer_free.argtypes = [vp]
    L.moge_peer_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.moge_peer_close.argtypes = [vp]
    L.moge_peer_copy.argtypes = [vp, vp, C.c_size_t, vp]
    L.moge_peer_flag_set.argtypes = [vp, ci, vp]
    L.moge_peer_flag_wait.argtypes = [vp, ci, vp]
    L.moge_op_linear.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    L.moge_op_linear_ln.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    L.moge_op_attention.argtypes = [vp, vp, ci, ci, ci, ci, ci, vp]
    L.moge_op_layernorm.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
    L.moge_op_conv.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp]
    for name in EXPORTS:
        if name not in ("moge_last_error", "moge_version", "moge_engine_destroy"):
            getattr(L, name).restype = ci
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
    if not t.is_cuda:
        raise MogeError("moge_b200 operates on CUDA tensors only (no CPU fallback)")
    if not t.is_contiguous():
        raise MogeError("tensor must be contiguous")
    return t.data_ptr()


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
