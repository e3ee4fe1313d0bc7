"""Model configurations and token-grid arithmetic for the MoGe-2 hot path.

The ViT-L dictionary restates the only in-repo MoGe-2 architecture definition of the reference
(/root/reference/configs/train/v2.json:237-285).  The ViT-B / ViT-S dictionaries are the test
configurations proposed in SURVEY.md section 8 (the true HF checkpoints' decoder widths are not in the
reference repo); the engine itself is config-driven and accepts any `model_config` of this shape.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, Tuple

_BACKBONES = {
    # name: (embed_dim, depth, heads)   /root/reference/moge/model/dinov2/models/vision_transformer.py:351-390
    "dinov2_vits14": (384, 12, 6),
    "dinov2_vitb14": (768, 12, 12),
    "dinov2_vitl14": (1024, 24, 16),
}

PATCH = 14
POS_GRID = 37            # pretrained pos-embed grid (img 518 / patch 14), hub/backbones.py:18-61
INTERP_OFFSET = 0.1      # DINOv2 interpolate_offset, vision_transformer.py:202-207
LN_EPS = 1e-6            # vision_transformer.py:95
IMAGE_MEAN = (0.485, 0.456, 0.406)   # modules.py:96-97
IMAGE_STD = (0.229, 0.224, 0.225)


def backbone_dims(name: str) -> Tuple[int, int, int]:
    if name not in _BACKBONES:
        raise ValueError(f"unsupported backbone {name!r} (ViT-g / SwiGLU is outside the hot path)")
    return _BACKBONES[name]


def _decoder(dim0: int, with_normal: bool) -> Dict:
    widths = [dim0, 256, 128, 64, 32]
    resamplers = ["conv_transpose", "conv_transpose", "conv_transpose", "bilinear"]

    def head(cout):
        return {
            "dim_in": list(widths), "dim_out": [None, None, None, None, cout],
            "dim_res_blocks": list(widths), "num_res_blocks": [0, 1, 1, 1, 0],
            "res_block_in_norm": "none", "res_block_hidden_norm": "none",
            "resamplers": list(resamplers),
        }

    cfg = {
        "neck": {
            "dim_in": [dim0 + 2, 2, 2, 2, 2], "dim_out": None,
            "dim_res_blocks": list(widths), "num_res_blocks": [0, 2, 2, 2, 0],
            "res_block_in_norm": "none", "res_block_hidden_norm": "none",
            "resamplers": list(resamplers),
        },
        "points_head": head(3),
        "mask_head": head(1),
    }
    if with_normal:
        cfg["normal_head"] = head(3)
    return cfg


def model_config(size: str = "vitl", with_normal: bool = True) -> Dict:
    """size in {'vits','vitb','vitl'} -> kwargs for MoGeModel(**cfg)."""
    size = size.lower()
    if size == "vitl":
        backbone, taps = "dinov2_vitl14", [5, 11, 17, 23]
    elif size == "vitb":
        backbone, taps = "dinov2_vitb14", [2, 5, 8, 11]
    elif size == "vits":
        backbone, taps = "dinov2_vits14", [2, 5, 8, 11]
    else:
        raise ValueError(size)
    D = backbone_dims(backbone)[0]
    cfg = {"encoder": {"backbone": backbone, "intermediate_layers": taps, "dim_out": D}}
    cfg.update(_decoder(D, with_normal))
    cfg["scale_head"] = {"dims": [D, D, D, 1]}
    cfg["remap_output"] = "exp"
    cfg["num_tokens_range"] = [1200, 3600]
    return copy.deepcopy(cfg)


def v1_model_config(size: str = "vitl") -> Dict:
    """MoGe-1 kwargs (moge.model.v1.MoGeModel(**cfg)).  ViT-L is /root/reference/configs/train/v1.json as is; ViT-S / ViT-B are
    smaller test configurations (ViT-B also takes the list form of intermediate_layers and one res block with hidden == width)."""
    size = size.lower()
    if size == "vitl":
        cfg = {"encoder": "dinov2_vitl14", "remap_output": "exp", "intermediate_layers": 4, "dim_upsample": [256, 128, 64],
               "dim_times_res_block_hidden": 2, "num_res_blocks": 2, "num_tokens_range": [1200, 2500], "last_conv_channels": 32,
               "last_conv_size": 1}
    elif size == "vitb":
        cfg = {"encoder": "dinov2_vitb14", "remap_output": "exp", "intermediate_layers": [2, 5, 8, 11], "dim_proj": 256,
               "dim_upsample": [128, 128, 64], "dim_times_res_block_hidden": 1, "num_res_blocks": 1, "num_tokens_range": [1200, 2500]}
    elif size == "vits":
        cfg = {"encoder": "dinov2_vits14", "remap_output": "exp", "intermediate_layers": 4, "dim_proj": 256,
               "dim_upsample": [128, 64, 64], "dim_times_res_block_hidden": 2, "num_res_blocks": 1, "num_tokens_range": [1200, 2500]}
    else:
        raise ValueError(size)
    return copy.deepcopy(cfg)


def v1_resized_size(height: int, width: int, num_tokens: int) -> Tuple[int, int]:
    """(resized_height, resized_width) exactly as /root/reference/moge/model/v1.py:273-274 (int() truncation); the token grid
    is (rh // 14, rw // 14)."""
    resize_factor = ((num_tokens * 14 ** 2) / (height * width)) ** 0.5
    return int(height * resize_factor), int(width * resize_factor)


def token_grid(height: int, width: int, num_tokens: int) -> Tuple[int, int]:
    """(base_h, base_w) exactly as /root/reference/moge/model/v2.py:142-147 (Python round = half-to-even)."""
    aspect = width / height
    return round((num_tokens / aspect) ** 0.5), round((num_tokens * aspect) ** 0.5)


def default_num_tokens(num_tokens_range, resolution_level: int = 9) -> int:
    """/root/reference/moge/model/v2.py:236-238"""
    lo, hi = num_tokens_range
    return int(lo + (resolution_level / 9) * (hi - lo))


def uv_spans(aspect: float) -> Tuple[float, float]:
    """Half extents of the normalized view plane, geometry_torch.py:45-46."""
    d = math.sqrt(1.0 + aspect * aspect)
    return aspect / d, 1.0 / d
