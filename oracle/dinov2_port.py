"""The DINOv2 backbone's get_intermediate_layers (moge/model/dinov2/models/vision_transformer.py:283-333) restated on a state
dict with the oracle port's encoder pieces (oracle/moge_port.py: pos_embed_for_grid, vit_block).  TEST AND BENCHMARK
INFRASTRUCTURE ONLY: the fp32 checker of tests/test_gpu_dinov2.py and, run in half precision, the comparator of
tools/bench_dinov2.py.  It runs on whatever device and dtype its inputs have."""
from typing import Dict, List

import torch
import torch.nn.functional as F

from moge_b200.configs import LN_EPS, PATCH
from oracle.moge_port import pos_embed_for_grid, vit_block


def intermediate_layers(sd: Dict[str, torch.Tensor], x: torch.Tensor, layers: List[int], heads: int, prefix: str = "",
                        norm: bool = True) -> List[torch.Tensor]:
    """x (B,3,H,W) normalised -> the patch tokens (B, T, D) after each block of `layers`, through the final norm (norm=True);
    `prefix` is the backbone's key prefix in `sd` ('' for a backbone state dict, 'encoder.backbone.' for MoGe-2)."""
    p = prefix
    D = sd[p + "cls_token"].shape[-1]
    h, w = x.shape[-2] // PATCH, x.shape[-1] // PATCH
    depth = 1 + max(int(k[len(p) + 7:].split(".")[0]) for k in sd if k.startswith(p + "blocks."))
    t = F.conv2d(x, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"], stride=PATCH)
    B = t.shape[0]
    t = t.flatten(2).transpose(1, 2)
    t = torch.cat([sd[p + "cls_token"].expand(B, -1, -1), t], dim=1) + pos_embed_for_grid(sd[p + "pos_embed"], h, w).to(t.dtype)
    out = []
    for i in range(depth):
        t = vit_block(t, sd, f"{p}blocks.{i}.", heads)
        if i in layers:
            y = F.layer_norm(t, (D,), sd[p + "norm.weight"], sd[p + "norm.bias"], LN_EPS) if norm else t
            out.append(y[:, 1:])
    return out
