"""CPU oracle for the MoGe-1 `forward()` / `infer()` path.  TEST INFRASTRUCTURE ONLY.

A functional fp32 restatement (plain torch ops on a state dict) of /root/reference/moge/model/v1.py, written from the algorithm:
  forward()      v1.py:269-299 (Head.forward :111-142, ResidualConvBlock :24-58, DINOv2 get_intermediate_layers)
  postprocess()  v1.py:352-380
  infer()        v1.py:301-392
It shares the DINOv2 block, pos-embed resampling, UV planes, remap and focal/shift solve of oracle/moge_port.py.
oracle/make_v1_golden.py pins it against the unmodified reference; on the GPU box it is the checker of tests/test_gpu_v1.py.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from moge_b200.configs import backbone_dims, v1_resized_size, PATCH, LN_EPS
from oracle.moge_port import pos_embed_for_grid, vit_block, view_plane_uv, remap_points, recover_focal_shift


def _taps(cfg: Dict, depth: int):
    t = cfg.get("intermediate_layers", 4)
    return list(range(depth - t, depth)) if isinstance(t, int) else list(t)


def encode(cfg: Dict, sd: Dict[str, torch.Tensor], x14: torch.Tensor):
    """normalised (B,3,14h,14w) -> the normalised patch tokens of the tapped blocks, each (B,D,h,w)."""
    D, depth, heads = backbone_dims(cfg["encoder"])
    B, _, H14, W14 = x14.shape
    h, w = H14 // PATCH, W14 // PATCH
    x = F.conv2d(x14, sd["backbone.patch_embed.proj.weight"], sd["backbone.patch_embed.proj.bias"], stride=PATCH)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat([sd["backbone.cls_token"].expand(B, -1, -1), x], dim=1)
    x = x + pos_embed_for_grid(sd["backbone.pos_embed"], h, w).to(x.dtype)
    taps = _taps(cfg, depth)
    feats = []
    for i in range(depth):
        x = vit_block(x, sd, f"backbone.blocks.{i}.", heads)
        if i in taps:
            y = F.layer_norm(x, (D,), sd["backbone.norm.weight"], sd["backbone.norm.bias"], LN_EPS)
            feats.append(y[:, 1:].permute(0, 2, 1).reshape(B, D, h, w))
    return feats


def _conv3(x, w, b):
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), w, b)


def _cat_uv(x, aspect):
    B, _, h, w = x.shape
    uv = view_plane_uv(w, h, aspect, x.dtype, x.device).permute(2, 0, 1)[None].expand(B, -1, -1, -1)
    return torch.cat([x, uv], dim=1)


@torch.no_grad()
def forward(cfg: Dict, sd: Dict[str, torch.Tensor], image: torch.Tensor, num_tokens: int) -> Dict[str, torch.Tensor]:
    """v1.py:269-299.  image (B,3,H,W) in [0,1]; runs in the dtype / on the device of its inputs."""
    B, _, H, W = image.shape
    rh, rw = v1_resized_size(H, W, int(num_tokens))
    x = F.interpolate(image, (rh, rw), mode="bicubic", align_corners=False, antialias=True)
    x = (x - sd["image_mean"]) / sd["image_std"]
    x14 = F.interpolate(x, (rh // PATCH * PATCH, rw // PATCH * PATCH), mode="bilinear", align_corners=False, antialias=True)
    feats = encode(cfg, sd, x14)
    y = sum(F.conv2d(f, sd[f"head.projects.{j}.weight"], sd[f"head.projects.{j}.bias"]) for j, f in enumerate(feats))
    aspect = rw / rh
    norm = cfg.get("res_block_norm", "group_norm")
    for l in range(len(cfg.get("dim_upsample", [256, 128, 128]))):
        p = f"head.upsample_blocks.{l}."
        y = F.conv_transpose2d(_cat_uv(y, aspect), sd[p + "0.0.weight"], sd[p + "0.0.bias"], stride=2)
        y = _conv3(y, sd[p + "0.1.weight"], sd[p + "0.1.bias"])
        for r in range(cfg.get("num_res_blocks", 1)):
            q = f"{p}{1 + r}.layers."
            hid = sd[q + "3.weight"].shape[0]
            t = F.relu(F.group_norm(y, 1, sd[q + "0.weight"], sd[q + "0.bias"], 1e-5))
            t = _conv3(t, sd[q + "2.weight"], sd[q + "2.bias"])
            t = F.relu(F.group_norm(t, hid // 32 if norm == "group_norm" else 1, sd[q + "3.weight"], sd[q + "3.bias"], 1e-5))
            y = y + _conv3(t, sd[q + "5.weight"], sd[q + "5.bias"])
    y = _cat_uv(F.interpolate(y, (rh, rw), mode="bilinear", align_corners=False), aspect)
    outs = []
    for k in range(2):
        p = f"head.output_block.{k}."
        t = F.relu(_conv3(y, sd[p + "0.weight"], sd[p + "0.bias"]))
        outs.append(F.conv2d(t, sd[p + "2.weight"], sd[p + "2.bias"]))
    points = F.interpolate(outs[0], (H, W), mode="bilinear", align_corners=False)
    mask = F.interpolate(outs[1], (H, W), mode="bilinear", align_corners=False)
    return {"points": remap_points(points.permute(0, 2, 3, 1), cfg.get("remap_output", "linear")), "mask": mask.squeeze(1)}


def postprocess(points: torch.Tensor, mask: torch.Tensor, aspect: float, mask_threshold: float = 0.5, fov_x=None,
                force_projection: bool = True, apply_mask: bool = True, focal_shift=None) -> Dict[str, torch.Tensor]:
    """v1.py:352-380 on raw forward() outputs (fp32, batched).  focal_shift=(focal, shift) injects a given solve."""
    points = points.clone().float()
    mask_b = mask.float() > mask_threshold
    if focal_shift is not None:
        focal, shift = focal_shift
    elif fov_x is None:
        focal, shift = recover_focal_shift(points, mask_b)
    else:
        focal = aspect / (1 + aspect ** 2) ** 0.5 / torch.tan(torch.deg2rad(torch.as_tensor(fov_x, dtype=points.dtype, device=points.device) / 2))
        if focal.ndim == 0:
            focal = focal[None].expand(points.shape[0])
        _, shift = recover_focal_shift(points, mask_b, focal=focal)
    fx = focal / 2 * (1 + aspect ** 2) ** 0.5 / aspect
    fy = focal / 2 * (1 + aspect ** 2) ** 0.5
    K = torch.zeros(points.shape[0], 3, 3, dtype=points.dtype, device=points.device)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = fx, fy, 0.5, 0.5, 1.0
    depth = points[..., 2] + shift[:, None, None]
    if force_projection:
        Hh, Ww = depth.shape[-2:]
        u = (torch.arange(Ww, dtype=depth.dtype, device=depth.device) + 0.5) / Ww
        v = (torch.arange(Hh, dtype=depth.dtype, device=depth.device) + 0.5) / Hh
        x = (u[None, None, :] - 0.5) / fx[:, None, None] * depth
        y = (v[None, :, None] - 0.5) / fy[:, None, None] * depth
        points = torch.stack([x, y, depth], dim=-1)
    else:
        points[..., 2] += shift[:, None, None]
    if apply_mask:
        points = torch.where(mask_b[..., None], points, torch.inf)
        depth = torch.where(mask_b, depth, torch.inf)
    return {"points": points, "intrinsics": K, "depth": depth, "mask": mask_b}


@torch.no_grad()
def infer(cfg: Dict, sd: Dict[str, torch.Tensor], image: torch.Tensor, fov_x=None, resolution_level: int = 9,
          num_tokens: Optional[int] = None, apply_mask: bool = True, force_projection: bool = True, mask_threshold: float = 0.5):
    """v1.py:301-392 with use_fp16=False.  image (B,3,H,W) or (3,H,W) fp32 in [0,1]."""
    squeeze = image.dim() == 3
    if squeeze:
        image = image[None]
    H, W = image.shape[-2:]
    if num_tokens is None:
        lo, hi = cfg.get("num_tokens_range", [1200, 2500])
        num_tokens = int(lo + (resolution_level / 9) * (hi - lo))
    raw = forward(cfg, sd, image.float(), num_tokens)
    ret = postprocess(raw["points"], raw["mask"], W / H, mask_threshold, fov_x, force_projection, apply_mask)
    if squeeze:
        ret = {k: v[0] for k, v in ret.items()}
    return ret
