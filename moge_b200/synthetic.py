"""Deterministic synthetic (random-init) MoGe-2 checkpoints.

No pretrained weights are reachable offline, so every parity test and benchmark runs on a seeded
random-init checkpoint in the reference's own file format ({'model_config', 'model'}, written by
/root/reference/moge/scripts/train.py:379-387 and read by v2.py:99-105).  The state-dict keys and shapes
restate what `MoGeModel(**cfg).state_dict()` of the reference produces (verified against the real
reference by oracle/make_golden.py); the values come from a CPU torch.Generator, so the same seed
gives the same bits here and on the GPU box.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict

import torch

from .configs import backbone_dims, PATCH, POS_GRID, IMAGE_MEAN, IMAGE_STD


def _shapes(cfg: Dict) -> "OrderedDict[str, tuple]":
    D, depth, _ = backbone_dims(cfg["encoder"]["backbone"])
    s: "OrderedDict[str, tuple]" = OrderedDict()
    s["encoder.image_mean"] = (1, 3, 1, 1)
    s["encoder.image_std"] = (1, 3, 1, 1)
    bb = "encoder.backbone."
    s[bb + "cls_token"] = (1, 1, D)
    s[bb + "pos_embed"] = (1, 1 + POS_GRID * POS_GRID, D)
    s[bb + "mask_token"] = (1, D)
    s[bb + "patch_embed.proj.weight"] = (D, 3, PATCH, PATCH)
    s[bb + "patch_embed.proj.bias"] = (D,)
    for i in range(depth):
        p = f"{bb}blocks.{i}."
        s[p + "norm1.weight"] = (D,); s[p + "norm1.bias"] = (D,)
        s[p + "attn.qkv.weight"] = (3 * D, D); s[p + "attn.qkv.bias"] = (3 * D,)
        s[p + "attn.proj.weight"] = (D, D); s[p + "attn.proj.bias"] = (D,)
        s[p + "ls1.gamma"] = (D,)
        s[p + "norm2.weight"] = (D,); s[p + "norm2.bias"] = (D,)
        s[p + "mlp.fc1.weight"] = (4 * D, D); s[p + "mlp.fc1.bias"] = (4 * D,)
        s[p + "mlp.fc2.weight"] = (D, 4 * D); s[p + "mlp.fc2.bias"] = (D,)
        s[p + "ls2.gamma"] = (D,)
    s[bb + "norm.weight"] = (D,); s[bb + "norm.bias"] = (D,)
    for j in range(len(cfg["encoder"]["intermediate_layers"])):
        s[f"encoder.output_projections.{j}.weight"] = (cfg["encoder"]["dim_out"], D, 1, 1)
        s[f"encoder.output_projections.{j}.bias"] = (cfg["encoder"]["dim_out"],)
    for stack in ("neck", "points_head", "mask_head", "normal_head"):
        if cfg.get(stack) is None:
            continue
        c = cfg[stack]
        widths = c["dim_res_blocks"]
        nlev = len(widths)
        dim_in = c["dim_in"] if isinstance(c["dim_in"], (list, tuple)) else [c["dim_in"]] * nlev
        dim_out = c["dim_out"] if isinstance(c["dim_out"], (list, tuple)) else [c["dim_out"]] * nlev
        nres = c["num_res_blocks"] if isinstance(c["num_res_blocks"], (list, tuple)) else [c["num_res_blocks"]] * nlev
        res = c["resamplers"] if isinstance(c["resamplers"], (list, tuple)) else [c["resamplers"]] * (nlev - 1)
        for l in range(nlev):
            if dim_in[l] is not None:
                s[f"{stack}.input_blocks.{l}.weight"] = (widths[l], dim_in[l], 1, 1)
                s[f"{stack}.input_blocks.{l}.bias"] = (widths[l],)
        for l in range(nlev - 1):
            if res[l] == "conv_transpose":
                s[f"{stack}.resamplers.{l}.0.weight"] = (widths[l], widths[l + 1], 2, 2)
                s[f"{stack}.resamplers.{l}.0.bias"] = (widths[l + 1],)
                s[f"{stack}.resamplers.{l}.1.weight"] = (widths[l + 1], widths[l + 1], 3, 3)
                s[f"{stack}.resamplers.{l}.1.bias"] = (widths[l + 1],)
            elif res[l] == "bilinear":
                s[f"{stack}.resamplers.{l}.1.weight"] = (widths[l + 1], widths[l], 3, 3)
                s[f"{stack}.resamplers.{l}.1.bias"] = (widths[l + 1],)
            else:
                raise ValueError(f"resampler {res[l]!r} is not used by any MoGe-2 config")
        for l in range(nlev):
            for r in range(nres[l]):
                for k in (2, 5):
                    s[f"{stack}.res_blocks.{l}.{r}.layers.{k}.weight"] = (widths[l], widths[l], 3, 3)
                    s[f"{stack}.res_blocks.{l}.{r}.layers.{k}.bias"] = (widths[l],)
        for l in range(nlev):
            if dim_out[l] is not None:
                s[f"{stack}.output_blocks.{l}.weight"] = (dim_out[l], widths[l], 1, 1)
                s[f"{stack}.output_blocks.{l}.bias"] = (dim_out[l],)
    if cfg.get("scale_head") is not None:
        dims = cfg["scale_head"]["dims"]
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            s[f"scale_head.{2 * i}.weight"] = (b, a)
            s[f"scale_head.{2 * i}.bias"] = (b,)
    return s


def expected_keys(cfg: Dict):
    """State-dict keys of `MoGeModel(**cfg)` in the reference's order (for load_state_dict's missing / unexpected report)."""
    return list(_shapes(cfg).keys())


def make_state_dict(cfg: Dict, seed: int = 0, mask_bias: float = 0.7, well_posed: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """Seeded fp32 state dict with well-scaled values (activations O(1) through all layers).

    `mask_bias` shifts the mask head's output bias so that `mask > 0.5` holds for most pixels and the
    focal/shift solve is exercised (SURVEY.md appendix B item 14).
    `well_posed=True` rewires a handful of last-level weights (see `_make_well_posed`) so that the predicted point map
    looks like a pinhole view (xy proportional to the UV planes times depth, depth within a factor of ~5): the focal/shift
    solve of infer() is then well-conditioned and the five infer() outputs can be compared end to end.  It also gives the
    normal head a dominant camera-facing component, like a trained model whose normals are near unit length: with plain random
    init the three raw components are zero-mean, |n| is close to 0 on many pixels and F.normalize (v2.py:178) amplifies the
    relative error of the raw output by sqrt(E[1/|n|^2] E[|n|^2]) ~ 1.7 (DESIGN.md section 2)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in _shapes(cfg).items():
        def randn(std=1.0):
            return torch.randn(shape, generator=g, dtype=torch.float32) * std
        if name.endswith("image_mean"):
            t = torch.tensor(IMAGE_MEAN).view(shape)
        elif name.endswith("image_std"):
            t = torch.tensor(IMAGE_STD).view(shape)
        elif name.endswith("pos_embed") or name.endswith("cls_token") or name.endswith("mask_token"):
            t = randn(0.25)
        elif "norm" in name and name.endswith(".weight") and len(shape) == 1:
            t = 1.0 + randn(0.1)
        elif "norm" in name and name.endswith(".bias"):
            t = randn(0.05)
        elif name.endswith(".gamma"):
            t = 0.25 + randn(0.05)
        elif name.endswith(".bias"):
            t = randn(0.05)
            if name.startswith("mask_head.output_blocks"):
                t = t + mask_bias
        elif name.endswith(".weight"):
            if ".resamplers." in name and name.endswith(".0.weight"):
                fan_in = shape[0]                     # ConvTranspose2d: (C_in, C_out, 2, 2)
            else:
                fan_in = 1
                for d in shape[1:]:
                    fan_in *= d
            gain = 1.0
            if name.split(".")[0] in ("neck", "points_head", "normal_head", "mask_head"):
                gain = 0.9                     # keeps the signal alive through ~30 ReLU convs without blowing up
            if "output_blocks" in name:
                gain = 0.3 if name.startswith("points_head") else 0.5     # log-depth logit within a few units
            t = randn(gain / fan_in ** 0.5)
        else:
            raise AssertionError(name)
        sd[name] = t.contiguous()
    if well_posed:
        _make_well_posed(cfg, sd)
    return sd


def _make_well_posed(cfg: Dict, sd: Dict[str, torch.Tensor], k: float = 4.0, g: float = 0.3, z_gain: float = 0.35,
                     z_bias: float = 0.8, xy_noise: float = 0.1) -> None:
    """Route the UV planes (the neck's level-4 input, v2.py:154-160) through channels 0/1 of the last decoder level into the
    x/y outputs of the points head, and temper the log-depth output: with remap 'exp' the point map becomes
    (g k u e^z, g k v e^z, e^z) + noise, i.e. a pinhole camera of focal ~ 1/(g k) looking at a rough surface at depth e^z."""
    if cfg.get("points_head") is None:
        return
    last = len(cfg["neck"]["dim_res_blocks"]) - 1
    w = sd[f"neck.input_blocks.{last}.weight"]
    w[0] = 0; w[1] = 0; w[0, 0, 0, 0] = k; w[1, 1, 0, 0] = k
    w = sd[f"points_head.input_blocks.{last}.weight"]
    w[0] = 0; w[1] = 0; w[0, 0, 0, 0] = 1; w[1, 1, 0, 0] = 1
    w = sd[f"points_head.output_blocks.{last}.weight"]
    w[0] *= xy_noise; w[1] *= xy_noise; w[2] *= z_gain; w[0, 0, 0, 0] = g; w[1, 1, 0, 0] = g
    sd[f"points_head.output_blocks.{last}.bias"][2] += z_bias
    if cfg.get("normal_head") is not None:
        sd[f"normal_head.output_blocks.{last}.weight"] *= 0.6
        sd[f"normal_head.output_blocks.{last}.bias"] += torch.tensor([0.3, -0.4, -1.2])


def save_checkpoint(path, cfg: Dict, seed: int = 0, **kw) -> None:
    """Write a reference-format checkpoint file (v2.py:99-105 reads it with weights_only=True)."""
    torch.save({"model_config": cfg, "model": make_state_dict(cfg, seed, **kw)}, path)


def synthetic_images(batch: int, height: int, width: int, seed: int = 0) -> torch.Tensor:
    """Uniform [0,1) RGB images, fp32, (B,3,H,W) -- the synthetic input of BASELINE.md section 3."""
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    return torch.rand(batch, 3, height, width, generator=g, dtype=torch.float32)


def synthetic_point_map(batch: int, height: int, width: int, focal: float, shift: float, noise: float = 0.0,
                        mask_mode: str = "all", seed: int = 0):
    """A well-posed affine point map: a smooth depth surface seen by a pinhole camera whose focal length is
    `focal` (relative to the half diagonal), with the z axis displaced by `-shift` so that the focal/shift
    solve (geometry_torch.py:115-170) should recover (focal, shift).  Returns (points (B,H,W,3), mask (B,H,W))."""
    g = torch.Generator(device="cpu").manual_seed(2000 + seed)
    aspect = width / height
    sx, sy = aspect / (1 + aspect ** 2) ** 0.5, 1 / (1 + aspect ** 2) ** 0.5
    u = (2 * (torch.arange(width, dtype=torch.float32) + 0.5) / width - 1) * sx
    v = (2 * (torch.arange(height, dtype=torch.float32) + 0.5) / height - 1) * sy
    vv, uu = torch.meshgrid(v, u, indexing="ij")
    pts, masks = [], []
    for b in range(batch):
        a = torch.rand(6, generator=g)
        z = 2.0 + 0.6 * torch.sin(3.0 * uu * (1 + a[0]) + 6.28 * a[1]) * torch.cos(2.5 * vv * (1 + a[2]) + 6.28 * a[3]) \
            + 0.5 * a[4] * uu + 0.5 * a[5] * vv
        z = z * (1.0 + 0.1 * b)
        x, y = uu * z / focal, vv * z / focal
        p = torch.stack([x, y, z - shift], dim=-1)
        if noise > 0:
            p = p + noise * torch.randn(p.shape, generator=g)
        if mask_mode == "all":
            m = torch.ones(height, width, dtype=torch.bool)
        elif mask_mode == "none":
            m = torch.zeros(height, width, dtype=torch.bool)
        elif mask_mode == "random":
            m = torch.rand(height, width, generator=g) > 0.3
        elif mask_mode == "half":
            m = torch.zeros(height, width, dtype=torch.bool); m[:, : width // 2] = True
        elif mask_mode == "single":
            m = torch.zeros(height, width, dtype=torch.bool); m[0, 0] = True
        else:
            raise ValueError(mask_mode)
        pts.append(p); masks.append(m)
    return torch.stack(pts), torch.stack(masks)
