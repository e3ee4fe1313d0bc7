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


def _v1_shapes(cfg: Dict) -> "OrderedDict[str, tuple]":
    """State-dict shapes of the reference `moge.model.v1.MoGeModel(**cfg)` (v1.py:145-204): its buffers, the DINOv2 backbone under
    `backbone.`, and the Head under `head.`."""
    D, depth, _ = backbone_dims(cfg["encoder"])
    s: "OrderedDict[str, tuple]" = OrderedDict()
    s["image_mean"] = (1, 3, 1, 1)
    s["image_std"] = (1, 3, 1, 1)
    for k, v in _shapes({"encoder": {"backbone": cfg["encoder"], "intermediate_layers": [], "dim_out": D}}).items():
        if k.startswith("encoder.backbone."):
            s[k[len("encoder."):]] = v
    taps = cfg.get("intermediate_layers", 4)
    nt = taps if isinstance(taps, int) else len(taps)
    P = cfg.get("dim_proj", 512)
    ups = list(cfg.get("dim_upsample", [256, 128, 128]))
    hm, nres = cfg.get("dim_times_res_block_hidden", 1), cfg.get("num_res_blocks", 1)
    lc, lcs, lrb = cfg.get("last_conv_channels", 32), cfg.get("last_conv_size", 1), cfg.get("last_res_blocks", 0)

    def res_block(p, c, hid):
        s[p + "layers.0.weight"] = (c,); s[p + "layers.0.bias"] = (c,)
        s[p + "layers.2.weight"] = (hid, c, 3, 3); s[p + "layers.2.bias"] = (hid,)
        s[p + "layers.3.weight"] = (hid,); s[p + "layers.3.bias"] = (hid,)
        s[p + "layers.5.weight"] = (c, hid, 3, 3); s[p + "layers.5.bias"] = (c,)

    for j in range(nt):
        s[f"head.projects.{j}.weight"] = (P, D, 1, 1)
        s[f"head.projects.{j}.bias"] = (P,)
    for l, (ci, co) in enumerate(zip([P] + ups[:-1], ups)):
        p = f"head.upsample_blocks.{l}."
        s[p + "0.0.weight"] = (ci + 2, co, 2, 2); s[p + "0.0.bias"] = (co,)
        s[p + "0.1.weight"] = (co, co, 3, 3); s[p + "0.1.bias"] = (co,)
        for r in range(nres):
            res_block(f"{p}{1 + r}.", co, hm * co)
    for k, n in enumerate((3, 1)):
        p = f"head.output_block.{k}."
        s[p + "0.weight"] = (lc, ups[-1] + 2, 3, 3); s[p + "0.bias"] = (lc,)
        for r in range(lrb):
            res_block(f"{p}{1 + r}.", lc, hm * lc)
        s[f"{p}{2 + lrb}.weight"] = (n, lc, lcs, lcs); s[f"{p}{2 + lrb}.bias"] = (n,)
    return s


def v1_expected_keys(cfg: Dict):
    """State-dict keys of the reference `moge.model.v1.MoGeModel(**cfg)`, in its order."""
    return list(_v1_shapes(cfg).keys())


def make_v1_state_dict(cfg: Dict, seed: int = 0, mask_bias: float = 1.0, well_posed: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """Seeded fp32 MoGe-1 state dict, values scaled as make_state_dict's.  The v1 mask is thresholded raw (no sigmoid) at 0.5, so
    `mask_bias` lifts the mask output's bias until most pixels pass.  `well_posed=True`: the points branch of the output block
    carries the UV planes (u, v at the centre tap of channels 0 / 1 of its 3x3 conv, kept positive through the ReLU by a bias) into
    x / y, and its log-depth output is tempered: with remap 'exp' the point map is (g u e^z, g v e^z, e^z) + noise, a pinhole view
    with focal ~ 1/g, so the focal/shift solve of infer() is well-conditioned."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in _v1_shapes(cfg).items():
        def randn(std=1.0):
            return torch.randn(shape, generator=g, dtype=torch.float32) * std
        if name == "image_mean":
            t = torch.tensor(IMAGE_MEAN).view(shape)
        elif name == "image_std":
            t = torch.tensor(IMAGE_STD).view(shape)
        elif name.endswith("pos_embed") or name.endswith("cls_token") or name.endswith("mask_token"):
            t = randn(0.25)
        elif len(shape) == 1 and name.endswith(".weight"):          # LayerNorm / GroupNorm scales
            t = 1.0 + randn(0.1)
        elif name.endswith(".gamma"):
            t = 0.25 + randn(0.05)
        elif name.endswith(".bias"):
            t = randn(0.05)
            if name.startswith("head.output_block.1.") and shape == (1,):
                t = t + mask_bias
        else:
            if ".upsample_blocks." in name and name.endswith(".0.0.weight"):
                fan_in = shape[0]                     # ConvTranspose2d: (C_in, C_out, 2, 2)
            else:
                fan_in = 1
                for d in shape[1:]:
                    fan_in *= d
            gain = 0.3 if (name.startswith("head.output_block.") and shape[-1] == cfg.get("last_conv_size", 1) and shape[0] <= 3) else 1.0
            t = randn(gain / fan_in ** 0.5)
        sd[name] = t.contiguous()
    if well_posed:
        _make_v1_well_posed(cfg, sd)
    return sd


def _make_v1_well_posed(cfg: Dict, sd: Dict[str, torch.Tensor], gf: float = 1.2, lift: float = 2.0, z_gain: float = 0.35,
                        z_bias: float = 0.8, xy_noise: float = 0.1) -> None:
    C = list(cfg.get("dim_upsample", [256, 128, 128]))[-1]
    w = sd["head.output_block.0.0.weight"]
    w[0] = 0; w[1] = 0; w[0, C, 1, 1] = 1.0; w[1, C + 1, 1, 1] = 1.0
    b = sd["head.output_block.0.0.bias"]
    b[0] = lift; b[1] = lift                              # relu(u + lift) = u + lift: |u|, |v| < 1
    last = 2 + cfg.get("last_res_blocks", 0)
    wo = sd[f"head.output_block.0.{last}.weight"]
    bo = sd[f"head.output_block.0.{last}.bias"]
    wo[0] *= xy_noise; wo[1] *= xy_noise; wo[2] *= z_gain
    wo[0, 0] = gf; wo[1, 1] = gf; wo[0, 1] = 0; wo[1, 0] = 0
    bo[0] = -gf * lift; bo[1] = -gf * lift; bo[2] += z_bias


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


def synthetic_alignment_case(batch_shape, n: int, seed: int = 0, single_positive: bool = False):
    """Seeded inputs of the alignment solvers (moge_b200.alignment): points_src, points_tgt (*batch_shape, n, 3) and weight
    (*batch_shape, n), fp32.  tgt ~ scale * src + shift per image with a known scale and shift, plus small noise, ~10 % gross
    outliers, ~30 % zero weights, x and y components of both signs, and ~5 % of the points duplicated (src, tgt and weight) from
    other points.  single_positive: the first image keeps one positive weight only."""
    g = torch.Generator(device="cpu").manual_seed(3000 + seed)
    bs = tuple(batch_shape)
    tgt = torch.randn(*bs, n, 3, generator=g) + torch.tensor([0.0, 0.0, 3.0])
    scale = 0.5 + torch.rand(*bs, 1, 1, generator=g)
    shift = 0.3 * torch.randn(*bs, 1, 3, generator=g)
    src = (tgt - shift) / scale + 0.01 * torch.randn(*bs, n, 3, generator=g)
    outlier = torch.rand(*bs, n, 1, generator=g) < 0.1
    src = torch.where(outlier, src + 2.0 * torch.randn(*bs, n, 3, generator=g), src)
    weight = 0.1 + torch.rand(*bs, n, generator=g)
    weight = torch.where(torch.rand(*bs, n, generator=g) < 0.3, torch.zeros_like(weight), weight)
    dup = torch.randperm(n, generator=g)[: max(1, n // 20)]
    orig = torch.randint(0, n, (dup.numel(),), generator=g)
    src[..., dup, :], tgt[..., dup, :], weight[..., dup] = src[..., orig, :], tgt[..., orig, :], weight[..., orig]
    if single_positive:
        first = weight.reshape(-1, n)[0]
        first.zero_()
        first[n // 2] = 0.7
    return src.contiguous(), tgt.contiguous(), weight.contiguous()


ALIGNMENT_FUNCTIONS = ("align", "align_depth_scale", "align_depth_affine", "align_points_scale", "align_points_scale_z_shift",
                       "align_points_scale_xyz_shift", "align_points_z_shift", "align_points_xyz_shift", "align_affine_lstsq")


def alignment_arguments(fn: str, batch_shape, n: int, seed: int, trunc=None, single_positive: bool = False):
    """Positional arguments of alignment function `fn` on synthetic_alignment_case(batch_shape, n, seed): depth functions, align
    and align_affine_lstsq take the z components.  trunc: None, a float, or "per_element" (align only: a seeded (..., n) tensor);
    align_affine_lstsq takes trunc = "weighted" for its weights (else w = None)."""
    src, tgt, w = synthetic_alignment_case(batch_shape, n, seed, single_positive)
    if fn == "align_affine_lstsq":
        return (src[..., 2], tgt[..., 2], w if trunc == "weighted" else None)
    if trunc == "per_element":
        g = torch.Generator(device="cpu").manual_seed(4000 + seed)
        trunc = 0.05 + 0.1 * torch.rand(*tuple(batch_shape), n, generator=g)
    if fn in ("align", "align_depth_scale", "align_depth_affine"):
        return (src[..., 2], tgt[..., 2], w, trunc)
    return (src, tgt, w, trunc)


METRICS_KEYS = {
    "moge2": ("points_metric", "depth_metric", "intrinsics"),
    "moge1": ("points_scale_invariant", "depth_scale_invariant", "intrinsics"),
    "depth_affine": ("depth_affine_invariant",),
    "disparity": ("disparity_affine_invariant",),
    "points_affine": ("points_affine_invariant",),
}


def _unproject(depth: torch.Tensor, fx: float, fy: float) -> torch.Tensor:
    H, W = depth.shape
    u = (torch.arange(W, dtype=torch.float32) + 0.5) / W
    v = (torch.arange(H, dtype=torch.float32) + 0.5) / H
    return torch.stack([(u[None, :] - 0.5) / fx * depth, (v[:, None] - 0.5) / fy * depth, depth], dim=-1)


def _box(g: torch.Generator, H: int, W: int, lo: float, hi: float):
    h = max(1, int(H * (lo + (hi - lo) * torch.rand((), generator=g).item())))
    w = max(1, int(W * (lo + (hi - lo) * torch.rand((), generator=g).item())))
    i = int(torch.randint(0, max(1, H - h), (), generator=g))
    j = int(torch.randint(0, max(1, W - w), (), generator=g))
    return i, j, h, w


def _scene(g: torch.Generator, H: int, W: int):
    """The GT scene of synthetic_metrics_case: (fx, fy, depth, points, mask) -- piecewise-planar depth (a tilted background plane
    and occluding tilted boxes), points by unprojection with normalised intrinsics, a mask with box holes and 5 % dropouts."""
    fx = 0.55 + 0.4 * torch.rand((), generator=g).item()
    fy = fx * W / H
    u = (torch.arange(W, dtype=torch.float32) + 0.5) / W
    v = (torch.arange(H, dtype=torch.float32) + 0.5) / H
    depth = 6.0 + 2.0 * (u[None, :] - 0.5) + 3.0 * (v[:, None] - 0.5)
    for _ in range(4):
        i, j, h, w = _box(g, H, W, 0.15, 0.4)
        z = 1.5 + 3.0 * torch.rand((), generator=g).item()
        tilt = 0.5 * (torch.rand(2, generator=g) - 0.5)
        depth[i:i + h, j:j + w] = z + tilt[0] * (u[None, j:j + w] - 0.5) + tilt[1] * (v[i:i + h, None] - 0.5)
    points = _unproject(depth, fx, fy)
    mask = torch.ones(H, W, dtype=torch.bool)
    for _ in range(3):
        i, j, h, w = _box(g, H, W, 0.05, 0.15)
        mask[i:i + h, j:j + w] = False
    mask &= torch.rand(H, W, generator=g) > 0.05
    return fx, fy, depth, points, mask


def synthetic_metrics_case(seed: int, H: int, W: int, keys, is_metric: bool = True, sharp: bool = True, segments: int = 0,
                           negative: bool = False):
    """(pred, gt) dicts of CPU fp32 tensors for compute_metrics, from a seeded generator.

    GT: piecewise-planar depth (a tilted background plane and occluding tilted boxes), points by unprojection with normalised
    intrinsics, a mask with box holes and 5 % dropouts.  With `segments` > 0, box segments (later ones overwrite earlier ones)
    plus one tiny segment (under 10 low-resolution pixels), one label whose id is absent from the map and one duplicated id.
    Predictions: GT perturbed by scale, shift, smooth noise, 1 % outliers and a blur across the occlusion edges; `negative` puts a
    few negative depths in.  `keys` names the predicted entries (METRICS_KEYS)."""
    g = torch.Generator().manual_seed(seed)
    fx, fy, depth, points, mask = _scene(g, H, W)
    K = torch.tensor([[fx, 0, 0.5], [0, fy, 0.5], [0, 0, 1]], dtype=torch.float32)
    gt = {"depth": depth, "points": points, "depth_mask": mask, "intrinsics": K, "is_metric": is_metric, "has_sharp_boundary": sharp}
    if segments:
        seg = torch.zeros(H, W, dtype=torch.int32)
        labels = {}
        for s in range(1, segments + 1):
            i, j, h, w = _box(g, H, W, 0.1, 0.35)
            seg[i:i + h, j:j + w] = s
            labels[f"seg{s}"] = s
        ti, tj = H // 2, W // 2
        seg[ti:ti + max(1, H // 40), tj:tj + max(1, W // 40)] = segments + 1     # tiny: a handful of low-resolution pixels
        labels["tiny"] = segments + 1
        labels["absent"] = segments + 1000
        labels["duplicate"] = 1
        gt["segmentation_mask"], gt["segmentation_labels"] = seg, labels
    # prediction: smooth noise, blurred edges, outliers
    smooth = torch.nn.functional.interpolate(torch.randn(1, 1, 8, 8, generator=g), size=(H, W), mode="bilinear", align_corners=False)[0, 0]
    blurred = torch.nn.functional.avg_pool2d(depth[None, None], 5, 1, 2, count_include_pad=False)[0, 0]
    pd = blurred * (1 + 0.03 * smooth)
    out = torch.rand(H, W, generator=g) < 0.01
    pd = torch.where(out, pd * (0.3 + 2 * torch.rand(H, W, generator=g)), pd)
    if negative:
        pd = torch.where(torch.rand(H, W, generator=g) < 0.002, -pd, pd)
    scale, shift = 0.7 + 0.6 * torch.rand((), generator=g).item(), 0.3 * torch.rand((), generator=g).item()
    pfx = fx * (1 + 0.1 * (torch.rand((), generator=g).item() - 0.5))
    ppts = _unproject(pd, pfx, pfx * W / H)
    pred = {}
    for k in keys:
        if k == "intrinsics":
            pred[k] = torch.tensor([[pfx, 0, 0.5], [0, pfx * W / H, 0.5], [0, 0, 1]], dtype=torch.float32)
        elif k == "depth_metric":
            pred[k] = pd.clone()
        elif k == "depth_scale_invariant":
            pred[k] = pd * scale
        elif k == "depth_affine_invariant":
            pred[k] = pd * scale + shift
        elif k == "disparity_affine_invariant":
            pred[k] = scale / pd + 0.05 * shift
        elif k == "points_metric":
            pred[k] = ppts + torch.tensor([0.02, -0.01, 0.05])
        elif k == "points_scale_invariant":
            pred[k] = ppts * scale
        elif k == "points_affine_invariant":
            pred[k] = ppts * scale + torch.tensor([0.1, -0.05, shift])
        else:
            raise KeyError(k)
    return pred, gt


def synthetic_mesh_case(seed: int, B: int, H: int, W: int):
    """(output, image) for mesh_from_output, CPU tensors from a seeded generator: `output` looks like infer()'s batched output
    (points (B, H, W, 3), depth (B, H, W), mask (B, H, W), normal (B, H, W, 3), intrinsics (B, 3, 3)) on synthetic_metrics_case's
    GT scenes (image b from seed + b), with depth and points +inf and normals 0 off the mask as infer(apply_mask=True) leaves
    them; normals are unit length.  `image` is (B, H, W, 3) uint8."""
    out = {k: [] for k in ("points", "depth", "mask", "normal", "intrinsics")}
    images = []
    for b in range(B):
        g = torch.Generator().manual_seed(5000 + seed + b)
        fx, fy, depth, points, mask = _scene(g, H, W)
        normal = torch.nn.functional.normalize(torch.randn(H, W, 3, generator=g) + torch.tensor([0.0, 0.0, -2.0]), dim=-1)
        inf = torch.tensor(float("inf"))
        out["depth"].append(torch.where(mask, depth, inf))
        out["points"].append(torch.where(mask[..., None], points, inf))
        out["normal"].append(torch.where(mask[..., None], normal, torch.zeros(())))
        out["mask"].append(mask)
        out["intrinsics"].append(torch.tensor([[fx, 0, 0.5], [0, fy, 0.5], [0, 0, 1]], dtype=torch.float32))
        images.append(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8))
    return {k: torch.stack(v) for k, v in out.items()}, torch.stack(images)


# ------------------------------------------------------------------------------------------------------------ panorama
PANORAMA_ROOM_LO, PANORAMA_ROOM_HI = (-2.0, -3.0, -1.2), (4.0, 2.5, 1.8)      # box walls around the panorama's centre


def synthetic_panorama(H: int, W: int, seed: int = 0):
    """(H, W, 3) uint8 RGB panorama (numpy): smooth colour, a grid of lines crossing the seam, coloured seam columns, bright / dark
    caps at the poles, seeded noise."""
    import numpy as np
    rs = np.random.RandomState(seed)
    i, j = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    img = np.stack([128 + 100 * np.sin(2 * np.pi * j / W * 3 + c) * np.cos(np.pi * i / H * 2 + c) for c in range(3)], -1)
    img[(j % 17 < 2) | (i % 13 < 2)] = [250, 20, 60]
    img[:, :3] = [0, 255, 0]
    img[:, -3:] = [0, 0, 255]
    img[:max(2, H // 20)] = [230, 230, 230]
    img[-max(2, H // 20):] = [10, 10, 10]
    img = img + rs.randint(-20, 21, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def synthetic_room_views(res: int, seed: int = 7):
    """Distance maps (12, res, res) float32 and masks (12, res, res) bool (numpy) of a box room seen from an off-centre point
    through the 12 panorama cameras: the exact distance along each pixel's ray times (1 + 0.01 noise), three round holes per view
    (radius res / 24 to res / 8) where the mask is off and the distance is tripled.  fp64 elementwise arithmetic, so the same
    seed gives the same bits on any host with the same numpy."""
    import numpy as np
    from .panorama import get_panorama_cameras, uv_map
    extr, intr = get_panorama_cameras()
    lo, hi = np.array(PANORAMA_ROOM_LO), np.array(PANORAMA_ROOM_HI)
    rs = np.random.RandomState(seed)
    uv = uv_map(res, res).astype(np.float64)
    ii, jj = np.meshgrid(np.arange(res), np.arange(res), indexing="ij")
    dist, masks = [], []
    for k in range(len(extr)):
        K, R = intr[k], extr[k, :3, :3].astype(np.float64)
        c = ((uv[..., 0] - K[0, 2]) / K[0, 0], (uv[..., 1] - K[1, 2]) / K[1, 1], np.ones((res, res)))
        d = np.stack([R[0, r] * c[0] + R[1, r] * c[1] + R[2, r] * c[2] for r in range(3)], -1)
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(d > 0, hi / d, np.where(d < 0, lo / d, np.inf)).min(-1)
        dd = t * np.sqrt((d * d).sum(-1)) * (1 + 0.01 * rs.randn(res, res))
        m = np.ones((res, res), bool)
        for _ in range(3):
            ci, cj = rs.randint(0, res, 2)
            r = rs.randint(res // 24, res // 8)
            m &= (ii - ci) ** 2 + (jj - cj) ** 2 > r * r
        dd[~m] *= 3.0
        dist.append(dd.astype(np.float32))
        masks.append(m)
    return np.stack(dist), np.stack(masks)


def synthetic_panorama_scene(H: int, W: int, seed: int = 0):
    """An analytic infer_panorama()-style output for mesh_from_panorama, numpy: the box room of PANORAMA_ROOM_LO / HI seen from its
    origin, with a box standing on the floor in front of a wall (its position from the seed) occluding part of it.  Returns
    points (H, W, 3) float32 = depth * the panorama rays, depth (H, W) float32 (the exact fp64 distance, rounded), mask (H, W)
    bool (off in four seeded round holes and at the pole rows) and image (H, W, 3) uint8 (synthetic_panorama).  The room's
    corners are normal edges, the box's silhouette is a depth and normal edge, and the holes cut the mask."""
    import numpy as np
    from .panorama import spherical_uv_to_directions, uv_map
    rs = np.random.RandomState(seed)
    dirs = spherical_uv_to_directions(uv_map(H, W)).astype(np.float32)
    d = dirs.astype(np.float64)
    lo, hi = np.array(PANORAMA_ROOM_LO), np.array(PANORAMA_ROOM_HI)
    x0, y0 = 1.2 + 0.8 * rs.rand(), -1.5 + 1.5 * rs.rand()
    blo, bhi = np.array([x0, y0, lo[2]]), np.array([x0 + 1.0, y0 + 1.2, lo[2] + 1.1 + 0.4 * rs.rand()])
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(d > 0, hi / d, np.where(d < 0, lo / d, np.inf)).min(-1)
        a, b = blo / d, bhi / d
        near, far = np.minimum(a, b).max(-1), np.maximum(a, b).min(-1)
    hit = (near <= far) & (near > 0)
    t = np.where(hit, np.minimum(t, near), t)
    depth = t.astype(np.float32)
    points = depth[..., None] * dirs
    ii, jj = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    mask = np.ones((H, W), bool)
    for _ in range(4):
        ci, cj, r = rs.randint(0, H), rs.randint(0, W), rs.randint(max(1, H // 40), max(2, H // 12))
        mask &= (ii - ci) ** 2 + (jj - cj) ** 2 > r * r
    mask[:max(1, H // 64)] = False
    mask[-max(1, H // 64):] = False
    return points, depth, mask, synthetic_panorama(H, W, seed)


def array_digest(*arrays) -> str:
    """SHA-256 of the arrays' bytes, in order (C order)."""
    import hashlib
    import numpy as np
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def synthetic_loss_case(seed: int, batch_shape, H: int, W: int, empty_image: bool = False):
    """Inputs of the training losses as a dict of CPU fp32 / bool tensors, from a seeded generator: gt_points (..., H, W, 3) from
    _scene's piecewise-planar depth with +inf where its mask is off (with empty_image, the first image has no valid point at
    all), pred_points = a per-image scale and shift of the GT plus noise, pred_mask (..., H, W) probabilities in (0, 1),
    gt_mask_pos / gt_mask_neg disjoint bool masks, scale_pred / scale_gt (...) (some scale_gt <= 0)."""
    g = torch.Generator().manual_seed(seed)
    n = 1
    for d in batch_shape:
        n *= d
    gts, preds = [], []
    for b in range(n):
        _, _, _, points, mask = _scene(g, H, W)
        if empty_image and b == 0:
            mask[:] = False
        scale = 0.5 + torch.rand((), generator=g).item()
        shift = torch.tensor([0.0, 0.0, 0.5 * (torch.rand((), generator=g).item() - 0.5)])
        preds.append(points / scale + shift + 0.03 * torch.randn(H, W, 3, generator=g))
        gts.append(torch.where(mask[..., None], points, torch.tensor(float("inf"))))
    shape = (*batch_shape, H, W)
    gt_points = torch.stack(gts).reshape(*shape, 3)
    pred_points = torch.stack(preds).reshape(*shape, 3)
    pred_mask = torch.sigmoid(2.0 * torch.randn(shape, generator=g))
    r = torch.rand(shape, generator=g)
    gt_mask_pos, gt_mask_neg = r < 0.5, r > 0.7
    scale_pred = 0.5 + torch.rand(batch_shape, generator=g)
    scale_gt = torch.rand(batch_shape, generator=g) * 2.0 - 0.5
    return {"pred_points": pred_points, "gt_points": gt_points, "pred_mask": pred_mask, "gt_mask_pos": gt_mask_pos,
            "gt_mask_neg": gt_mask_neg, "scale_pred": scale_pred, "scale_gt": scale_gt}


def _unit(v: torch.Tensor) -> torch.Tensor:
    return v / torch.sqrt(v[..., 0:1] * v[..., 0:1] + v[..., 1:2] * v[..., 1:2] + v[..., 2:3] * v[..., 2:3])


def synthetic_normal_map_case(seed: int, batch_shape, H: int, W: int, empty_image: bool = False):
    """Inputs of normal_map_loss as a dict of CPU fp32 tensors, from a seeded generator (elementwise arithmetic only):
    gt_normal (..., H, W, 3) unit normals facing the camera, with about 4 % of pixels invalid (one coordinate NaN, +inf or -inf;
    with empty_image, every pixel of the first image); pred_normal = the GT tilted by noise of a per-pixel size in [0, 0.6) and
    scaled by 0.5 to 2 (non-unit), except about 4 % of pixels that are exactly the GT times 0.5, 1 or 2 (angle 0), 4 % exactly
    its opposite (angle pi) and 5 % in a random direction."""
    g = torch.Generator().manual_seed(seed)
    n = 1
    for d in batch_shape:
        n *= d
    gt = _unit(torch.randn(n, H, W, 3, generator=g) + torch.tensor([0.0, 0.0, 1.5]))
    tilt = 0.6 * torch.rand(n, H, W, 1, generator=g) * torch.randn(n, H, W, 3, generator=g)
    pred = (gt + tilt) * (0.5 + 1.5 * torch.rand(n, H, W, 1, generator=g))
    r = torch.rand(n, H, W, 1, generator=g)
    exact = gt * (2.0 ** torch.randint(-1, 2, (n, H, W, 1), generator=g).float())
    pred = torch.where(r < 0.04, exact, torch.where(r < 0.08, -exact, pred))
    pred = torch.where((r >= 0.08) & (r < 0.13), torch.randn(n, H, W, 3, generator=g), pred)
    bad = torch.rand(n, H, W, generator=g) < 0.04
    if empty_image:
        bad[0] = True
    coord = torch.randint(0, 3, (n, H, W, 1), generator=g)
    value = torch.tensor([float("nan"), float("inf"), -float("inf")])[torch.randint(0, 3, (n, H, W, 1), generator=g)]
    gt = torch.where(bad[..., None] & (torch.arange(3) == coord), value, gt)
    shape = (*batch_shape, H, W, 3)
    return {"pred_normal": pred.reshape(shape).contiguous(), "gt_normal": gt.reshape(shape).contiguous()}


def synthetic_geometry_case(seed: int, batch_shape, H: int, W: int, mask_mode: str = "sparse"):
    """Inputs of the geometry utilities (moge_b200.geometry) as a dict of CPU fp32 / bool tensors, from a seeded generator
    (arithmetic and sqrt only): depth (..., H, W) > 0, the piecewise-planar depth of _scene; normal (..., H, W, 3), unit normals
    of its points by central differences (one-sided at the border), turned to face the camera and tilted by noise of 0.05;
    intrinsics (..., 3, 3), normalised, with the principal point within 0.02 of the centre; mask (..., H, W): 'all', 'none',
    'sparse' (about 30 % valid) or 'scene' (_scene's mask); image (prod(batch_shape), 3, H, W) in [0, 1)."""
    g = torch.Generator().manual_seed(4000 + seed)
    n = 1
    for d in batch_shape:
        n *= d
    depths, normals, intrs, masks = [], [], [], []
    for _ in range(n):
        fx, fy, depth, points, scene_mask = _scene(g, H, W)
        cx, cy = (0.5 + 0.04 * (torch.rand(2, generator=g) - 0.5)).tolist()
        K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)
        jr, jl = torch.arange(W).add(1).clamp_max(W - 1), torch.arange(W).sub(1).clamp_min(0)
        ib, it = torch.arange(H).add(1).clamp_max(H - 1), torch.arange(H).sub(1).clamp_min(0)
        du, dv = points[:, jr] - points[:, jl], points[ib] - points[it]
        nx = du[..., 1] * dv[..., 2] - du[..., 2] * dv[..., 1]
        ny = du[..., 2] * dv[..., 0] - du[..., 0] * dv[..., 2]
        nz = du[..., 0] * dv[..., 1] - du[..., 1] * dv[..., 0]
        nrm = torch.stack([nx, ny, nz], dim=-1)
        nrm = torch.where(nz[..., None] > 0, -nrm, nrm)
        nrm = _unit(_unit(nrm) + 0.05 * torch.randn(H, W, 3, generator=g))
        if mask_mode == "all":
            mask = torch.ones(H, W, dtype=torch.bool)
        elif mask_mode == "none":
            mask = torch.zeros(H, W, dtype=torch.bool)
        elif mask_mode == "sparse":
            mask = torch.rand(H, W, generator=g) < 0.3
        elif mask_mode == "scene":
            mask = scene_mask
        else:
            raise ValueError(mask_mode)
        depths.append(depth); normals.append(nrm); intrs.append(K); masks.append(mask)
    image = torch.rand(n, 3, H, W, generator=g)
    shape = (*batch_shape, H, W)
    return {"depth": torch.stack(depths).reshape(shape), "normal": torch.stack(normals).reshape(*shape, 3).contiguous(),
            "intrinsics": torch.stack(intrs).reshape(*batch_shape, 3, 3), "mask": torch.stack(masks).reshape(shape), "image": image}


def make_dinov2_state_dict(size: str = "vits", seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded fp32 state dict of a DINOv2 ViT-S/B/L/14 backbone under its own keys (moge/model/dinov2): the `encoder.backbone.*`
    tensors of the synthetic MoGe-2 state dict of the same size and seed, with the prefix dropped."""
    from .configs import model_config
    p = "encoder.backbone."
    return OrderedDict((k[len(p):], v) for k, v in make_state_dict(model_config(size), seed).items() if k.startswith(p))


def synthetic_dino_input(batch: int, height: int, width: int, seed: int = 0) -> torch.Tensor:
    """(B, 3, H, W) fp32: a normalised image as the DINOv2 backbone takes it (ImageNet mean / std applied), seeded."""
    mean = torch.tensor(IMAGE_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(IMAGE_STD).view(1, 3, 1, 1)
    return (synthetic_images(batch, height, width, seed) - mean) / std
