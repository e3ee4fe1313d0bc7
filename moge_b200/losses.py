"""Training losses on the GPU: the deterministic losses of the reference's `moge/train/losses.py` (`affine_invariant_global_loss`,
`normal_loss`, `edge_loss`, `normal_map_loss`, `mask_l2_loss`, `mask_bce_loss`, `metric_scale_loss`, `monitoring`) with the
reference's signatures, defaults, batch semantics and return conventions (loss tensors of the batch shape, or a scalar for
`normal_loss`; `misc` dicts of Python floats under the reference's keys).  The sampled local loss
(`affine_invariant_local_loss`, `compute_anchor_sampling_weight`) is in moge_b200.local_loss.  `moge.train.losses` re-exports
both modules as a drop-in for the reference's module.  `__all__` keeps the names of this module's first release, so a star
import of it brings in what it always did; `normal_map_loss` is imported by name.

The per-pixel work runs in the kernels of moge_b200/csrc/losses.cu, forward and backward, behind one `torch.autograd.Function`
per loss: per-image sums are fp64 over fixed pixel tiles added in a fixed order, and each pixel's gradient is written by one
thread, so losses, misc values and gradients are bitwise reproducible and an image gives the same loss alone or inside a batch.
`affine_invariant_global_loss` aligns with moge_b200.metrics.masked_nearest_resize and
moge_b200.alignment.align_points_scale_z_shift; its kernel's backward returns dL/dpred (the direct term) together with dL/dscale
and dL/dshift, and autograd chains those through the alignment's gathers as it does in the reference.  The only device-to-host
copy is the single copy of the global loss's two misc values.  `metric_scale_loss` (B scalars) and `monitoring` (one `std`) are
the reference's torch expressions: there is nothing to fuse.

Inputs must be CUDA tensors (there is no CPU fallback).  Arithmetic is fp32; fp16 and bf16 predictions are accepted, losses are
returned in fp32 and gradients come back in the prediction's dtype.

Divergences from the reference:
  - sums are accumulated in fp64 (the reference sums fp32), so losses agree to ~1e-6 relative rather than bit for bit;
  - pixels with invalid GT are skipped in the global loss's misc sums, where the reference multiplies them by a 0 mask: a
    non-finite prediction at such a pixel gives NaN misc values in the reference and finite ones here (the loss terms
    themselves are multiplied by their masks, as in the reference);
  - the alignment may resolve a near-tie of its objective (within 1e-6) with another solution than the reference's solver
    (moge_b200.alignment), so scale and shift agree with the reference to 1e-5 relative rather than bit for bit;
  - an fp16 / bf16 prediction is upcast before any arithmetic, where the reference computes in the promoted dtypes of its
    operands: `normal_map_loss` normalises an fp16 prediction in fp16 there, and agrees with it to ~1e-4 relative.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from . import alignment as A
from . import capi
from .capi import MogeError
from .metrics import masked_nearest_resize

__all__ = [
    "affine_invariant_global_loss", "monitoring", "normal_loss", "edge_loss", "mask_l2_loss", "mask_bce_loss", "metric_scale_loss",
]


def sum_buffer(B: int, device) -> torch.Tensor:
    """An uninitialised (B, LOSS_SUMS) fp64 buffer for a loss kernel's per-image (or per-patch) sums."""
    return torch.empty(B, capi.LOSS_SUMS, dtype=torch.float64, device=device)


# ------------------------------------------------------------------------------------------------------------ mask losses
class _MaskLoss(torch.autograd.Function):
    """Per-image mean over (H, W) of a mask loss term of x (B, H, W) fp32 with factors a, b (see moge_loss_mask)."""

    @staticmethod
    def forward(ctx, x, a, b, kind):
        B, H, W = x.shape
        sums, ws = sum_buffer(B, x.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=x.device)
        capi.check(capi.lib().moge_loss_mask(kind, x.data_ptr(), a.data_ptr(), b.data_ptr(), B, H, W, None, None, sums.data_ptr(),
                                             ws.data_ptr(), ws.numel(), capi.current_stream()))
        ctx.save_for_backward(x, a, b)
        ctx.kind = kind
        return (sums[:, 0] / (H * W)).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        x, a, b = ctx.saved_tensors
        B, H, W = x.shape
        coef = (g.to(torch.float32) / (H * W)).contiguous()
        grad = torch.empty_like(x)
        capi.check(capi.lib().moge_loss_mask(ctx.kind, x.data_ptr(), a.data_ptr(), b.data_ptr(), B, H, W, coef.data_ptr(),
                                             grad.data_ptr(), None, None, 0, capi.current_stream()))
        return grad, None, None, None


def _mask_loss(kind: int, pred: torch.Tensor, a: torch.Tensor, b: torch.Tensor):
    capi.require_cuda("moge_b200.losses", pred, a, b)
    *batch_shape, H, W = pred.shape
    flat = (-1, H, W)
    x = pred.to(torch.float32).reshape(flat).contiguous()
    a = a.detach().to(torch.float32).expand(pred.shape).reshape(flat).contiguous()
    b = b.detach().to(torch.float32).expand(pred.shape).reshape(flat).contiguous()
    return _MaskLoss.apply(x, a, b, kind).reshape(batch_shape), {}


def mask_l2_loss(pred_mask: torch.Tensor, gt_mask_pos: torch.Tensor, gt_mask_neg: torch.Tensor):
    """Mean over (H, W) of gt_mask_neg * pred_mask^2 + gt_mask_pos * (1 - pred_mask)^2; returns (loss (...), {})."""
    return _mask_loss(capi.LOSS_MASK_L2, pred_mask, gt_mask_neg, gt_mask_pos)


def mask_bce_loss(pred_mask_prob: torch.Tensor, gt_mask_pos: torch.Tensor, gt_mask_neg: torch.Tensor):
    """Mean over (H, W) of (gt_mask_pos | gt_mask_neg) * binary_cross_entropy(pred_mask_prob, gt_mask_pos), with torch's -100 log
    clamp; returns (loss (...), {})."""
    capi.require_cuda("moge_b200.losses", gt_mask_pos, gt_mask_neg)
    return _mask_loss(capi.LOSS_MASK_BCE, pred_mask_prob, gt_mask_pos | gt_mask_neg, gt_mask_pos)


# ------------------------------------------------------------------------------------------------------------ stencil losses
class _StencilLoss(torch.autograd.Function):
    """EDGE: per image (mean angle term of the vertical pairs, of the horizontal pairs) (B, 2); NORMAL: the mean quad term over
    the whole batch (a scalar)."""

    @staticmethod
    def forward(ctx, points, gt, kind):
        B, H, W, _ = points.shape
        sums, ws = sum_buffer(B, points.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=points.device)
        capi.check(capi.lib().moge_loss_stencil(kind, points.data_ptr(), gt.data_ptr(), B, H, W, None, None, sums.data_ptr(),
                                                ws.data_ptr(), ws.numel(), capi.current_stream()))
        ctx.save_for_backward(points, gt)
        ctx.kind = kind
        if kind == capi.LOSS_EDGE:
            return torch.stack([sums[:, 0] / ((H - 1) * W), sums[:, 1] / (H * (W - 1))], dim=-1).to(torch.float32)
        return (sums[:, 0].sum() / (B * (H - 1) * (W - 1))).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        points, gt = ctx.saved_tensors
        B, H, W, _ = points.shape
        g = g.to(torch.float32)
        if ctx.kind == capi.LOSS_EDGE:
            coef = torch.stack([g[:, 0] / ((H - 1) * W), g[:, 1] / (H * (W - 1))], dim=-1)
        else:
            coef = (g / (B * (H - 1) * (W - 1))).expand(B, 2)
        coef = coef.contiguous()
        grad = torch.empty_like(points)
        capi.check(capi.lib().moge_loss_stencil(ctx.kind, points.data_ptr(), gt.data_ptr(), B, H, W, coef.data_ptr(), grad.data_ptr(),
                                                None, None, 0, capi.current_stream()))
        return grad, None, None


def point_maps(points: torch.Tensor, gt_points: torch.Tensor, what: str = "point maps"):
    """Check a prediction and its GT (..., H, W, 3) and flatten them: (batch shape, H, W, prediction, detached GT), both
    (B, H, W, 3) contiguous fp32."""
    capi.require_cuda("moge_b200.losses", points, gt_points)
    if points.shape != gt_points.shape or points.dim() < 3 or points.shape[-1] != 3:
        raise MogeError(f"{what} must be (..., H, W, 3) of one shape, got {tuple(points.shape)} and {tuple(gt_points.shape)}")
    *batch_shape, H, W, _ = points.shape
    p = points.to(torch.float32).reshape(-1, H, W, 3).contiguous()
    g = gt_points.detach().to(torch.float32).reshape(-1, H, W, 3).contiguous()
    return batch_shape, H, W, p, g


def normal_loss(points: torch.Tensor, gt_points: torch.Tensor):
    """The angle between each of the four triangle normals of every quad and its GT normal (clamped to [1, 90] degrees, smoothed
    below 3 degrees), where its three GT corners are valid, averaged over the batch and divided by 4 max(H, W).  Returns
    (loss (), {})."""
    _, H, W, p, g = point_maps(points, gt_points)
    return _StencilLoss.apply(p, g, capi.LOSS_NORMAL) / (4 * max(H, W)), {}


def edge_loss(points: torch.Tensor, gt_points: torch.Tensor):
    """The angle between each vertical and horizontal neighbour difference and its GT difference (clamped to [0.1, 90] degrees,
    smoothed below 3 degrees), where both GT points are valid: per image, (mean over vertical pairs + mean over horizontal pairs)
    / (2 max(H, W)).  Returns (loss (...), {})."""
    batch_shape, H, W, p, g = point_maps(points, gt_points)
    means = _StencilLoss.apply(p, g, capi.LOSS_EDGE)
    return ((means[:, 0] + means[:, 1]) / (2 * max(H, W))).reshape(batch_shape), {}


# ------------------------------------------------------------------------------------------------------------ normal map loss
class _NormalMapLoss(torch.autograd.Function):
    """Per image, the mean over (H, W) of mask * angle_between(pred, gt)^2 (see moge_loss_normal_map)."""

    @staticmethod
    def forward(ctx, pred, gt):
        B, H, W, _ = pred.shape
        sums, ws = sum_buffer(B, pred.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=pred.device)
        capi.check(capi.lib().moge_loss_normal_map(pred.data_ptr(), gt.data_ptr(), B, H, W, None, None, sums.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), capi.current_stream()))
        ctx.save_for_backward(pred, gt)
        return (sums[:, 0] / (H * W)).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        pred, gt = ctx.saved_tensors
        B, H, W, _ = pred.shape
        coef = (g.to(torch.float32) / (H * W)).contiguous()
        grad = torch.empty_like(pred)
        capi.check(capi.lib().moge_loss_normal_map(pred.data_ptr(), gt.data_ptr(), B, H, W, coef.data_ptr(), grad.data_ptr(), None,
                                                   None, 0, capi.current_stream()))
        return grad, None


def normal_map_loss(pred_normal: torch.Tensor, gt_normal: torch.Tensor):
    """Per image, the mean over (H, W) of mask * angle_between(pred_normal, gt_normal)^2, where mask marks the GT normals with
    three finite coordinates (the others read as (1, 1, 1)) and angle_between(a, b) = 2 atan2(|a^ - b^|, |a^ + b^|), v^ = v / |v|
    (utils3d's half-angle form).  The mask multiplies: a zero or non-finite prediction gives NaN even at an invalid pixel, as in
    the reference.  Returns (loss (...), {})."""
    batch_shape, _, _, p, g = point_maps(pred_normal, gt_normal, "normal maps")
    return _NormalMapLoss.apply(p, g).reshape(batch_shape), {}


# ------------------------------------------------------------------------------------------------------------ global loss
class _GlobalLoss(torch.autograd.Function):
    """Per image, the mean over (H, W, 3) of smooth(|scale p + shift - g| min(w, cap)), and (not differentiable) the misc sums
    (sum of min(err, 1), count of err < 1) over the mask."""

    @staticmethod
    def forward(ctx, pred, scale, shift, gt, fixed, beta):
        B, H, W, _ = pred.shape
        params = torch.cat([scale.detach()[:, None], shift.detach(), fixed, torch.zeros_like(fixed)], dim=-1).contiguous()
        sums, ws = sum_buffer(B, pred.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=pred.device)
        capi.check(capi.lib().moge_loss_global(pred.data_ptr(), gt.data_ptr(), params.data_ptr(), beta, 1, B, H, W, None, sums.data_ptr(),
                                               ws.data_ptr(), ws.numel(), capi.current_stream()))
        ctx.save_for_backward(pred, gt, params)
        ctx.beta = beta
        misc = sums[:, 1:3].clone()
        ctx.mark_non_differentiable(misc)
        return (sums[:, 0] / (3 * H * W)).to(torch.float32), misc

    @staticmethod
    def backward(ctx, g, _):
        pred, gt, params = ctx.saved_tensors
        B, H, W, _ = pred.shape
        params = params.clone()
        params[:, 6] = g.to(torch.float32) / (3 * H * W)
        grad = torch.empty_like(pred)
        sums, ws = sum_buffer(B, pred.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=pred.device)
        capi.check(capi.lib().moge_loss_global(pred.data_ptr(), gt.data_ptr(), params.data_ptr(), ctx.beta, 2, B, H, W, grad.data_ptr(),
                                               sums.data_ptr(), ws.data_ptr(), ws.numel(), capi.current_stream()))
        return grad, sums[:, 0].to(torch.float32), sums[:, 1:4].to(torch.float32), None, None, None


def affine_invariant_global_loss(pred_points: torch.Tensor, gt_points: torch.Tensor, align_resolution: int = 64, beta: float = 0.0,
                                 trunc: float = 1.0, sparsity_aware: bool = False):
    """Per-image truncated-L1 scale / z-shift alignment of pred_points (..., H, W, 3) to gt_points (inf / NaN = invalid) on the
    align_resolution^2 masked nearest resize, then the weighted L1 of the aligned points.  Returns (loss (...), misc
    {'truncated_error', 'delta'}, scale (...) detached)."""
    batch_shape, H, W, pred, gt = point_maps(pred_points, gt_points)
    if not beta >= 0.0:
        raise MogeError(f"beta must be >= 0 (got {beta})")
    B, dev = pred.shape[0], pred.device
    mask = torch.isfinite(gt).all(dim=-1)
    gt_filled = torch.where(mask[..., None], gt, 1)
    pred_lr, gt_lr, lr_mask = masked_nearest_resize(pred, gt_filled, mask=mask, size=(align_resolution, align_resolution))
    scale, shift = A.align_points_scale_z_shift(pred_lr.flatten(-3, -2), gt_lr.flatten(-3, -2),
                                                lr_mask.flatten(-2, -1) / gt_lr[..., 2].flatten(-2, -1).clamp_min(1e-2), trunc=trunc)
    valid = scale > 0
    scale, shift = torch.where(valid, scale, 0), torch.where(valid[..., None], shift, 0)

    # pass 0: the per-image weighted mean of the weights, for the clamp_max
    params = torch.zeros(B, 8, dtype=torch.float32, device=dev)
    params[:, 4] = valid.to(torch.float32)
    sums, ws = sum_buffer(B, dev), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=dev)
    capi.check(capi.lib().moge_loss_global(pred.data_ptr(), gt.data_ptr(), params.data_ptr(), float(beta), 0, B, H, W, None,
                                           sums.data_ptr(), ws.data_ptr(), ws.numel(), capi.current_stream()))
    hw = H * W
    wmean = ((sums[:, 0] / hw) / (sums[:, 1] / hw + 1e-7)).to(torch.float32)
    fixed = torch.stack([valid.to(torch.float32), 10.0 * wmean], dim=-1)

    loss, misc_sums = _GlobalLoss.apply(pred, scale, shift, gt, fixed, float(beta))
    if sparsity_aware:
        sparsity = (sums[:, 1] / hw).to(torch.float32) / lr_mask.float().mean(dim=(-2, -1))
        loss = loss / (sparsity + 1e-7)

    n = B * hw
    count = sums[:, 1].sum() / n
    misc_t = torch.stack([(misc_sums[:, 0].sum() / n) / (count + 1e-7), (misc_sums[:, 1].sum() / n) / (count + 1e-7)])
    te, delta = misc_t.to(torch.float32).cpu().tolist()
    return loss.reshape(batch_shape), {"truncated_error": te, "delta": delta}, scale.detach().reshape(batch_shape)


# ------------------------------------------------------------------------------------------------------------ torch expressions
def monitoring(points: torch.Tensor) -> Dict[str, float]:
    capi.require_cuda("moge_b200.losses", points)
    return {"std": points.std().item()}


def metric_scale_loss(scale_pred: torch.Tensor, scale_gt: torch.Tensor) -> Tuple[torch.Tensor, Dict]:
    capi.require_cuda("moge_b200.losses", scale_pred, scale_gt)
    valid = scale_gt > 0
    return torch.where(valid, F.mse_loss(scale_pred.log(), torch.where(valid, scale_gt.log(), 0), reduction="none"), 0), {}
