"""The sampled local loss of the reference's `moge/train/losses.py` on the GPU: `affine_invariant_local_loss` and
`compute_anchor_sampling_weight`, with the reference's signatures, defaults and return conventions (a loss tensor of the batch
shape and a `misc` dict of Python floats, or the scalar `(0.0, {})` when no patch is kept).  The other training losses are in
moge_b200.losses.

Both functions make the reference's three random calls, with its arguments and in its order, on the default generator of the
tensors' device: `torch.randint` twice for the (H, W, 64) test offsets and one `torch.multinomial` over the batch's valid
pixels for the anchors.  So from one seed they use the reference's offsets and leave the generator where the reference does,
and they pick the reference's anchors wherever the sampling weights are bitwise equal.  The two int64 offset tensors (1 KiB per
pixel) are the only large tensors allocated besides the u8 patch masks; the per-pixel tests, the patch masks, the loss and its
gradient run in the kernels of moge_b200/csrc/losses.cu without gathering patch copies of the point maps.  A call waits for the
host three times: the valid-pixel compaction for `multinomial`, the selection of the patches with at least 32 points, and the
one copy of the misc values.  A batch's anchors come from one `multinomial` over all of its images, as in the reference, so an
image does not give the same loss alone and inside a batch.  Given the anchors, losses, misc values and gradients are bitwise
reproducible (fp64 sums over fixed tiles, one writer per gradient element, no float atomics); `torch.multinomial` on CUDA
itself may pick a few anchors differently from run to run over large inputs.

Inputs must be CUDA tensors (there is no CPU fallback).  Arithmetic is fp32; fp16 and bf16 predictions are accepted, losses are
returned in fp32 and gradients come back in the prediction's dtype.

Divergences from the reference:
  - sums are accumulated in fp64 (the reference sums fp32), so losses agree to ~1e-6 relative rather than bit for bit;
  - positions outside a patch's mask are skipped where the reference multiplies them by a 0 weight (a non-finite prediction
    there gives NaN in the reference);
  - the kernels' fp32 |d| may differ from torch's `norm` by an ulp, so a test or patch point whose distance lies within an ulp
    of the radius may be counted the other way;
  - for a batch of more than one image it follows the evident intent of the reference's code, which raises there: each image's
    focal scales its own radii, and `global_scale > 0` is tested on the patch's own image.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import alignment as A
from . import capi
from .capi import MogeError
from .losses import point_maps, sum_buffer
from .metrics import masked_nearest_resize

__all__ = ["compute_anchor_sampling_weight", "affine_invariant_local_loss"]

MINIMUM_POINTS_PER_PATCH = 32


def _anchor_weight(points: torch.Tensor, mask: torch.Tensor, radius_2d: int, radius_3d: torch.Tensor, num_test: int, draws=None):
    """compute_anchor_sampling_weight on (B, H, W, 3) fp32 points, (B, H, W) bool mask and (B, H, W) radius_3d.  draws: the two
    (H, W, num_test) int64 offset tensors, or None to draw them as the reference does."""
    B, H, W, _ = points.shape
    dev = points.device
    if draws is None:
        di = torch.randint(-radius_2d, radius_2d + 1, (H, W, num_test), device=dev)
        dj = torch.randint(-radius_2d, radius_2d + 1, (H, W, num_test), device=dev)
    else:
        di, dj = (d.to(device=dev, dtype=torch.int64).contiguous() for d in draws)
    weight = torch.empty(B, H, W, dtype=torch.float32, device=dev)
    m = capi.mask_u8(mask)
    capi.check(capi.lib().moge_loss_anchor_weight(points.data_ptr(), m.data_ptr(), di.data_ptr(), dj.data_ptr(), radius_3d.data_ptr(),
                                                  B, H, W, num_test, weight.data_ptr(), capi.current_stream()))
    return weight / weight.sum(dim=(-2, -1), keepdim=True).add(1e-7), (di, dj)


def compute_anchor_sampling_weight(points: torch.Tensor, mask: torch.Tensor, radius_2d: int, radius_3d: torch.Tensor,
                                   num_test: int = 64) -> torch.Tensor:
    """Per pixel of points (..., H, W, 3) with mask (..., H, W): 1 / the number of its num_test random neighbours (offsets drawn
    in [-radius_2d, radius_2d] by two torch.randint calls, as in the reference) that are inside the map, valid and within
    radius_3d (..., H, W) of it; 0 off the mask; normalised to sum 1 per image.  Returns (..., H, W) fp32."""
    capi.require_cuda("moge_b200.local_loss", points, mask, radius_3d)
    *batch_shape, H, W, _ = points.shape
    p = points.detach().to(torch.float32).reshape(-1, H, W, 3).contiguous()
    m = mask.to(torch.bool).expand(*batch_shape, H, W).reshape(-1, H, W)
    r = radius_3d.detach().to(torch.float32).expand(*batch_shape, H, W).reshape(-1, H, W).contiguous()
    return _anchor_weight(p, m, int(radius_2d), r, int(num_test))[0].reshape(*batch_shape, H, W)


class _LocalLoss(torch.autograd.Function):
    """Per kept patch, the sum over its marked positions and xyz of smooth(|scale p + shift - g| w) (fp64, differentiable in pred,
    scale and shift) and (not differentiable) the sums (position count, sum of min(err, 1), count of err < 1)."""

    @staticmethod
    def forward(ctx, pred, scale, shift, gt, anchor, params, pmask, beta, r):
        B, H, W, _ = pred.shape
        P, S = anchor.shape[0], 2 * r + 1
        params = params.clone()
        params[:, 0], params[:, 1:4] = scale.detach(), shift.detach()
        sums, ws = sum_buffer(P, pred.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, P, S, S, device=pred.device)
        capi.check(capi.lib().moge_loss_local(pred.data_ptr(), gt.data_ptr(), anchor.data_ptr(), params.data_ptr(), pmask.data_ptr(),
                                              beta, 1, B, H, W, P, r, None, sums.data_ptr(), ws.data_ptr(), ws.numel(),
                                              capi.current_stream()))
        ctx.save_for_backward(pred, gt, anchor, params, pmask)
        ctx.beta, ctx.r = beta, r
        misc = sums[:, 1:4].clone()
        ctx.mark_non_differentiable(misc)
        return sums[:, 0].clone(), misc

    @staticmethod
    def backward(ctx, g, _):
        pred, gt, anchor, params, pmask = ctx.saved_tensors
        B, H, W, _ = pred.shape
        P, r = anchor.shape[0], ctx.r
        S = 2 * r + 1
        params = params.clone()
        params[:, 7] = g.to(torch.float32)
        grad = torch.empty_like(pred)
        sums, ws = sum_buffer(P, pred.device), capi.workspace(capi.lib().moge_loss_workspace_bytes, P, S, S, device=pred.device)
        capi.check(capi.lib().moge_loss_local(pred.data_ptr(), gt.data_ptr(), anchor.data_ptr(), params.data_ptr(), pmask.data_ptr(),
                                              ctx.beta, 2, B, H, W, P, r, grad.data_ptr(), sums.data_ptr(), ws.data_ptr(), ws.numel(),
                                              capi.current_stream()))
        return grad, sums[:, 0].to(torch.float32), sums[:, 1:4].to(torch.float32), None, None, None, None, None, None


def _local_loss(pred_points, gt_points, focal, global_scale, level, align_resolution=32, num_patches=16, beta=0.0, trunc=1.0,
                sparsity_aware=False, draws=None):
    """affine_invariant_local_loss; returns (loss, misc, info).  draws: None to draw as the reference does, or a dict with the
    offsets "delta_i", "delta_j" (H, W, 64) and the multinomial's "selection" (num_patches B).  info holds the draws, the kept
    patches' indices into the selection, their anchors (image, i, j), and the alignment's scale and shift before the validity
    test (None where no patch is kept)."""
    batch_shape, H, W, pred, gt = point_maps(pred_points, gt_points)
    capi.require_cuda("moge_b200.local_loss", focal, global_scale)
    if not beta >= 0.0:
        raise MogeError(f"beta must be >= 0 (got {beta})")
    B, dev = pred.shape[0], pred.device
    gt_mask = torch.isfinite(gt).all(dim=-1)
    gt_filled = torch.where(gt_mask[..., None], gt, 1)
    focal = focal.detach().to(torch.float32).reshape(-1).contiguous()
    if global_scale is not None:
        global_scale = global_scale.detach().reshape(-1)

    # anchors: the reference's three draws (two randint, one multinomial over the valid pixels of the batch)
    radius_2d = math.ceil(0.5 / level * (H ** 2 + W ** 2) ** 0.5)
    radius_3d = (0.5 / level / focal)[:, None, None] * gt_filled[..., 2]
    weights, (di, dj) = _anchor_weight(gt_filled, gt_mask, radius_2d, radius_3d.contiguous(), 64,
                                       None if draws is None else (draws["delta_i"], draws["delta_j"]))
    where_mask = torch.where(gt_mask)                                                   # host wait 1
    if draws is None:
        selection = torch.multinomial(weights[where_mask], num_patches * B, replacement=True)
    else:
        selection = draws["selection"].to(dev)
    anchor = torch.stack([idx[selection] for idx in where_mask], dim=-1).contiguous()   # (P, 3): image, i, j
    info = {"delta_i": di, "delta_j": dj, "selection": selection, "kept": None, "anchor": None, "scale": None, "shift": None}

    # patch masks, kept patches
    P, r = anchor.shape[0], radius_2d
    S = 2 * r + 1
    pmask = torch.empty(P, S, S, dtype=torch.bool, device=dev)
    count = torch.empty(P, dtype=torch.int32, device=dev)
    radius = torch.empty(P, dtype=torch.float32, device=dev)
    capi.check(capi.lib().moge_loss_patch_mask(gt.data_ptr(), capi.mask_u8(gt_mask).data_ptr(), anchor.data_ptr(),
                                               focal.data_ptr(), 0.5 / level, B, H, W, P, r, pmask.data_ptr(), count.data_ptr(),
                                               radius.data_ptr(), capi.current_stream()))
    kept = torch.where(count >= MINIMUM_POINTS_PER_PATCH)[0]                           # host wait 2
    if kept.numel() == 0:
        return torch.tensor(0.0, dtype=torch.float32, device=dev), {}, info
    anchor, pmask, radius = anchor[kept].contiguous(), pmask[kept].contiguous(), radius[kept]
    P, img = anchor.shape[0], anchor[:, 0]
    info["kept"], info["anchor"] = kept, anchor

    # alignment on the masked nearest resize of each patch, gathered from the full maps through the patch's offset
    lr_mask, (_, i, j) = masked_nearest_resize(mask=pmask, size=(align_resolution, align_resolution), return_index=True)
    lr_i = (anchor[:, 1, None, None] - r + i).clamp(0, H - 1)
    lr_j = (anchor[:, 2, None, None] - r + j).clamp(0, W - 1)
    pred_lr, gt_lr = pred[img[:, None, None], lr_i, lr_j], gt_filled[img[:, None, None], lr_i, lr_j]
    local_scale, local_shift = A.align_points_scale_xyz_shift(pred_lr.flatten(-3, -2), gt_lr.flatten(-3, -2),
                                                              lr_mask.flatten(-2) / radius[:, None].add(1e-7), trunc=trunc)
    info["scale"], info["shift"] = local_scale.detach(), local_shift.detach()
    if global_scale is not None:
        scale_differ = local_scale / global_scale[img]
        patch_valid = (scale_differ > 0.1) & (scale_differ < 10.0) & (global_scale[img] > 0)
    else:
        patch_valid = local_scale > 0
    local_scale, local_shift = torch.where(patch_valid, local_scale, 0), torch.where(patch_valid[:, None], local_shift, 0)

    # the harmonic mean of the GT depth per image, for the weights' floor
    hsums, ws = sum_buffer(B, dev), capi.workspace(capi.lib().moge_loss_workspace_bytes, B, H, W, device=dev)
    capi.check(capi.lib().moge_loss_local(None, gt.data_ptr(), None, None, None, float(beta), 0, B, H, W, 0, 0, None, hsums.data_ptr(),
                                          ws.data_ptr(), ws.numel(), capi.current_stream()))
    hw = H * W
    gt_mean = ((hsums[:, 0] / hw) / (hsums[:, 1] / hw + 1e-7) + 1e-7).reciprocal().to(torch.float32)

    params = torch.zeros(P, capi.LOSS_LOCAL_PARAMS, dtype=torch.float32, device=dev)
    params[:, 4], params[:, 5], params[:, 6] = patch_valid.to(torch.float32), 0.1 * gt_mean[img], radius
    sums, misc_sums = _LocalLoss.apply(pred, local_scale, local_shift, gt, anchor, params, pmask, float(beta), r)
    loss = sums / (3 * S * S)
    if sparsity_aware:
        sparsity = (misc_sums[:, 0] / (S * S)) / lr_mask.to(torch.float64).mean(dim=(-2, -1))
        loss = loss / (sparsity + 1e-7)
    # per image, a fixed-order fp64 sum over its patches
    onehot = img[None, :] == torch.arange(B, device=dev)[:, None]
    loss = (torch.where(onehot, loss[None, :], 0).sum(dim=-1) / num_patches).to(torch.float32).reshape(batch_shape)

    n = P * S * S
    count = misc_sums[:, 0].sum() / n
    misc_t = torch.stack([(misc_sums[:, 1].sum() / n) / (count + 1e-7), (misc_sums[:, 2].sum() / n) / (count + 1e-7)])
    te, delta = misc_t.to(torch.float32).cpu().tolist()                                 # host wait 3
    return loss, {"truncated_error": te, "delta": delta}, info


def affine_invariant_local_loss(pred_points: torch.Tensor, gt_points: torch.Tensor, focal: torch.Tensor,
                                global_scale: Optional[torch.Tensor], level: int, align_resolution: int = 32, num_patches: int = 16,
                                beta: float = 0.0, trunc: float = 1.0, sparsity_aware: bool = False):
    """The reference's sampled local loss.  Per image of pred_points (..., H, W, 3) against gt_points (inf / NaN = invalid) with
    focal (...): num_patches anchors per image drawn from compute_anchor_sampling_weight's weights by one torch.multinomial over
    the batch (the reference's draws, on the default generator of the tensors' device), patches of radius
    ceil(0.5 / level * diagonal) pixels holding the GT points within 0.5 / level / focal * anchor z of the anchor, those with at
    least 32 points kept; each kept patch is aligned (scale and xyz shift, truncated L1 on its align_resolution^2 masked nearest
    resize), rejected unless its scale is within (0.1, 10) times global_scale (...) (or positive when global_scale is None), and
    contributes the mean of smooth(|aligned - gt| / max(gt z, 0.1 harmonic-mean GT z)) over its (2r+1)^2 positions and xyz.
    Returns (loss (...), misc {'truncated_error', 'delta'}), or (0.0, {}) when no patch is kept."""
    loss, misc, _ = _local_loss(pred_points, gt_points, focal, global_scale, level, align_resolution, num_patches, beta, trunc,
                                sparsity_aware)
    return loss, misc
