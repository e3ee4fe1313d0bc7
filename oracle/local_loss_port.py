"""A plain-torch restatement of the reference's sampled local loss (`compute_anchor_sampling_weight` and
`affine_invariant_local_loss` of `moge/train/losses.py`).  TEST INFRASTRUCTURE ONLY: the host-side checker of
tests/golden/local_loss.pt and of moge_b200.local_loss.

The local loss takes its random draws as an optional `draws` dict ("delta_i", "delta_j": the two randint offset tensors,
"selection": the multinomial's result); without it, it makes the reference's three calls.  It also takes
`align(pred_lr, gt_lr, weight, trunc) -> (scale, shift)`: the reference's `align_points_scale_xyz_shift`, the engine's, or
recorded values.  Its batch semantics are the evident intent of the reference's code, which raises for more than one image:
each image's focal scales its own radii, and `global_scale > 0` is tested per patch on its image's scale.  For one image the
two are the same expressions.  `masked_nearest_resize` is the utils3d stand-in of oracle/utils3d_metrics.py.
"""
import math

import torch

from oracle.losses_port import smooth, weighted_mean
from oracle.utils3d_metrics import masked_nearest_resize


def harmonic_mean(x, w, dim, eps=1e-7):
    return weighted_mean(x.add(eps).reciprocal(), w, dim=dim, eps=eps).add(eps).reciprocal()


def compute_anchor_sampling_weight(points, mask, radius_2d, radius_3d, num_test=64, draws=None):
    height, width = points.shape[-3:-1]
    pixel_i, pixel_j = torch.meshgrid(torch.arange(height, device=points.device), torch.arange(width, device=points.device), indexing="ij")
    if draws is None:
        test_delta_i = torch.randint(-radius_2d, radius_2d + 1, (height, width, num_test), device=points.device)
        test_delta_j = torch.randint(-radius_2d, radius_2d + 1, (height, width, num_test), device=points.device)
    else:
        test_delta_i, test_delta_j = (d.to(points.device) for d in draws)
    test_i, test_j = pixel_i[..., None] + test_delta_i, pixel_j[..., None] + test_delta_j
    test_mask = (test_i >= 0) & (test_i < height) & (test_j >= 0) & (test_j < width)
    test_i, test_j = test_i.clamp(0, height - 1), test_j.clamp(0, width - 1)
    test_mask = test_mask & mask[..., test_i, test_j]
    test_points = points[..., test_i, test_j, :]
    test_dist = (test_points - points[..., None, :]).norm(dim=-1)
    weight = 1 / ((test_dist <= radius_3d[..., None]) & test_mask).float().sum(dim=-1).clamp_min(1)
    weight = torch.where(mask, weight, 0)
    return weight / weight.sum(dim=(-2, -1), keepdim=True).add(1e-7), (test_delta_i, test_delta_j)


def affine_invariant_local_loss(pred_points, gt_points, focal, global_scale, level, align, align_resolution=32, num_patches=16,
                                beta=0.0, trunc=1.0, sparsity_aware=False, draws=None, record=None):
    """The reference's local loss; `record` (a dict), when given, receives the draws, the kept patches and the alignment."""
    device, dtype = pred_points.device, pred_points.dtype
    *batch_shape, height, width, _ = pred_points.shape
    batch_size = math.prod(batch_shape)
    gt_mask = torch.isfinite(gt_points).all(dim=-1)
    gt_points = torch.where(gt_mask[..., None], gt_points, 1)
    pred_points, gt_points, gt_mask = pred_points.reshape(-1, height, width, 3), gt_points.reshape(-1, height, width, 3), gt_mask.reshape(-1, height, width)
    focal = focal.reshape(-1)
    global_scale = global_scale.reshape(-1) if global_scale is not None else None
    record = {} if record is None else record

    radius_2d = math.ceil(0.5 / level * (height ** 2 + width ** 2) ** 0.5)
    radius_3d = (0.5 / level / focal)[:, None, None] * gt_points[..., 2]
    weights, (record["delta_i"], record["delta_j"]) = compute_anchor_sampling_weight(
        gt_points, gt_mask, radius_2d, radius_3d, 64, None if draws is None else (draws["delta_i"], draws["delta_j"]))
    where_mask = torch.where(gt_mask)
    if draws is None:
        random_selection = torch.multinomial(weights[where_mask], num_patches * batch_size, replacement=True)
    else:
        random_selection = draws["selection"].to(device)
    record["selection"] = random_selection
    patch_batch_idx, patch_anchor_i, patch_anchor_j = [indices[random_selection] for indices in where_mask]

    patch_i, patch_j = torch.meshgrid(torch.arange(-radius_2d, radius_2d + 1, device=device),
                                      torch.arange(-radius_2d, radius_2d + 1, device=device), indexing="ij")
    patch_i, patch_j = patch_i + patch_anchor_i[:, None, None], patch_j + patch_anchor_j[:, None, None]
    patch_mask = (patch_i >= 0) & (patch_i < height) & (patch_j >= 0) & (patch_j < width)
    patch_i, patch_j = patch_i.clamp(0, height - 1), patch_j.clamp(0, width - 1)
    gt_patch_anchor_points = gt_points[patch_batch_idx, patch_anchor_i, patch_anchor_j]
    gt_patch_radius_3d = 0.5 / level / focal[patch_batch_idx] * gt_patch_anchor_points[:, 2]
    gt_patch_points = gt_points[patch_batch_idx[:, None, None], patch_i, patch_j]
    gt_patch_dist = (gt_patch_points - gt_patch_anchor_points[:, None, None, :]).norm(dim=-1)
    patch_mask &= gt_mask[patch_batch_idx[:, None, None], patch_i, patch_j]
    patch_mask &= gt_patch_dist <= gt_patch_radius_3d[:, None, None]

    nonempty = torch.where(patch_mask.sum(dim=(-2, -1)) >= 32)
    record["kept"] = nonempty[0]
    if nonempty[0].shape[0] == 0:
        return torch.tensor(0.0, dtype=dtype, device=device), {}
    patch_batch_idx, patch_i, patch_j = patch_batch_idx[nonempty], patch_i[nonempty], patch_j[nonempty]
    patch_mask = patch_mask[nonempty]
    gt_patch_points = gt_patch_points[nonempty]
    gt_patch_radius_3d = gt_patch_radius_3d[nonempty]
    pred_patch_points = pred_points[patch_batch_idx[:, None, None], patch_i, patch_j]

    pred_patch_points_lr, gt_patch_points_lr, patch_lr_mask = masked_nearest_resize(pred_patch_points, gt_patch_points, mask=patch_mask,
                                                                                    size=(align_resolution, align_resolution))
    local_scale, local_shift = align(pred_patch_points_lr.flatten(-3, -2), gt_patch_points_lr.flatten(-3, -2),
                                     patch_lr_mask.flatten(-2) / gt_patch_radius_3d[:, None].add(1e-7), trunc)
    record["scale"], record["shift"] = local_scale.detach(), local_shift.detach()
    if global_scale is not None:
        scale_differ = local_scale / global_scale[patch_batch_idx]
        patch_valid = (scale_differ > 0.1) & (scale_differ < 10.0) & (global_scale[patch_batch_idx] > 0)
    else:
        patch_valid = local_scale > 0
    local_scale, local_shift = torch.where(patch_valid, local_scale, 0), torch.where(patch_valid[:, None], local_shift, 0)
    patch_mask &= patch_valid[:, None, None]
    pred_patch_points = local_scale[:, None, None, None] * pred_patch_points + local_shift[:, None, None, :]

    gt_mean = harmonic_mean(gt_points[..., 2], gt_mask, dim=(-2, -1))
    patch_weight = patch_mask.float() / gt_patch_points[..., 2].clamp_min(0.1 * gt_mean[patch_batch_idx, None, None])
    loss = smooth((pred_patch_points - gt_patch_points).abs() * patch_weight[..., None], beta=beta).mean(dim=(-3, -2, -1))
    if sparsity_aware:
        sparsity = patch_mask.float().mean(dim=(-2, -1)) / patch_lr_mask.float().mean(dim=(-2, -1))
        loss = loss / (sparsity + 1e-7)
    loss = torch.scatter_reduce(torch.zeros(batch_size, dtype=dtype, device=device), dim=0, index=patch_batch_idx, src=loss,
                                reduce="sum") / num_patches
    loss = loss.reshape(batch_shape)
    err = (pred_patch_points.detach() - gt_patch_points).norm(dim=-1) / gt_patch_radius_3d[..., None, None]
    misc = {"truncated_error": weighted_mean(err.clamp_max(1), patch_mask).item(), "delta": weighted_mean((err < 1).float(), patch_mask).item()}
    return loss, misc
