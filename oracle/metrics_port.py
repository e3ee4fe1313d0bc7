"""Functional plain-torch restatement of the reference's `compute_metrics` (moge/test/metrics.py): the checker of
moge_b200.metrics on fresh inputs, on the CPU or on CUDA.

It follows the reference's branch logic and fp32 arithmetic; masked nearest resize and sliding windows come from
oracle/utils3d_metrics.py, depth_map_to_point_map from the utils3d stand-in (oracle/utils3d_shim).  The alignment solvers are
passed in as a module with the reference's alignment API: the reference's own `moge.utils.alignment` where it is importable
(oracle/make_metrics_golden.py), moge_b200.alignment on CUDA.
"""
import math

import torch

from oracle.utils3d_metrics import install

u3d = install()

F1_T = torch.linspace(0.05, 0.25, 10).tolist()


def _rel_depth(p, g):
    return ((p - g).abs() / (g + 1e-6)).mean().item()


def _delta_depth(p, g):
    return (torch.maximum(g / p, p / g) < 1.25).float().mean().item()


def _rel_point(p, g):
    return ((p - g).norm(dim=-1) / (g.norm(dim=-1) + 1e-6)).mean().item()


def _delta_point(p, g):
    return ((p - g).norm(dim=-1) < 0.25 * torch.minimum(g.norm(dim=-1), p.norm(dim=-1))).float().mean().item()


def boundary_counts(pred, gt, mask, radius):
    """(TP, GT, pred) label counts per threshold, as int64 (10, 3)."""
    k = 2 * radius + 1
    y, x = torch.meshgrid(torch.arange(-radius, radius + 1.0), torch.arange(-radius, radius + 1.0), indexing="ij")
    disc = ((x ** 2 + y ** 2) <= radius ** 2 + 1e-5).to(pred.device)
    pw, gw = u3d.sliding_window_2d(pred, k, 1, dim=(-2, -1)), u3d.sliding_window_2d(gt, k, 1, dim=(-2, -1))
    mw = disc & u3d.sliding_window_2d(mask, k, 1, dim=(-2, -1))
    c = (slice(radius, -radius), slice(radius, -radius))
    pr, gr = pw / pred[c][..., None, None], gw / gt[c][..., None, None]
    valid = mask[c][..., None, None] & mw
    out = []
    for t in F1_T:
        pl, gl = pr > 1 + t, gr > 1 + t
        out.append([(pl & gl & valid).sum().item(), (gl & valid).sum().item(), (pl & valid).sum().item()])
    return torch.tensor(out, dtype=torch.int64)


def boundary_f1(pred, gt, mask, radius):
    f1s = []
    for tp, g, p in boundary_counts(pred, gt, mask, radius).float():
        precision, recall = tp / g.clamp_min(1e-12), tp / p.clamp_min(1e-12)
        f1s.append((2 * precision * recall / (precision + recall).clamp_min(1e-12)).item())
    return sum(w * f for w, f in zip(F1_T, f1s)) / sum(F1_T)


def _key_average(dicts):
    out = {}
    for k in sorted({k for d in dicts for k in d}):
        vals = [d[k] for d in dicts if not math.isnan(d[k])]
        out[k] = sum(vals) / len(vals) if vals else float("nan")
    return out


def compute_metrics(pred, gt, vis=False, alignment=None):
    """(metrics, misc) of one image, as the reference computes them; `alignment`: the solver module."""
    al = alignment
    mask, gd, gp = gt["depth_mask"], gt["depth"], gt["points"]
    lr_mask, lr_index = u3d.masked_nearest_resize(mask=mask, size=(64, 64), return_index=True)
    metrics, misc = {}, {}
    depth_aligned = points_aligned = None
    first = lambda keys: next((pred[k] for k in keys if k in pred), None)  # noqa: E731
    lr = lambda x: x[lr_index][lr_mask]  # noqa: E731

    def depth_entry(p):
        return {"rel": _rel_depth(p[mask], gd[mask]), "delta1": _delta_depth(p[mask], gd[mask])}

    def points_entry(p):
        return {"rel": _rel_point(p[mask], gp[mask]), "delta1": _delta_point(p[mask], gp[mask])}

    if "depth_metric" in pred and gt["is_metric"]:
        metrics["depth_metric"] = depth_entry(pred["depth_metric"])
        depth_aligned = pred["depth_metric"]
    src = first(("depth_scale_invariant", "depth_metric"))
    if src is not None:
        s = al.align_depth_scale(lr(src), lr(gd), 1 / lr(gd))
        metrics["depth_scale_invariant"] = depth_entry(src * s)
        depth_aligned = src * s if depth_aligned is None else depth_aligned
    src = first(("depth_affine_invariant", "depth_scale_invariant", "depth_metric"))
    if src is not None:
        s, b = al.align_depth_affine(lr(src), lr(gd), 1 / lr(gd))
        metrics["depth_affine_invariant"] = depth_entry(src * s + b)
        depth_aligned = src * s + b if depth_aligned is None else depth_aligned
    if "disparity_affine_invariant" in pred:
        disp = pred["disparity_affine_invariant"]
    else:
        d = first(("depth_scale_invariant", "depth_metric"))
        disp = None if d is None else 1 / d
    if disp is not None:
        s, b = al.align_affine_lstsq(disp[mask], 1 / gd[mask])
        disp = disp * s + b
        metrics["disparity_affine_invariant"] = depth_entry(1 / disp.clamp_min(1 / gd[mask].max().item()))
        depth_aligned = 1 / disp.clamp_min(1e-6) if depth_aligned is None else depth_aligned
    w_pts = lambda: 1 / lr(gp).norm(dim=-1)  # noqa: E731
    if "points_metric" in pred and gt["is_metric"]:
        src = pred["points_metric"]
        metrics["points_metric"] = points_entry(src + al.align_points_xyz_shift(lr(src), lr(gp), w_pts()))
        points_aligned = src
    src = first(("points_scale_invariant", "points_metric"))
    if src is not None:
        s = al.align_points_scale(lr(src), lr(gp), w_pts())
        metrics["points_scale_invariant"] = points_entry(src * s)
        if vis and points_aligned is None:
            points_aligned = pred["points_scale_invariant"] * s
    src = first(("points_affine_invariant", "points_scale_invariant", "points_metric"))
    if src is not None:
        s, b = al.align_points_scale_xyz_shift(lr(src), lr(gp), w_pts())
        metrics["points_affine_invariant"] = points_entry(src * s + b)
        if vis and points_aligned is None:
            points_aligned = pred["points_affine_invariant"] * s + b
    if "segmentation_mask" in gt and any("points" in k for k in pred):
        src = next(pred[k] for k in pred if "points" in k)
        seg, seg_lr = gt["segmentation_mask"], gt["segmentation_mask"][lr_index]
        local = []
        for sid in gt["segmentation_labels"].values():
            m_lr = (seg_lr == sid) & lr_mask
            if m_lr.sum().item() < 10:
                continue
            m = (seg == sid) & mask
            g = gp[m]
            diam = (g.max(dim=0).values - g.min(dim=0).values).max()
            s, b = al.align_points_scale_xyz_shift(src[lr_index][m_lr], gp[lr_index][m_lr], 1 / diam.expand(int(m_lr.sum().item())))
            e = (src[m] * s + b - g).norm(dim=-1)
            local.append({"rel": (e / diam).mean().item(), "delta1": (e < 0.25 * diam).float().mean().item()})
        metrics["local_points"] = _key_average(local)
    if "intrinsics" in pred and "intrinsics" in gt:
        fov = lambda K: 2 * torch.atan(0.5 / K[..., 0, 0])  # noqa: E731
        diff = torch.rad2deg(fov(pred["intrinsics"]) - fov(gt["intrinsics"]))
        metrics["fov_x"] = {"mae": diff.abs().mean().item(), "deviation": diff.item()}
    if depth_aligned is not None and gt["has_sharp_boundary"]:
        metrics["boundary"] = {f"radius{r}_f1": boundary_f1(depth_aligned, gd, mask, r) for r in (1, 2, 3)}
    if vis:
        if points_aligned is not None:
            misc["pred_points"] = points_aligned
        if not any("point" in k for k in pred):
            misc["pred_points"] = u3d.depth_map_to_point_map(depth_aligned, intrinsics=gt["intrinsics"])
        if depth_aligned is not None:
            misc["pred_depth"] = depth_aligned
    return metrics, misc
