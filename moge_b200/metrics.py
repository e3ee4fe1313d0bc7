"""Evaluation metrics on the GPU: the reference's `moge/test/metrics.py` (`compute_metrics` and its public helpers) with the same
signatures and return structure, plus `compute_metrics_batch` for same-shape stacks of images.

The work runs in the kernels of moge_b200/csrc/metrics.cu: the masked nearest resize to the 64 x 64 alignment grid (with the
valid low-resolution pixels compacted into fixed-size lists), a statistics pass (disparity least squares, max GT depth, segment
extents), one metric pass over every variant and segment, and the boundary-F1 counts.  The alignments run in moge_b200.alignment
on the fixed-size lists, where padding entries carry weight 0 (the candidate sets and objectives are those of the unpadded
problems).  Nothing is copied to the host until one non-blocking copy of a small result buffer per call; the final divisions
follow the reference's fp32 arithmetic on the host.

Divergences from the reference:
  - an image without a valid low-resolution pixel gets NaN for every aligned variant and for the boundary F1 (the reference
    raises inside its alignment solvers);
  - means are accumulated in fp64 (the reference sums fp32), so `rel` agrees to ~1e-6 relative rather than bit for bit.
"""
from __future__ import annotations

import math
from numbers import Number
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import alignment as A
from . import capi
from .capi import MogeError

__all__ = [
    "compute_metrics", "compute_metrics_batch", "masked_nearest_resize", "rel_depth", "delta1_depth", "rel_point", "delta1_point",
    "rel_point_local", "delta1_point_local", "boundary_f1", "F1_WEIGHTS", "F1_THRESHOLDS",
]

LR_SIZE = (64, 64)
# the reference's thresholds t (torch.linspace(0.05, 0.25, 10) in fp32, as Python floats) are also the weights of the average;
# a label is `ratio > 1 + t`, compared in fp32
F1_WEIGHTS: List[float] = torch.linspace(0.05, 0.25, 10).tolist()
F1_THRESHOLDS = np.array([np.float32(1 + t) for t in F1_WEIGHTS], dtype=np.float32)
MIN_SEGMENT_LR_PIXELS = 10


# ------------------------------------------------------------------------------------------------------------ public helpers
def rel_depth(pred: torch.Tensor, gt: torch.Tensor, eps: float = 1e-6):
    return ((pred - gt).abs() / (gt + eps)).mean().item()


def delta1_depth(pred: torch.Tensor, gt: torch.Tensor, eps: float = 1e-6):
    return (torch.maximum(gt / pred, pred / gt) < 1.25).float().mean().item()


def rel_point(pred: torch.Tensor, gt: torch.Tensor, eps: float = 1e-6):
    return (torch.norm(pred - gt, dim=-1) / (torch.norm(gt, dim=-1) + eps)).mean().item()


def delta1_point(pred: torch.Tensor, gt: torch.Tensor, eps: float = 1e-6):
    bound = 0.25 * torch.minimum(torch.norm(gt, dim=-1), torch.norm(pred, dim=-1))
    return (torch.norm(pred - gt, dim=-1) < bound).float().mean().item()


def rel_point_local(pred: torch.Tensor, gt: torch.Tensor, diameter: torch.Tensor):
    return (torch.norm(pred - gt, dim=-1) / diameter).mean().item()


def delta1_point_local(pred: torch.Tensor, gt: torch.Tensor, diameter: torch.Tensor):
    return (torch.norm(pred - gt, dim=-1) < 0.25 * diameter).float().mean().item()


def boundary_f1(pred: torch.Tensor, gt: torch.Tensor, mask: torch.Tensor, radius: int = 1):
    """Weighted F1 of the depth-ratio edge labels of pred against gt (H, W) within `radius`, on the boundary kernel."""
    if radius not in (1, 2, 3):
        raise MogeError(f"boundary_f1: radius {radius} is not one of 1, 2, 3")
    pred, gt, mask = _f32(pred)[None], _f32(gt)[None], _mask_u8(mask)[None]
    _same_shape(pred, gt, mask)
    counts = torch.zeros(1, capi.METRICS_F1_COUNTS, dtype=torch.int64, device=pred.device)
    var = capi.MetricVariant(capi.MV_DEPTH, pred.data_ptr(), None)
    _boundary(gt, mask, var, counts, counts.stride(0))
    return _f1_average(counts.cpu().numpy()[0], radius)


def masked_nearest_resize(*image: torch.Tensor, mask: torch.Tensor, size: Tuple[int, int], return_index: bool = False):
    """utils3d.pt.masked_nearest_resize: resize image(s) (..., H, W[, C]) to `size` by taking, per target pixel, the valid source
    pixel nearest its centre within a window of ceil(H / h) x ceil(W / w) source pixels.  Returns (*resized, resized_mask) and
    with return_index the index tuple (*batch indices, i, j) into the source."""
    capi.require_cuda("masked_nearest_resize", mask)
    H, W = mask.shape[-2:]
    th, tw = size
    batch_shape = mask.shape[:-2]
    lr_mask, lr_index, _, _, _ = _resize(capi.mask_u8(mask).reshape(-1, H, W), th, tw)
    lr_mask = lr_mask.reshape(*batch_shape, th, tw)
    lr_index = lr_index.reshape(*batch_shape, th, tw)
    batch_indices = [torch.arange(n, device=mask.device).reshape([1] * i + [n] + [1] * (len(batch_shape) - i - 1) + [1, 1])
                     for i, n in enumerate(batch_shape)]
    index = (*batch_indices, lr_index // W, lr_index % W)
    resized = tuple(x[index] for x in image)
    if return_index:
        return (*resized, lr_mask, index)
    return (*resized, lr_mask) if resized else lr_mask


# ------------------------------------------------------------------------------------------------------------ kernels
def _f32(t: torch.Tensor) -> torch.Tensor:
    capi.require_cuda("moge_b200.metrics", t)
    return t.detach().to(torch.float32).contiguous()


def _mask_u8(m: torch.Tensor) -> torch.Tensor:
    capi.require_cuda("moge_b200.metrics", m)
    return capi.mask_u8(m)


def _same_shape(*ts):
    shape = ts[0].shape[:3]
    for t in ts:
        if t.shape[:3] != shape:
            raise MogeError(f"shape mismatch: {tuple(t.shape)} vs {tuple(ts[0].shape)}")


def _resize(mask_u8: torch.Tensor, th: int, tw: int):
    B, H, W = mask_u8.shape
    dev = mask_u8.device
    n = th * tw
    lr_mask = torch.empty(B, th, tw, dtype=torch.uint8, device=dev)
    lr_index = torch.empty(B, th, tw, dtype=torch.int64, device=dev)
    lst = torch.empty(B, n, dtype=torch.int64, device=dev)
    lst_w = torch.empty(B, n, dtype=torch.float32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    capi.check(capi.lib().moge_metrics_resize(mask_u8.data_ptr(), B, H, W, th, tw, lr_mask.data_ptr(), lr_index.data_ptr(), lst.data_ptr(),
                                              lst_w.data_ptr(), count.data_ptr(), capi.current_stream()))
    return lr_mask.view(torch.bool), lr_index, lst, lst_w, count


def _boundary(gt_depth, mask_u8, var, counts_ptr_tensor, stride, offset: int = 0):
    B, H, W = gt_depth.shape
    thr = (capi.C.c_float * len(F1_THRESHOLDS))(*[float(t) for t in F1_THRESHOLDS])
    capi.check(capi.lib().moge_metrics_boundary(gt_depth.data_ptr(), mask_u8.data_ptr(), capi.C.byref(var), thr, B, H, W,
                                                counts_ptr_tensor.data_ptr() + offset, stride, capi.current_stream()))


def _f1_average(counts: np.ndarray, radius: int) -> float:
    """The reference's per-threshold fp32 precision / recall / F1 (its `precision` divides by the GT count, its `recall` by the
    predicted count; F1 is symmetric), then the t-weighted average in Python doubles."""
    two, tiny = np.float32(2), np.float32(1e-12)
    f1_list = []
    for t in range(capi.METRICS_F1_THRESHOLDS):
        tp, g, p = (np.float32(counts[(radius - 1) * 30 + t * 3 + k]) for k in range(3))
        precision = tp / max(g, tiny)
        recall = tp / max(p, tiny)
        f1_list.append(float(two * precision * recall / max(precision + recall, tiny)))
    return sum(w * f1 for w, f1 in zip(F1_WEIGHTS, f1_list)) / sum(F1_WEIGHTS)


def _key_average(list_of_dicts: List[Dict[str, float]]) -> Dict[str, float]:
    """Average of each key over the dicts, NaN skipped (NaN when nothing is left); an empty list gives {}."""
    keys = sorted({k for d in list_of_dicts for k in d})
    out = {}
    for k in keys:
        vals = [d[k] for d in list_of_dicts if k in d and d[k] is not None and not math.isnan(d[k])]
        out[k] = sum(vals) / len(vals) if vals else float("nan")
    return out


def _first(pred: Dict[str, torch.Tensor], keys: Sequence[str]) -> Optional[str]:
    return next((k for k in keys if k in pred), None)


class _Call:
    """The device side of one batched call, up to the single device-to-host copy."""


def _launch(pred: Dict[str, torch.Tensor], gt: Dict, labels: Optional[List[Dict]], vis: bool) -> _Call:
    mask = gt["depth_mask"]
    if not isinstance(mask, torch.Tensor) or mask.dim() != 3:
        raise MogeError("depth_mask must be a (B, H, W) tensor")
    mask_u8 = _mask_u8(mask)
    B, H, W = mask_u8.shape
    dev = mask_u8.device
    gt_depth, gt_points = _f32(gt["depth"]), _f32(gt["points"])
    if gt_depth.shape != (B, H, W) or gt_points.shape != (B, H, W, 3):
        raise MogeError(f"gt depth {tuple(gt_depth.shape)} / points {tuple(gt_points.shape)} do not match the mask {(B, H, W)}")
    preds = {}
    for k, v in pred.items():
        t = _f32(v)
        want = (B, 3, 3) if k == "intrinsics" else ((B, H, W, 3) if "point" in k else (B, H, W))
        if tuple(t.shape) != want:
            raise MogeError(f"pred[{k!r}] has shape {tuple(t.shape)}, expected {want}")
        preds[k] = t
    is_metric = bool(gt["is_metric"])
    local = "segmentation_mask" in gt and "points" in gt and any("points" in k for k in pred)
    seg_ids: List[List[int]] = []
    if local:
        if labels is None or len(labels) != B:
            raise MogeError("segmentation_labels must give one dict per image")
        seg_ids = [sorted(set(int(v) for v in lab.values())) for lab in labels]
        for ids in seg_ids:
            if len(ids) > capi.METRICS_MAX_SEGMENTS:
                raise MogeError(f"{len(ids)} segment ids in one image: at most {capi.METRICS_MAX_SEGMENTS} are supported")
            if ids and (ids[0] < -2 ** 31 or ids[-1] >= 2 ** 31):
                raise MogeError("segment ids must fit in int32")
        seg_map = gt["segmentation_mask"]
        if not isinstance(seg_map, torch.Tensor) or not seg_map.is_cuda or tuple(seg_map.shape) != (B, H, W):
            raise MogeError(f"segmentation_mask must be a CUDA (B, H, W) tensor matching the mask {(B, H, W)}")
    S = max((len(i) for i in seg_ids), default=0)
    has_seg = local and S > 0
    L = capi.lib()
    st = capi.current_stream()

    c = _Call()
    c.B, c.H, c.W, c.S, c.vis, c.local, c.labels, c.seg_ids = B, H, W, S, vis, local, labels, seg_ids
    lr_mask, lr_index, lst, lst_w, count = _resize(mask_u8, *LR_SIZE)
    c.lr_mask, c.lr_index = lr_mask, lr_index
    valid = lst_w > 0
    ok = (count > 0)
    nan = float("nan")
    n = lst.shape[1]
    idx3 = lst[..., None].expand(B, n, 3)

    def gd(x):
        return x.reshape(B, -1).gather(1, lst)

    def gp(x):
        return x.reshape(B, -1, 3).gather(1, idx3)

    g_d, g_p = gd(gt_depth), gp(gt_points)
    zero = torch.zeros((), dtype=torch.float32, device=dev)
    w_depth = torch.where(valid, 1 / g_d, zero)
    w_points = torch.where(valid, 1 / g_p.norm(dim=-1), zero)

    def params(scale=None, shift=None, third=None):
        p = torch.zeros(B, 4, dtype=torch.float32, device=dev)
        if scale is not None:
            p[:, 0] = torch.where(ok, scale, nan)
        if shift is not None:
            if shift.dim() == 2:
                p[:, 1:] = torch.where(ok[:, None], shift, nan)
            else:
                p[:, 1] = torch.where(ok, shift, nan)
        if third is not None:
            p[:, 2] = third
        return p

    variants = []          # (name, kind, src, params)
    aligned = None         # (kind, src, params) of pred_depth_aligned
    c.points_vis = None
    if "depth_metric" in preds and is_metric:
        p = params()
        variants.append(("depth_metric", capi.MV_DEPTH, preds["depth_metric"], p))
        aligned = aligned or (capi.MV_DEPTH, preds["depth_metric"], p)
    k = _first(preds, ("depth_scale_invariant", "depth_metric"))
    if k is not None:
        p = params(scale=A.align_depth_scale(gd(preds[k]), g_d, w_depth))
        variants.append(("depth_scale_invariant", capi.MV_DEPTH_SCALE, preds[k], p))
        aligned = aligned or (capi.MV_DEPTH_SCALE, preds[k], p)
    k = _first(preds, ("depth_affine_invariant", "depth_scale_invariant", "depth_metric"))
    if k is not None:
        scale, shift = A.align_depth_affine(gd(preds[k]), g_d, w_depth)
        p = params(scale=scale, shift=shift)
        variants.append(("depth_affine_invariant", capi.MV_DEPTH_AFFINE, preds[k], p))
        aligned = aligned or (capi.MV_DEPTH_AFFINE, preds[k], p)
    k = _first(preds, ("disparity_affine_invariant", "depth_scale_invariant", "depth_metric"))
    disp = None
    if k is not None:
        disp = (capi.MV_DISPARITY if k == "disparity_affine_invariant" else capi.MV_DISPARITY_FROM_DEPTH, preds[k])

    # statistics pass: disparity least squares, max GT depth, segment diameters
    ws = capi.workspace(L.moge_metrics_workspace_bytes, B, H, W, S if has_seg else 0, device=dev)
    disp_params = torch.empty(B, 4, dtype=torch.float32, device=dev)
    seg = ids_t = nseg_t = diameter = None
    if has_seg:
        seg = gt["segmentation_mask"].detach().to(torch.int32).contiguous()
        ids_h = torch.zeros(B, S, dtype=torch.int32, pin_memory=True)
        nseg_h = torch.zeros(B, dtype=torch.int32, pin_memory=True)
        for b, ids in enumerate(seg_ids):
            ids_h[b, :len(ids)] = torch.tensor(ids, dtype=torch.int32)
            nseg_h[b] = len(ids)
        ids_t, nseg_t = ids_h.to(dev, non_blocking=True), nseg_h.to(dev, non_blocking=True)
        diameter = torch.empty(B, S, dtype=torch.float32, device=dev)
    if disp is not None or has_seg:
        capi.check(L.moge_metrics_stats(gt_depth.data_ptr(), gt_points.data_ptr(), mask_u8.data_ptr(),
                                        None if disp is None else disp[1].data_ptr(), int(disp is not None and disp[0] == capi.MV_DISPARITY_FROM_DEPTH),
                                        capi.ptr(seg), capi.ptr(ids_t), capi.ptr(nseg_t), S if has_seg else 0, B, H, W,
                                        disp_params.data_ptr(), capi.ptr(diameter), ws.data_ptr(), ws.numel(), st))
    if disp is not None:
        p = params(scale=disp_params[:, 0], shift=disp_params[:, 1], third=disp_params[:, 2])
        variants.append(("disparity_affine_invariant", disp[0], disp[1], p))
        if aligned is None:
            aligned = (disp[0], disp[1], params(scale=disp_params[:, 0], shift=disp_params[:, 1], third=1e-6))

    if "points_metric" in preds and is_metric:
        src = preds["points_metric"]
        p = params(shift=A.align_points_xyz_shift(gp(src), g_p, w_points))
        variants.append(("points_metric", capi.MV_POINTS_SHIFT, src, p))
        if c.points_vis is None:
            c.points_vis = (pred["points_metric"], None, None)
    k = _first(preds, ("points_scale_invariant", "points_metric"))
    if k is not None:
        scale = A.align_points_scale(gp(preds[k]), g_p, w_points)
        p = params(scale=scale)
        variants.append(("points_scale_invariant", capi.MV_POINTS_SCALE, preds[k], p))
        if vis and c.points_vis is None:
            c.points_vis = (pred["points_scale_invariant"], p[:, 0], None)
    k = _first(preds, ("points_affine_invariant", "points_scale_invariant", "points_metric"))
    if k is not None:
        scale, shift = A.align_points_scale_xyz_shift(gp(preds[k]), g_p, w_points)
        p = params(scale=scale, shift=shift)
        variants.append(("points_affine_invariant", capi.MV_POINTS_AFFINE, preds[k], p))
        if vis and c.points_vis is None:
            c.points_vis = (pred["points_affine_invariant"], p[:, 0], p[:, 1:])

    # result buffer: eval outputs, F1 counts (int64 view), per-slot low-resolution counts, valid low-resolution count, fx
    o_f1 = capi.METRICS_OUT_SEGMENTS + 3 * S
    o_lr = o_f1 + capi.METRICS_F1_COUNTS
    o_count = o_lr + S
    o_fx = o_count + 1
    K = o_fx + 2
    out = torch.zeros(B, K, dtype=torch.float64, device=dev)
    local_src = seg_params = None
    if has_seg:
        local_src = preds[next(k for k in pred if "points" in k)]
        seg_c = seg.reshape(B, -1).gather(1, lst)
        match = (seg_c[:, None, :] == ids_t[:, :, None]) & valid[:, None, :]
        w_seg = torch.where(match, (1 / diameter)[:, :, None], zero)
        out[:, o_lr:o_lr + S] = match.sum(-1).to(torch.float64)
        scale, shift = A.align_points_scale_xyz_shift(gp(local_src)[:, None].expand(B, S, n, 3), g_p[:, None].expand(B, S, n, 3), w_seg)
        seg_params = torch.cat([scale[..., None], shift], dim=-1).contiguous()
    vs = (capi.MetricVariant * max(1, len(variants)))(*[capi.MetricVariant(kind, src.data_ptr(), p.data_ptr())
                                                         for _, kind, src, p in variants])
    capi.check(L.moge_metrics_eval(gt_depth.data_ptr(), gt_points.data_ptr(), mask_u8.data_ptr(), vs, len(variants), capi.ptr(local_src),
                                   capi.ptr(seg), capi.ptr(ids_t), capi.ptr(nseg_t), S if has_seg else 0, capi.ptr(seg_params),
                                   capi.ptr(diameter), B, H, W, out.data_ptr(), K, ws.data_ptr(), ws.numel(), st))
    c.boundary = aligned is not None and bool(gt["has_sharp_boundary"])
    if c.boundary:
        var = capi.MetricVariant(aligned[0], aligned[1].data_ptr(), aligned[2].data_ptr())
        _boundary(gt_depth, mask_u8, var, out, K, offset=o_f1 * 8)
    out[:, o_count] = count.to(torch.float64)
    c.fov = "intrinsics" in pred and "intrinsics" in gt
    if c.fov:
        out[:, o_fx] = preds["intrinsics"][:, 0, 0].to(torch.float64)
        out[:, o_fx + 1] = _f32(gt["intrinsics"]).reshape(B, 3, 3)[:, 0, 0].to(torch.float64)
    c.variants = [(name, kind) for name, kind, _, _ in variants]
    c.o_f1, c.o_lr, c.o_count, c.o_fx = o_f1, o_lr, o_count, o_fx
    c.aligned = aligned
    c.only_depth = not any("point" in k for k in pred)
    c.gt_intrinsics = gt.get("intrinsics")
    c.out = out
    c.host = torch.empty(out.shape, dtype=torch.float64, pin_memory=True)
    c.host.copy_(out, non_blocking=True)
    c.event = torch.cuda.Event()
    c.event.record()
    return c


def _aligned_depth_map(aligned, b: int) -> torch.Tensor:
    kind, src, p = aligned
    x = src[b]
    if kind == capi.MV_DEPTH:
        return x
    if kind == capi.MV_DEPTH_SCALE:
        return x * p[b, 0]
    if kind == capi.MV_DEPTH_AFFINE:
        return x * p[b, 0] + p[b, 1]
    d = 1 / x if kind == capi.MV_DISPARITY_FROM_DEPTH else x
    return 1 / torch.maximum(d * p[b, 0] + p[b, 1], p[b, 2])


def _depth_map_to_point_map(depth: torch.Tensor, intrinsics: torch.Tensor) -> torch.Tensor:
    """utils3d.pt.depth_map_to_point_map with normalized intrinsics and pixel-centre UV (u = (j + 0.5) / W, v = (i + 0.5) / H)."""
    H, W = depth.shape[-2:]
    u = (torch.arange(W, dtype=depth.dtype, device=depth.device) + 0.5) / W
    v = (torch.arange(H, dtype=depth.dtype, device=depth.device) + 0.5) / H
    fx, fy, cx, cy = intrinsics[..., 0, 0], intrinsics[..., 1, 1], intrinsics[..., 0, 2], intrinsics[..., 1, 2]
    x = (u[None, :] - cx[..., None, None]) / fx[..., None, None] * depth
    y = (v[:, None] - cy[..., None, None]) / fy[..., None, None] * depth
    return torch.stack([x, y, depth], dim=-1)


def _finish(c: _Call) -> List[Tuple[Dict[str, Dict[str, Number]], Dict[str, torch.Tensor]]]:
    c.event.synchronize()
    host = c.host.numpy()
    f1_view = c.host[:, c.o_f1:c.o_f1 + capi.METRICS_F1_COUNTS].view(torch.int64).numpy()
    nan = float("nan")
    results = []
    for b in range(c.B):
        row = host[b]
        ok = row[c.o_count] > 0
        n = row[2 * capi.METRICS_MAX_VARIANTS]
        n32 = np.float32(n)
        metrics: Dict[str, Dict[str, Number]] = {}
        for v, (name, kind) in enumerate(c.variants):
            if not ok and kind != capi.MV_DEPTH:
                metrics[name] = {"rel": nan, "delta1": nan}
                continue
            with np.errstate(divide="ignore", invalid="ignore"):
                rel = float(np.float32(row[2 * v] / n)) if n else nan
                delta1 = float(np.float32(row[2 * v + 1]) / n32)
            metrics[name] = {"rel": rel, "delta1": delta1}
        if c.local:
            ids = c.seg_ids[b]
            slot = {i: s for s, i in enumerate(ids)}
            local = []
            for _, sid in c.labels[b].items():
                s = slot[int(sid)]
                if row[c.o_lr + s] < MIN_SEGMENT_LR_PIXELS:
                    continue
                base = capi.METRICS_OUT_SEGMENTS + 3 * s
                rs, dc, pn = row[base], row[base + 1], row[base + 2]
                local.append({"rel": float(np.float32(rs / pn)), "delta1": float(np.float32(dc) / np.float32(pn))})
            metrics["local_points"] = _key_average(local)
        if c.fov:
            pfx = torch.tensor(row[c.o_fx], dtype=torch.float32)
            gfx = torch.tensor(row[c.o_fx + 1], dtype=torch.float32)
            diff = torch.rad2deg(2 * torch.atan(0.5 / pfx) - 2 * torch.atan(0.5 / gfx))
            metrics["fov_x"] = {"mae": diff.abs().mean().item(), "deviation": diff.item()}
        if c.boundary:
            if ok or c.aligned[0] == capi.MV_DEPTH:
                metrics["boundary"] = {f"radius{r}_f1": _f1_average(f1_view[b], r) for r in (1, 2, 3)}
            else:
                metrics["boundary"] = {f"radius{r}_f1": nan for r in (1, 2, 3)}
        misc: Dict[str, torch.Tensor] = {}
        if c.vis:
            depth_map = _aligned_depth_map(c.aligned, b) if c.aligned is not None else None
            if c.points_vis is not None:
                src, scale, shift = c.points_vis
                pts = src[b]
                if scale is not None:
                    pts = pts * scale[b]
                if shift is not None:
                    pts = pts + shift[b]
                misc["pred_points"] = pts
            if c.only_depth:
                misc["pred_points"] = _depth_map_to_point_map(depth_map, c.gt_intrinsics[b] if c.gt_intrinsics.dim() == 3 else c.gt_intrinsics)
            if depth_map is not None:
                misc["pred_depth"] = depth_map
        results.append((metrics, misc))
    return results


def compute_metrics_batch(pred: Dict[str, torch.Tensor], gt: Dict, vis: bool = False):
    """compute_metrics over a stack of same-shape images: pred / gt maps (B, H, W) and (B, H, W, 3), intrinsics (B, 3, 3), the
    mask (B, H, W), `segmentation_labels` a list of B dicts.  `is_metric` and `has_sharp_boundary` hold for the whole batch.
    Returns B (metrics, misc) pairs, each bitwise equal to compute_metrics on that image alone."""
    labels = gt.get("segmentation_labels")
    return _finish(_launch(pred, gt, labels, vis))


def compute_metrics(pred: Dict[str, torch.Tensor], gt: Dict, vis: bool = False):
    """The reference's compute_metrics(pred, gt, vis) -> (metrics, misc) on CUDA tensors of one image."""
    p = {k: v[None] for k, v in pred.items()}
    g = {k: (v[None] if isinstance(v, torch.Tensor) else v) for k, v in gt.items() if k != "segmentation_labels"}
    labels = [gt["segmentation_labels"]] if "segmentation_labels" in gt else None
    return _finish(_launch(p, g, labels, vis))[0]
