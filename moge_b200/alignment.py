"""Truncated-L1 alignment solvers on the GPU: the functions of the reference's `moge/utils/alignment.py` that its evaluation
metrics and training losses call, with the same signatures, batch semantics ((..., N) / (..., N, 3)) and return conventions.

The kernels (moge_b200/csrc/align.cu) choose the solution: the element of align(), or the (anchor, element) pair of the anchored
solvers.  Scale and shift are then rebuilt from those indices with torch gathers, by the reference's closed forms, so they are
differentiable with respect to the inputs as the reference's are.  Inputs must be CUDA tensors (there is no CPU fallback); they
are solved in fp32.

Divergences from the reference:
  - an image without a positive weight gets NaN scale and shift from the anchored solvers (the reference raises IndexError at
    batch 1 and, at batch > 1, returns a value built from another image's anchor);
  - the truncated objective is minimised with fp64 prefix sums, so among near-equal local minima the least one is found exactly;
  - align_affine_lstsq returns values without an autograd graph.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple, Union

import torch

from . import capi
from .capi import MogeError

__all__ = [
    "align", "align_depth_scale", "align_depth_affine", "align_points_scale", "align_points_scale_z_shift",
    "align_points_scale_xyz_shift", "align_points_z_shift", "align_points_xyz_shift", "align_affine_lstsq",
]


def _rows(t: torch.Tensor, shape) -> torch.Tensor:
    capi.require_cuda("moge_b200.alignment", t)
    return t.detach().reshape(shape).to(torch.float32).contiguous()


def _check_n(n: int, limit: int, what: str) -> None:
    if n < 1 or n > limit:
        raise MogeError(f"{what}: n = {n} is outside [1, {limit}] (at most {capi.ALIGN_MAX_POINTS} points per problem)")


def align(x: torch.Tensor, y: torch.Tensor, w: torch.Tensor, trunc: Optional[Union[float, torch.Tensor]] = None,
          eps: float = 1e-7) -> Tuple[torch.Tensor, torch.Tensor, torch.LongTensor]:
    """Solve `min_a sum_i w_i |a x_i - y_i|`, or `min_a sum_i min(trunc_i, w_i |a x_i - y_i|)` when trunc is given (w_i >= 0).

    x, y, w: (..., n); trunc: None, a float, or a tensor broadcastable to (..., n).
    Returns a (...) (differentiable), loss (...) (the objective at a; detached when truncated) and index (...), a = y[index] / x[index].
    """
    if eps != 1e-7:
        raise MogeError("align: only eps = 1e-7 (the reference's default) is supported")
    x, y, w = torch.broadcast_tensors(x, y, w)
    batch_shape, n = x.shape[:-1], x.shape[-1]
    _check_n(n, 3 * capi.ALIGN_MAX_POINTS, "align")
    batch = math.prod(batch_shape)
    xr, yr, wr = (_rows(t, (batch, n)) for t in (x, y, w))
    t_dev, per_elem = None, 0
    if trunc is not None:
        if isinstance(trunc, torch.Tensor) and trunc.numel() > 1:
            t_dev, per_elem = _rows(torch.broadcast_to(trunc, x.shape), (batch, n)), 1
        else:
            t_dev = torch.full((1,), float(trunc), dtype=torch.float32, device=x.device)
    a_k = torch.empty(batch, dtype=torch.float32, device=x.device)
    loss_k = torch.empty_like(a_k)
    index = torch.empty(batch, dtype=torch.int64, device=x.device)
    ws = capi.workspace(capi.lib().moge_align_workspace_bytes, capi.ALIGN_PLAIN, int(trunc is not None), batch, n, device=x.device)
    capi.check(capi.lib().moge_align(xr.data_ptr(), yr.data_ptr(), wr.data_ptr(), None if t_dev is None else t_dev.data_ptr(), per_elem,
                                     batch, n, a_k.data_ptr(), loss_k.data_ptr(), index.data_ptr(), ws.data_ptr(), ws.numel(),
                                     capi.current_stream()))
    sign = torch.sign(x)
    x, y = x * sign, y * sign
    idx = index.reshape(*batch_shape, 1)
    a = (torch.gather(y, -1, idx) / torch.gather(x, -1, idx).clamp_min(eps)).squeeze(-1)
    if trunc is None:
        loss = (w * (a[..., None] * x - y).abs()).sum(dim=-1)
    else:
        loss = loss_k.reshape(batch_shape)
    return a, loss, index.reshape(batch_shape)


def _anchored(mode: int, src: torch.Tensor, tgt: torch.Tensor, weight: torch.Tensor, trunc, batch: int, n: int):
    """(loss, anchor, index) per image; anchor = index = -1 for an image without a positive weight."""
    _check_n(n, capi.ALIGN_MAX_POINTS, "align")
    if trunc is not None:
        if isinstance(trunc, torch.Tensor) and trunc.numel() != 1:
            raise MogeError("the anchored solvers take a scalar trunc")
        trunc = float(trunc)
        if not trunc >= 0.0:
            raise MogeError(f"trunc must be >= 0 (got {trunc})")
    shape = (batch, n) if mode == capi.ANCHOR_DEPTH else (batch, n, 3)
    s, t, w = _rows(src, shape), _rows(tgt, shape), _rows(weight, (batch, n))
    loss = torch.empty(batch, dtype=torch.float32, device=src.device)
    anchor = torch.empty(batch, dtype=torch.int64, device=src.device)
    index = torch.empty_like(anchor)
    ws = capi.workspace(capi.lib().moge_align_workspace_bytes, mode, int(trunc is not None), batch, n, device=src.device)
    capi.check(capi.lib().moge_align_anchored(s.data_ptr(), t.data_ptr(), w.data_ptr(), mode, -1.0 if trunc is None else trunc, batch,
                                              n, loss.data_ptr(), anchor.data_ptr(), index.data_ptr(), ws.data_ptr(), ws.numel(),
                                              capi.current_stream()))
    return loss, anchor, index


def _gather(t: torch.Tensor, i: torch.Tensor) -> torch.Tensor:
    return torch.gather(t, 1, i[:, None]).squeeze(-1)


def align_depth_scale(depth_src: torch.Tensor, depth_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                      trunc: Optional[Union[float, torch.Tensor]] = None):
    """Scale (...) aligning depth_src (..., N) to depth_tgt (..., N)."""
    scale, _, _ = align(depth_src, depth_tgt, weight, trunc)
    return scale


def align_depth_affine(depth_src: torch.Tensor, depth_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                       trunc: Optional[Union[float, torch.Tensor]] = None):
    """Scale (...) and shift (...) aligning depth_src (..., N) to depth_tgt (..., N) with weights (..., N)."""
    batch_shape, n = depth_src.shape[:-1], depth_src.shape[-1]
    batch = math.prod(batch_shape)
    depth_src, depth_tgt, weight = depth_src.reshape(batch, n), depth_tgt.reshape(batch, n), weight.reshape(batch, n)
    _, anchor, index = _anchored(capi.ANCHOR_DEPTH, depth_src, depth_tgt, weight, trunc, batch, n)
    valid = anchor >= 0
    i1, i2 = anchor.clamp_min(0), index.clamp_min(0)
    tgt_1, src_1 = _gather(depth_tgt, i1), _gather(depth_src, i1)
    tgt_2, src_2 = _gather(depth_tgt, i2), _gather(depth_src, i2)
    scale = (tgt_2 - tgt_1) / torch.where(src_2 != src_1, src_2 - src_1, 1e-7)
    shift = tgt_1 - scale * src_1
    nan = torch.full_like(scale, float("nan"))
    scale, shift = torch.where(valid, scale, nan), torch.where(valid, shift, nan)
    return scale.reshape(batch_shape), shift.reshape(batch_shape)


def align_points_scale(points_src: torch.Tensor, points_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                       trunc: Optional[Union[float, torch.Tensor]] = None):
    """Scale (...) aligning points_src (..., N, 3) to points_tgt (..., N, 3) with weights (..., N)."""
    scale, _, _ = align(points_src.flatten(-2), points_tgt.flatten(-2), weight[..., None].expand_as(points_src).flatten(-2), trunc)
    return scale


def _points_scale_shift(mode: int, points_src, points_tgt, weight, trunc):
    batch_shape, n = points_src.shape[:-2], points_src.shape[-2]
    batch = math.prod(batch_shape)
    points_src, points_tgt, weight = points_src.reshape(batch, n, 3), points_tgt.reshape(batch, n, 3), weight.reshape(batch, n)
    _, anchor, index = _anchored(mode, points_src, points_tgt, weight, trunc, batch, n)
    valid = anchor >= 0
    anchor, index_2 = anchor.clamp_min(0), index.clamp_min(0)
    index_1 = anchor * 3 + index_2 % 3
    if mode == capi.ANCHOR_POINTS_Z:
        zeros = torch.zeros_like(points_src[..., 2])
        anchored_src = torch.stack([zeros, zeros, points_src[..., 2]], dim=-1)
        anchored_tgt = torch.stack([zeros, zeros, points_tgt[..., 2]], dim=-1)
    else:
        anchored_src, anchored_tgt = points_src, points_tgt
    src_1, tgt_1 = _gather(anchored_src.flatten(-2), index_1), _gather(anchored_tgt.flatten(-2), index_1)
    src_2, tgt_2 = _gather(points_src.flatten(-2), index_2), _gather(points_tgt.flatten(-2), index_2)
    scale = (tgt_2 - tgt_1) / torch.where(src_2 != src_1, src_2 - src_1, 1.0)
    ia = anchor[:, None, None].expand(-1, -1, 3)
    shift = torch.gather(anchored_tgt, 1, ia).squeeze(-2) - scale[..., None] * torch.gather(anchored_src, 1, ia).squeeze(-2)
    scale = torch.where(valid, scale, torch.full_like(scale, float("nan")))
    shift = torch.where(valid[:, None], shift, torch.full_like(shift, float("nan")))
    return scale.reshape(batch_shape), shift.reshape(*batch_shape, 3)


def align_points_scale_z_shift(points_src: torch.Tensor, points_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                               trunc: Optional[Union[float, torch.Tensor]] = None):
    """Shared xyz scale (...) and z shift (..., 3) (x and y shifts are zero) aligning points_src (..., N, 3) to points_tgt."""
    return _points_scale_shift(capi.ANCHOR_POINTS_Z, points_src, points_tgt, weight, trunc)


def align_points_scale_xyz_shift(points_src: torch.Tensor, points_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                                 trunc: Optional[Union[float, torch.Tensor]] = None, max_iters: int = 30, eps: float = 1e-6):
    """Shared xyz scale (...) and xyz shift (..., 3) aligning points_src (..., N, 3) to points_tgt (max_iters, eps: unused, as in
    the reference)."""
    return _points_scale_shift(capi.ANCHOR_POINTS_XYZ, points_src, points_tgt, weight, trunc)


def align_points_z_shift(points_src: torch.Tensor, points_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                         trunc: Optional[Union[float, torch.Tensor]] = None, max_iters: int = 30, eps: float = 1e-6):
    """z shift (..., 3) (x and y zero) aligning points_src (..., N, 3) to points_tgt."""
    shift, _, _ = align(torch.ones_like(points_src[..., 2]), points_tgt[..., 2] - points_src[..., 2], weight, trunc)
    return torch.stack([torch.zeros_like(shift), torch.zeros_like(shift), shift], dim=-1)


def align_points_xyz_shift(points_src: torch.Tensor, points_tgt: torch.Tensor, weight: Optional[torch.Tensor],
                           trunc: Optional[Union[float, torch.Tensor]] = None, max_iters: int = 30, eps: float = 1e-6):
    """Per-axis shift (..., 3) aligning points_src (..., N, 3) to points_tgt."""
    shift, _, _ = align(torch.ones_like(points_src).swapaxes(-2, -1), (points_tgt - points_src).swapaxes(-2, -1), weight[..., None, :],
                        trunc)
    return shift


def align_affine_lstsq(x: torch.Tensor, y: torch.Tensor, w: torch.Tensor = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """a (...), b (...): the least-squares solution of [sqrt(w) x, 1] (a, b)^T = sqrt(w) y over the last axis, as the reference
    poses it to torch.linalg.lstsq (the column of ones is not weighted).  x, y, w: (..., N); any N."""
    batch_shape, n = x.shape[:-1], x.shape[-1]
    batch = math.prod(batch_shape)
    if batch == 0 or n == 0:
        raise MogeError(f"align_affine_lstsq: empty input {tuple(x.shape)}")
    xr, yr = _rows(x, (batch, n)), _rows(y, (batch, n))
    wr = None if w is None else _rows(torch.broadcast_to(w, x.shape), (batch, n))
    a = torch.empty(batch, dtype=torch.float32, device=x.device)
    b = torch.empty_like(a)
    capi.check(capi.lib().moge_align_affine_lstsq(xr.data_ptr(), yr.data_ptr(), None if wr is None else wr.data_ptr(), batch, n,
                                                  a.data_ptr(), b.data_ptr(), capi.current_stream()))
    return a.reshape(batch_shape), b.reshape(batch_shape)
