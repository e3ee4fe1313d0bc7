"""The two utils3d functions that the reference's evaluation metrics call (moge/test/metrics.py:71-73 and :128):
`sliding_window_2d` and `masked_nearest_resize`, restated from utils3d's published semantics.  TEST INFRASTRUCTURE ONLY.

`install()` adds them to the utils3d stand-in (oracle/utils3d_shim, which provides the infer() path's two functions) so that the
UNMODIFIED reference `moge.test.metrics` imports and runs against it.  No reference test pins them, so parity at this boundary
is "unpinned" (DESIGN.md §2); the engine's resize kernel matches this restatement's fp32 arithmetic exactly.
"""
import math
import os
import sys

import torch

SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "utils3d_shim")


def sliding_window_2d(x, window_size, stride, dim=(-2, -1)):
    """Windows of x along two dims: the result has the windowed dims shrunk to (n - k) // s + 1 and the window offsets
    (k0, k1) appended last, so out[..., i, j, ..., a, b] = x[..., i * s0 + a, j * s1 + b, ...]."""
    ks = (window_size, window_size) if isinstance(window_size, int) else tuple(window_size)
    ss = (stride, stride) if isinstance(stride, int) else tuple(stride)
    for d, k, s in zip([d % x.dim() for d in dim], ks, ss):
        x = x.unfold(d, k, s)
    return x


def masked_nearest_resize(*image, mask, size, return_index=False):
    """Nearest resize of a masked map to size (h, w).  Target pixel (i, j) has centre ((j + 0.5) / w * W, (i + 0.5) / h * H) and a
    window of ceil(max(1, H / h)) x ceil(max(1, W / w)) source pixels whose top-left corner is the centre minus half the
    fractional window size, rounded half to even.  The output is the valid window pixel whose centre is nearest (fp32
    sqrt(dx * dx + dy * dy)), the first in row-major window order on a tie; the output mask is true when the window has a valid
    pixel.  Returns (*resized images, mask) and, with return_index, the index tuple (*batch indices, i, j) into the source."""
    H, W = mask.shape[-2:]
    th, tw = size
    dev = mask.device
    fh, fw = max(1, H / th), max(1, W / tw)
    fhi, fwi = math.ceil(fh), math.ceil(fw)
    cx = (torch.arange(tw, dtype=torch.float32, device=dev) + 0.5) / tw * W
    cy = (torch.arange(th, dtype=torch.float32, device=dev) + 0.5) / th * H
    left = torch.round(cx - torch.tensor(fw / 2, dtype=torch.float32, device=dev)).long()
    top = torch.round(cy - torch.tensor(fh / 2, dtype=torch.float32, device=dev)).long()
    rows = (top[:, None] + torch.arange(fhi, device=dev))[:, None, :, None].expand(th, tw, fhi, fwi)
    cols = (left[:, None] + torch.arange(fwi, device=dev))[None, :, None, :].expand(th, tw, fhi, fwi)
    inside = ((rows >= 0) & (rows < H) & (cols >= 0) & (cols < W)).reshape(th, tw, fhi * fwi)
    idx = torch.where(inside, (rows * W + cols).reshape(th, tw, fhi * fwi), 0)
    dx = (cols.float() + 0.5) - cx[None, :, None, None]
    dy = (rows.float() + 0.5) - cy[:, None, None, None]
    dist = torch.sqrt(dx * dx + dy * dy).reshape(th, tw, fhi * fwi)
    batch_shape = mask.shape[:-2]
    flat = mask.reshape(-1, H * W)
    win = flat[:, idx.reshape(-1)].reshape(-1, th, tw, fhi * fwi) & inside
    d = torch.where(win, dist, torch.inf)
    nearest = torch.argmin(d, dim=-1, keepdim=True)
    nidx = torch.gather(idx.expand_as(win), -1, nearest).squeeze(-1).reshape(*batch_shape, th, tw)
    lr_mask = win.any(dim=-1).reshape(*batch_shape, th, tw)
    batch_indices = [torch.arange(n, device=dev).reshape([1] * i + [n] + [1] * (len(batch_shape) - i - 1) + [1, 1])
                     for i, n in enumerate(batch_shape)]
    index = (*batch_indices, nidx // W, nidx % W)
    resized = tuple(x[index] for x in image)
    if return_index:
        return (*resized, lr_mask, index)
    return (*resized, lr_mask) if resized else lr_mask


def install():
    """Put the shim on sys.path, add the two functions to `utils3d.pt` (also reachable as `utils3d.torch`) and return it."""
    if SHIM not in sys.path:
        sys.path.append(SHIM)
    from utils3d import pt
    pt.sliding_window_2d = sliding_window_2d
    pt.masked_nearest_resize = masked_nearest_resize
    return pt
