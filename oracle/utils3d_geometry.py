"""The utils3d functions that the reference's `moge/utils/geometry_torch.py` calls: `sliding_window` (dilate_with_mask,
refine_depth_with_normal), `sliding_window_2d` (refine_depth_with_normal) and `uv_map` (refine_depth_with_normal), restated
from utils3d's published semantics.  TEST INFRASTRUCTURE ONLY.

`install()` adds them to the utils3d stand-in (oracle/utils3d_shim) so that the UNMODIFIED reference module imports and runs
against it; `load_geometry()` returns the module compiled by oracle/compile_reference.py, the comparator of
tools/bench_geometry.py.  No reference test pins these functions, so parity at this boundary is "unpinned" (DESIGN.md §2):
  - sliding_window(x, window_size, stride, dim): windows of x along the dims `dim`, each windowed dim shrunk to
    (n - k) // s + 1 and the window offsets appended last in the order of `dim` (torch.Tensor.unfold per dim; a view);
  - sliding_window_2d: the same over two dims (oracle/utils3d_metrics.py);
  - uv_map((height, width), dtype, device): (height, width, 2) pixel-centre UV, u = (j + 0.5) / width, v = (i + 0.5) / height
    (the convention of the stand-in's depth_map_to_point_map).
"""
import torch

from oracle import compile_reference
from oracle.utils3d_metrics import install as _install_metrics
from oracle.utils3d_metrics import sliding_window_2d  # noqa: F401


def sliding_window(x, window_size, stride=1, dim=None):
    dims = tuple(range(x.dim())) if dim is None else ((dim,) if isinstance(dim, int) else tuple(dim))
    n = len(dims)
    ks = (window_size,) * n if isinstance(window_size, int) else tuple(window_size)
    ss = (stride,) * n if isinstance(stride, int) else tuple(stride)
    for d, k, s in zip([d % x.dim() for d in dims], ks, ss):
        x = x.unfold(d, k, s)
    return x


def uv_map(*size, dtype=None, device=None):
    height, width = size[0] if len(size) == 1 else size
    u = (torch.arange(width, dtype=dtype or torch.float32, device=device) + 0.5) / width
    v = (torch.arange(height, dtype=dtype or torch.float32, device=device) + 0.5) / height
    return torch.stack(torch.meshgrid(u, v, indexing="xy"), dim=-1)


def install():
    """Put the shim on sys.path (with utils3d_metrics' functions) and add these three to `utils3d.pt`; returns it."""
    pt = _install_metrics()
    pt.sliding_window = sliding_window
    pt.uv_map = uv_map
    return pt


def load_geometry():
    """The reference's `moge.utils.geometry_torch` compiled into oracle/_ref, or None when it was not built."""
    return compile_reference._load("utils/geometry_torch", "utils3d_geometry")
