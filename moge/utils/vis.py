"""Drop-in for the reference's `moge.utils.vis`: `colorize_depth`, `colorize_depth_affine`, `colorize_disparity` and
`colorize_normal` with the reference's signatures and numpy returns, computed on the current CUDA device (moge_b200.vis) and
bitwise equal to the reference's for float32 inputs (other float inputs are taken as float32).  The quantiles are taken over
the whole array, as np.nanquantile does.  Only the "Spectral" colour map is provided; any other `cmap` raises.

`colorize_segmentation` and `colorize_error_map` are not provided: they need matplotlib's "Set1" and "plasma" tables, which are
not restated here and could not be checked without matplotlib.
"""
import numpy as np
import torch

from moge_b200 import vis as _vis

__all__ = ["colorize_depth", "colorize_depth_affine", "colorize_disparity", "colorize_normal"]


def _device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


def _flat(x: np.ndarray, channels: int = 0) -> torch.Tensor:
    """The array as one (1, rows, columns[, C]) fp32 image on the device: the quantiles cover all of it."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    shape = x.shape[:-1] if channels else x.shape
    w = shape[-1] if len(shape) else 1
    return torch.from_numpy(x.reshape(1, -1, w, *([channels] if channels else []))).to(_device())


def _mask(mask, like: torch.Tensor):
    return None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=bool)).to(like.device).reshape(like.shape[:3])


def _shape(x: np.ndarray, channels: int = 0):
    return (x.shape[:-1] if channels else np.shape(x)) + (3,)


def colorize_depth(depth: np.ndarray, mask: np.ndarray = None, normalize: bool = True, cmap: str = 'Spectral') -> np.ndarray:
    d = _flat(depth)
    return _vis.colorize_depth(d, _mask(mask, d), normalize, cmap).cpu().numpy().reshape(_shape(depth))


def colorize_depth_affine(depth: np.ndarray, mask: np.ndarray = None, cmap: str = 'Spectral') -> np.ndarray:
    d = _flat(depth)
    return _vis.colorize_depth_affine(d, _mask(mask, d), cmap).cpu().numpy().reshape(_shape(depth))


def colorize_disparity(disparity: np.ndarray, mask: np.ndarray = None, normalize: bool = True, cmap: str = 'Spectral') -> np.ndarray:
    d = _flat(disparity)
    return _vis.colorize_disparity(d, _mask(mask, d), normalize, cmap).cpu().numpy().reshape(_shape(disparity))


def colorize_normal(normal: np.ndarray, mask: np.ndarray = None) -> np.ndarray:
    n = _flat(normal, channels=3)
    return _vis.colorize_normal(n, _mask(mask, n)).cpu().numpy().reshape(_shape(normal, channels=3))
