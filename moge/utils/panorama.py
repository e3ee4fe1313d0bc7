"""Drop-in for the reference's `moge.utils.panorama`: the functions its callers use, with the reference's signatures and numpy
returns.  `split_panorama_image` and `merge_panorama_depth` run on the current CUDA device (moge_b200.panorama).  The SciPy sparse
builders `poisson_equation` and `grad_equation` are not provided: the solver applies the same system as stencils."""
from typing import List

import numpy as np
import torch

from moge_b200.panorama import directions_to_spherical_uv, get_panorama_cameras, spherical_uv_to_directions  # noqa: F401
from moge_b200 import panorama as _pano

__all__ = ["get_panorama_cameras", "spherical_uv_to_directions", "directions_to_spherical_uv", "split_panorama_image",
           "merge_panorama_depth"]


def _device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


def split_panorama_image(image: np.ndarray, extrinsics: np.ndarray, intrinsics: np.ndarray, resolution: int) -> List[np.ndarray]:
    """The views (resolution, resolution, 3) uint8 of an (H, W, 3) uint8 panorama, one per camera."""
    img = torch.from_numpy(np.ascontiguousarray(image, dtype=np.uint8)).to(_device())
    _, views = _pano.split_panorama(img, extrinsics, intrinsics, resolution, return_uint8=True)
    return list(views.cpu().numpy())


def merge_panorama_depth(width: int, height: int, distance_maps: List[np.ndarray], pred_masks: List[np.ndarray],
                         extrinsics: List[np.ndarray], intrinsics: List[np.ndarray]):
    """(depth (height, width) float32, mask (height, width) bool) merged from per-view distance maps and masks."""
    dev = _device()
    dist = torch.from_numpy(np.ascontiguousarray(np.stack(distance_maps), dtype=np.float32)).to(dev)
    mask = torch.from_numpy(np.ascontiguousarray(np.stack(pred_masks)).astype(bool)).to(dev)
    depth, pmask = _pano.merge_panorama(width, height, dist, mask, extrinsics, intrinsics)
    return depth.cpu().numpy(), pmask.cpu().numpy()
