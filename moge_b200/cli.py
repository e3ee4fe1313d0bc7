"""The work behind `moge infer` and `moge infer_panorama` (moge/scripts): the reference's scripts (moge/scripts/infer.py,
moge/scripts/infer_panorama.py) with the colourisation and the mesh export on the GPU, writing the same files in the same
layout.

The reference handles one image after another, and the GPU idles while the host encodes.  Here the stages overlap:
- a reader thread decodes (cv2) and resizes the next images while the GPU works on the current one;
- per image, the GPU runs infer(), the colour kernels (moge_b200.vis) and the mesh export (moge_b200.mesh); every map is
  assembled in one device buffer and copied once into pinned host memory, and the mesh arrays follow it on the same stream;
- a small pool of host threads waits for that copy and encodes the files (cv2 releases the GIL while it encodes);
- at most WRITERS + 1 images are in flight, which bounds the pinned memory, and a writer's error is raised in the main thread.
Per image, the main thread waits on the host only inside the mesh call (for its counts).  The files do not depend on the
pipelining: every value is computed by the same calls in the same order.
"""
from __future__ import annotations

import os
os.environ['OPENCV_IO_ENABLE_OPENEXR'] = '1'          # before cv2 is imported, as the reference's scripts do

import itertools
import json
import warnings
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

INCLUDE_SUFFIXES = ['jpg', 'png', 'jpeg', 'JPG', 'PNG', 'JPEG']
DEFAULT_PRETRAINED = {"v1": "Ruicheng/moge-vitl", "v2": "Ruicheng/moge-2-vitl-normal"}
PANORAMA_PRETRAINED = "Ruicheng/moge-vitl"
MAP_FILES = ('image.jpg', 'depth_vis.png', 'depth.exr', 'mask.png', 'points.exr')
WRITERS = 4                                          # host encoding threads
PREFETCH = 2                                         # images decoded ahead of the GPU


class UsageError(ValueError):
    """An option this implementation does not provide (the click commands turn it into a usage error)."""


# ------------------------------------------------------------------------------------------------------------ planning
def list_images(input_path) -> List[Path]:
    """The reference's image list: sorted rglob over the six suffixes for a folder, the path itself for a file."""
    if Path(input_path).is_dir():
        paths = sorted(itertools.chain(*(Path(input_path).rglob(f'*.{suffix}') for suffix in INCLUDE_SUFFIXES)))
    else:
        paths = [Path(input_path)]
    if len(paths) == 0:
        raise FileNotFoundError(f'No image files found in {input_path}')
    return paths


def save_dir(output_path, input_path, image_path: Path) -> Path:
    """output / image_path.relative_to(input).parent / stem (for a single file: output / stem)."""
    return Path(output_path, Path(image_path).relative_to(input_path).parent, Path(image_path).stem)


def resized_size(height: int, width: int, resize_to: Optional[int]) -> Tuple[int, int]:
    """The reference's --resize rule: the longer side becomes resize_to, the other is truncated."""
    if resize_to is None:
        return height, width
    return min(resize_to, int(resize_to * height / width)), min(resize_to, int(resize_to * width / height))


def output_files(save_maps: bool, save_glb: bool, save_ply: bool, normal: bool) -> List[str]:
    """The files `infer` writes into an image's folder."""
    files = (list(MAP_FILES) + (['normal.png'] if normal else []) + ['fov.json']) if save_maps else []
    return files + (['mesh.glb'] if save_glb else []) + (['pointcloud.ply'] if save_ply else [])


def fov_json(intrinsics: np.ndarray) -> Dict[str, float]:
    """fov.json: utils3d's intrinsics_to_fov (2 arctan(0.5 / f)) on the fp32 intrinsics, in degrees, rounded to 2 places."""
    fov_x, fov_y = 2 * np.arctan(0.5 / intrinsics[..., 0, 0]), 2 * np.arctan(0.5 / intrinsics[..., 1, 1])
    return {'fov_x': round(float(np.rad2deg(fov_x)), 2), 'fov_y': round(float(np.rad2deg(fov_y)), 2)}


def formats(save_maps: bool, save_glb: bool, save_ply: bool) -> Tuple[bool, bool, bool]:
    if not any([save_maps, save_glb, save_ply]):
        warnings.warn('No output format specified. Defaults to saving all. Please use "--maps", "--glb", or "--ply" to specify the output.')
        return True, True, True
    return save_maps, save_glb, save_ply


def check_options(device_name: str, show: bool):
    """The device (a CUDA device: the engine has no CPU path) and no --show (no trimesh viewer)."""
    import torch
    if show:
        raise UsageError('--show is not provided: it needs trimesh and a window; write the mesh with --glb or --ply instead')
    try:
        device = torch.device(device_name)
    except RuntimeError as e:
        raise UsageError(f'--device {device_name}: {e}')
    if device.type != 'cuda':
        raise UsageError(f'--device {device_name}: moge_b200 runs on CUDA devices only (there is no CPU path)')
    return device


def read_image(path: Path, resize_to: Optional[int]) -> np.ndarray:
    """The reference's decode: cv2.imread, BGR -> RGB, and with --resize cv2.resize(image, (w, h), cv2.INTER_AREA), which passes
    INTER_AREA as `dst` and so interpolates bilinearly, as the reference does."""
    import cv2
    image = cv2.cvtColor(cv2.imread(str(path)), cv2.COLOR_BGR2RGB)
    height, width = image.shape[:2]
    if resize_to is not None:
        height, width = resized_size(height, width, resize_to)
        image = cv2.resize(image, (width, height), cv2.INTER_AREA)
    return image


# ------------------------------------------------------------------------------------------------------------ pipeline
class _Reader:
    """Decodes images on a thread, PREFETCH ahead; yields (path, uint8 RGB image, pinned fp32 image / 255 or None)."""

    def __init__(self, paths: Sequence[Path], resize_to: Optional[int], unit_float: bool = True):
        self.pool = ThreadPoolExecutor(1)
        self.paths, self.resize_to, self.unit_float = list(paths), resize_to, unit_float

    def _load(self, path: Path):
        import torch
        if not path.exists():
            raise FileNotFoundError(f'File {path} does not exist.')
        image = read_image(path, self.resize_to)
        # torch.tensor(image / 255, dtype=torch.float32): divided in float64, then rounded to fp32
        if not self.unit_float:
            return path, image, None
        return path, image, torch.from_numpy((image / 255).astype(np.float32)).pin_memory()

    def __iter__(self):
        ahead = deque(self.pool.submit(self._load, p) for p in self.paths[:PREFETCH])
        nxt = PREFETCH
        try:
            while ahead:
                item = ahead.popleft().result()
                if nxt < len(self.paths):
                    ahead.append(self.pool.submit(self._load, self.paths[nxt]))
                    nxt += 1
                yield item
        finally:
            for f in ahead:
                f.cancel()
            self.pool.shutdown(wait=True)


class _Writers:
    """A bounded pool of encoding threads.  Each image's jobs first wait for its copy event; at most WRITERS + 1 images are in
    flight; a job's exception is re-raised in the main thread."""

    def __init__(self):
        self.pool = ThreadPoolExecutor(WRITERS)
        self.inflight = deque()

    def _drain_one(self):
        for f in self.inflight.popleft():
            f.result()

    def submit(self, event, jobs: List[Callable[[], None]]):
        while len(self.inflight) > WRITERS:
            self._drain_one()

        def run(job):
            event.synchronize()
            job()
        self.inflight.append([self.pool.submit(run, j) for j in jobs])

    def close(self, ok: bool = True):
        try:
            while ok and self.inflight:
                self._drain_one()
        finally:
            self.pool.shutdown(wait=True, cancel_futures=not ok)


def _stage(device, specs) -> Dict[str, np.ndarray]:
    """Assemble maps in one device buffer and copy it once into pinned host memory (asynchronously).  specs: (name, shape, torch
    dtype, fill) with fill(view) writing the device view.  Returns numpy views of the pinned buffer, valid after the copy."""
    import torch
    offsets, total = [], 0
    for _, shape, dtype, _ in specs:
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        offsets.append((total, n))
        total += (n + 255) // 256 * 256
    dev = torch.empty(max(total, 256), dtype=torch.uint8, device=device)
    for (name, shape, dtype, fill), (off, n) in zip(specs, offsets):
        fill(dev[off:off + n].view(dtype).view(shape))
    host = torch.empty(dev.shape, dtype=torch.uint8, pin_memory=True)
    host.copy_(dev, non_blocking=True)
    return {name: host[off:off + n].view(dtype).view(shape).numpy() for (name, shape, dtype, _), (off, n) in zip(specs, offsets)}


def _pinned(t) -> np.ndarray:
    import torch
    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    h.copy_(t, non_blocking=True)
    return h.numpy()


def _copy(t) -> Callable:
    return lambda v: v.copy_(t)


def _imwrite(path: Path, image: np.ndarray, params=None) -> None:
    import cv2
    if not cv2.imwrite(str(path), image, *([params] if params else [])):
        raise OSError(f'cv2.imwrite could not write {path}')


def _exr_params():
    import cv2
    return [cv2.IMWRITE_EXR_TYPE, cv2.IMWRITE_EXR_TYPE_FLOAT]


def _rgb2bgr(x: np.ndarray) -> np.ndarray:
    import cv2
    return cv2.cvtColor(x, cv2.COLOR_RGB2BGR)


def _write_json(path: Path, obj) -> None:
    with open(path, 'w') as f:
        json.dump(obj, f)


def _load_model(version: str, pretrained: Optional[str], device, use_fp16: bool):
    if pretrained is None:
        pretrained = DEFAULT_PRETRAINED[version]
    if version == 'v1':
        from moge.model.v1 import MoGeModel
    else:
        from moge.model import import_model_class_by_version
        MoGeModel = import_model_class_by_version(version)
    model = MoGeModel.from_pretrained(pretrained).to(device).eval()
    if use_fp16:
        model.half()
    return model


# ------------------------------------------------------------------------------------------------------------ infer
def run_infer(input_path, fov_x_: Optional[float], output_path, pretrained: Optional[str], model_version: str, device_name: str,
              use_fp16: bool, resize_to: Optional[int], resolution_level: int, num_tokens: Optional[int], threshold: float,
              save_maps_: bool, save_glb_: bool, save_ply_: bool, show: bool) -> None:
    """moge/scripts/infer.py: for every image, infer() and the selected files under save_dir(output, input, image).  The engine
    has no fp32 network pass, so infer() always runs with use_fp16=True; --fp16 also casts the model with .half()."""
    device = check_options(device_name, show)
    import torch
    from . import vis
    from .export import save_glb, save_ply
    from .mesh import mesh_from_output

    image_paths = list_images(input_path)
    model = _load_model(model_version, pretrained, device, use_fp16)
    save_maps_, save_glb_, save_ply_ = formats(save_maps_, save_glb_, save_ply_)
    writers = _Writers()
    ok = False
    try:
        with torch.cuda.device(device):
            for image_path, image, image_f32 in _Reader(image_paths, resize_to):
                height, width = image.shape[:2]
                image_tensor = image_f32.to(device, non_blocking=True).permute(2, 0, 1)
                output = model.infer(image_tensor, fov_x=fov_x_, resolution_level=resolution_level, num_tokens=num_tokens,
                                     use_fp16=True)
                normal = output.get('normal')
                save_path = save_dir(output_path, input_path, image_path)
                save_path.mkdir(exist_ok=True, parents=True)
                jobs = []
                if save_maps_:
                    specs = [('depth', (height, width), torch.float32, _copy(output['depth'])),
                             ('points', (height, width, 3), torch.float32, _copy(output['points'])),
                             ('mask', (height, width), torch.bool, _copy(output['mask'])),
                             ('intrinsics', (3, 3), torch.float32, _copy(output['intrinsics'])),
                             ('depth_vis', (height, width, 3), torch.uint8, lambda v: vis.colorize_depth(output['depth'], bgr=True, out=v))]
                    if normal is not None:
                        specs.append(('normal_vis', (height, width, 3), torch.uint8, lambda v: vis.colorize_normal(normal, bgr=True, out=v)))
                    maps = _stage(device, specs)
                    jobs += [lambda p=save_path, im=image: _imwrite(p / 'image.jpg', _rgb2bgr(im)),
                             lambda p=save_path, m=maps: _imwrite(p / 'depth_vis.png', m['depth_vis']),
                             lambda p=save_path, m=maps: _imwrite(p / 'depth.exr', m['depth'], _exr_params()),
                             lambda p=save_path, m=maps: _imwrite(p / 'mask.png', (m['mask'] * 255).astype(np.uint8)),
                             lambda p=save_path, m=maps: _imwrite(p / 'points.exr', _rgb2bgr(m['points']), _exr_params()),
                             lambda p=save_path, m=maps: _write_json(p / 'fov.json', fov_json(m['intrinsics']))]
                    if normal is not None:
                        jobs.append(lambda p=save_path, m=maps: _imwrite(p / 'normal.png', m['normal_vis']))
                if save_glb_ or save_ply_:
                    image_u8 = torch.from_numpy(image).pin_memory().to(device, non_blocking=True)
                    mesh = {k: _pinned(v) for k, v in mesh_from_output(output, image_u8, threshold).items() if k != 'mask_cleaned'}
                    if save_glb_:
                        jobs.append(lambda p=save_path, m=mesh, im=image: save_glb(p / 'mesh.glb', m['vertices'], m['faces'], m['vertex_uvs'], im,
                                                                                    m.get('vertex_normals')))
                    if save_ply_:
                        jobs.append(lambda p=save_path, m=mesh: save_ply(p / 'pointcloud.ply', m['vertices'], np.zeros((0, 3), dtype=np.int32),
                                                                         m['vertex_colors'], m.get('vertex_normals')))
                event = torch.cuda.Event()
                event.record()
                writers.submit(event, jobs)
        ok = True
    finally:
        writers.close(ok)


# ------------------------------------------------------------------------------------------------------------ infer_panorama
def run_infer_panorama(input_path, output_path, pretrained: str, device_name: str, resize_to: Optional[int], resolution_level: int,
                       threshold: float, batch_size: int, save_splitted: bool, save_maps_: bool, save_glb_: bool, save_ply_: bool,
                       show: bool) -> None:
    """moge/scripts/infer_panorama.py: for every panorama, moge_b200.panorama.infer_panorama with a MoGe-1 model and the selected
    files.  --resolution_level is accepted and, as in the reference, not used by the panorama pass."""
    device = check_options(device_name, show)
    import torch
    from . import vis
    from .export import save_glb, save_ply
    from .mesh import mesh_from_panorama
    from .panorama import infer_panorama
    from moge.model.v1 import MoGeModel

    image_paths = list_images(input_path)
    save_maps_, save_glb_, save_ply_ = formats(save_maps_, save_glb_, save_ply_)
    model = MoGeModel.from_pretrained(pretrained).to(device).eval()
    writers = _Writers()
    ok = False
    try:
        with torch.cuda.device(device):
            for image_path, image, _ in _Reader(image_paths, resize_to, unit_float=False):
                height, width = image.shape[:2]
                image_u8 = torch.from_numpy(image).pin_memory().to(device, non_blocking=True)
                out = infer_panorama(model, image_u8, batch_size=batch_size, return_views=save_splitted)
                jobs = []
                specs = []
                if save_splitted:
                    n, res = out['views'].shape[:2]
                    specs += [('views', (n, res, res, 3), torch.uint8, _copy(out['views'])),
                              ('views_vis', (n, res, res, 3), torch.uint8,
                               lambda v: vis.colorize_depth(out['view_distance'], out['view_mask'], bgr=True, out=v))]
                if save_maps_:
                    specs += [('depth', (height, width), torch.float32, _copy(out['depth'])),
                              ('points', (height, width, 3), torch.float32, _copy(out['points'])),
                              ('mask', (height, width), torch.bool, _copy(out['mask'])),
                              ('depth_vis', (height, width, 3), torch.uint8,
                               lambda v: vis.colorize_depth(out['depth'], mask=out['mask'], bgr=True, out=v))]
                maps = _stage(device, specs) if specs else {}
                if save_splitted:
                    split_path = Path(output_path, image_path.stem, 'splitted')
                    split_path.mkdir(exist_ok=True, parents=True)
                    for i in range(maps['views'].shape[0]):
                        jobs += [lambda p=split_path / f'{i:02d}.jpg', m=maps, i=i: _imwrite(p, _rgb2bgr(m['views'][i])),
                                 lambda p=split_path / f'{i:02d}_distance_vis.png', m=maps, i=i: _imwrite(p, m['views_vis'][i])]
                save_path = save_dir(output_path, input_path, image_path)
                save_path.mkdir(exist_ok=True, parents=True)
                if save_maps_:
                    jobs += [lambda p=save_path, im=image: _imwrite(p / 'image.jpg', _rgb2bgr(im)),
                             lambda p=save_path, m=maps: _imwrite(p / 'depth_vis.png', m['depth_vis']),
                             lambda p=save_path, m=maps: _imwrite(p / 'depth.exr', m['depth'], _exr_params()),
                             lambda p=save_path, m=maps: _imwrite(p / 'points.exr', m['points'], _exr_params()),
                             lambda p=save_path, m=maps: _imwrite(p / 'mask.png', (m['mask'] * 255).astype(np.uint8))]
                if save_glb_ or save_ply_:
                    mesh = {k: _pinned(v) for k, v in mesh_from_panorama(out, image_u8, threshold).items() if k != 'mask_cleaned'}
                    if save_glb_:
                        jobs.append(lambda p=save_path, m=mesh, im=image: save_glb(p / 'mesh.glb', m['vertices'], m['faces'], m['vertex_uvs'], im))
                    if save_ply_:
                        jobs.append(lambda p=save_path, m=mesh: save_ply(p / 'mesh.ply', m['vertices'], m['faces'], m['vertex_colors']))
                event = torch.cuda.Event()
                event.record()
                writers.submit(event, jobs)
        ok = True
    finally:
        writers.close(ok)
