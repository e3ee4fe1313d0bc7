"""The inference CLI's GPU work and its end-to-end rate.  Prints one JSON line with the GPU name and power limit read in the same run.

    python tools/bench_cli.py [--iters 50] [--images 32] [--out FILE]

- colour kernels: CUDA events around colorize_depth (quantile select + colouring) and colorize_normal, at 518 x 518, 1024 x 768
  and 2048 x 1365, batch 1 and 8 (median of `iters` timed calls after a warm-up), with the bytes each reads and writes over the
  3.35 TB/s data-sheet bandwidth of the H100 SXM; against the reference's host path (oracle/vis_port.py, np.nanquantile and the
  restated colour map) on one image, host clock;
- end to end: `infer` with --maps --glb --ply over a folder of `images` seeded synthetic 1024 x 768 JPEGs on a random-init
  MoGe-2 ViT-L checkpoint, images/s of the pipelined CLI against a sequential run of the reference script's steps (the same
  infer(), then the oracle colourisers and mesh on the host and the same writes).  The sequential run also gives the split of
  its time into the GPU's part (infer() to a synchronise) and the host's (colour, mesh and encoding), which says where the
  pipelined run is bound.
Everything is written under a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

os.environ['OPENCV_IO_ENABLE_OPENEXR'] = '1'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import cli, vis  # noqa: E402
from moge_b200.export import save_glb, save_ply  # noqa: E402
from oracle import utils3d_mesh, vis_port  # noqa: E402
from oracle.utils3d_panorama import intrinsics_to_fov  # noqa: E402

DEV = "cuda"
SIZES = [(518, 518), (768, 1024), (1365, 2048)]
HBM_BYTES_PER_S = 3.35e12
EXR = [cv2.IMWRITE_EXR_TYPE, cv2.IMWRITE_EXR_TYPE_FLOAT]
# A random-init model's depth is rough at the pixel scale: the default 4 % edge rule would remove the whole mesh.  With no edge
# cleaning the mesh covers the whole mask, the largest GLB / PLY a 1024 x 768 image gives.
THRESHOLD = float("inf")


def kernels(iters):
    rows = []
    g = torch.Generator(device="cpu").manual_seed(0)
    for H, W in SIZES:
        for B in (1, 8):
            depth = (torch.rand(B, H, W, generator=g) * 10 + 0.5).to(DEV)
            normal = torch.nn.functional.normalize(torch.randn(B, H, W, 3, generator=g), dim=-1).to(DEV)
            px = B * H * W
            t_depth = summary(cuda_samples(lambda: vis.colorize_depth(depth), iters))["median"]
            t_normal = summary(cuda_samples(lambda: vis.colorize_normal(normal), iters))["median"]
            # colorize_depth: 4 select passes + the colouring pass each read the depth; the colouring writes 3 bytes
            bytes_depth, bytes_normal = px * (5 * 4 + 3), px * (12 + 3)
            row = {"H": H, "W": W, "batch": B, "colorize_depth_ms": round(t_depth, 4), "colorize_normal_ms": round(t_normal, 4),
                   "colorize_depth_GBps": round(bytes_depth / t_depth / 1e6, 1), "colorize_normal_GBps": round(bytes_normal / t_normal / 1e6, 1),
                   "colorize_depth_share_of_hbm": round(bytes_depth / t_depth / 1e-3 / HBM_BYTES_PER_S, 3),
                   "colorize_normal_share_of_hbm": round(bytes_normal / t_normal / 1e-3 / HBM_BYTES_PER_S, 3)}
            if B == 1:
                d, n = depth[0].cpu().numpy(), normal[0].cpu().numpy()
                t0 = time.perf_counter()
                want = vis_port.colorize_depth(d)
                t1 = time.perf_counter()
                want_n = vis_port.colorize_normal(n)
                t2 = time.perf_counter()
                row.update(host_colorize_depth_ms=round((t1 - t0) * 1e3, 2), host_colorize_normal_ms=round((t2 - t1) * 1e3, 2),
                           bitwise_equal=bool(np.array_equal(vis.colorize_depth(depth[0]).cpu().numpy(), want)
                                              and np.array_equal(vis.colorize_normal(normal[0]).cpu().numpy(), want_n)))
            rows.append(row)
    return rows


def make_inputs(root: Path, n: int):
    from moge_b200.configs import model_config
    from moge_b200.synthetic import make_state_dict, synthetic_images
    cfg = model_config("vitl", True)
    torch.save({"model_config": cfg, "model": make_state_dict(cfg, 0, well_posed=True)}, root / "vitl.pt")
    (root / "in").mkdir()
    for i in range(n):
        img = (synthetic_images(1, 768, 1024, i)[0].permute(1, 2, 0) * 255).round().to(torch.uint8).numpy()
        cv2.imwrite(str(root / "in" / f"{i:03d}.jpg"), img)
    return root / "vitl.pt", root / "in"


def sequential(model, src: Path, out: Path):
    """The reference script's steps one after another; returns (seconds, GPU seconds, host seconds)."""
    gpu = host = 0.0
    t_start = time.perf_counter()
    for path in cli.list_images(src):
        image = cv2.cvtColor(cv2.imread(str(path)), cv2.COLOR_BGR2RGB)
        t0 = time.perf_counter()
        output = model.infer(torch.tensor(image / 255, dtype=torch.float32, device=DEV).permute(2, 0, 1), use_fp16=True)
        points, depth, mask, intrinsics, normal = (output[k].cpu().numpy() for k in ("points", "depth", "mask", "intrinsics", "normal"))
        t1 = time.perf_counter()
        p = out / path.stem
        p.mkdir(parents=True, exist_ok=True)
        with np.errstate(divide="ignore", invalid="ignore"):
            cv2.imwrite(str(p / 'image.jpg'), cv2.cvtColor(image, cv2.COLOR_RGB2BGR))
            cv2.imwrite(str(p / 'depth_vis.png'), cv2.cvtColor(vis_port.colorize_depth(depth), cv2.COLOR_RGB2BGR))
            cv2.imwrite(str(p / 'depth.exr'), depth, EXR)
            cv2.imwrite(str(p / 'mask.png'), (mask * 255).astype(np.uint8))
            cv2.imwrite(str(p / 'points.exr'), cv2.cvtColor(points, cv2.COLOR_RGB2BGR), EXR)
            cv2.imwrite(str(p / 'normal.png'), cv2.cvtColor(vis_port.colorize_normal(normal), cv2.COLOR_RGB2BGR))
            fx, fy = intrinsics_to_fov(intrinsics)
            with open(p / 'fov.json', 'w') as f:
                json.dump({'fov_x': round(float(np.rad2deg(fx)), 2), 'fov_y': round(float(np.rad2deg(fy)), 2)}, f)
            mesh = utils3d_mesh.mesh_from_output(points, depth, mask, image, normal, threshold=THRESHOLD)
        save_glb(p / 'mesh.glb', mesh["vertices"], mesh["faces"], mesh["vertex_uvs"], image, mesh["vertex_normals"])
        save_ply(p / 'pointcloud.ply', mesh["vertices"], np.zeros((0, 3), dtype=np.int32), mesh["vertex_colors"], mesh["vertex_normals"])
        t2 = time.perf_counter()
        gpu += t1 - t0
        host += t2 - t1
    return time.perf_counter() - t_start, gpu, host


def end_to_end(n: int):
    from moge.model.v2 import MoGeModel
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        ckpt, src = make_inputs(root, n)
        args = dict(input_path=str(src), fov_x_=None, pretrained=str(ckpt), model_version="v2", device_name="cuda", use_fp16=False,
                    resize_to=None, resolution_level=9, num_tokens=None, threshold=THRESHOLD, save_maps_=True, save_glb_=True, save_ply_=True,
                    show=False)
        cli.run_infer(output_path=str(root / "warm"), **args)                 # warm-up: library, shapes, allocator
        model = MoGeModel.from_pretrained(str(ckpt)).to(DEV).eval()
        sequential(model, src, root / "seq_warm")
        runs = []
        for r in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cli.run_infer(output_path=str(root / f"cli{r}"), **args)
            runs.append(time.perf_counter() - t0)
            seq = sequential(model, src, root / f"seq{r}")
            runs.append(seq)
        cli_s = min(runs[0], runs[2])
        seq_s = min(runs[1], runs[3], key=lambda x: x[0])
        return {"images": n, "size": "1024x768", "model": "MoGe-2 ViT-L random init", "flags": "--maps --glb --ply --threshold inf",
                "cli_images_per_s": round(n / cli_s, 2), "sequential_images_per_s": round(n / seq_s[0], 2),
                "speedup": round(seq_s[0] / cli_s, 2),
                "sequential_gpu_s_per_image": round(seq_s[1] / n, 4), "sequential_host_s_per_image": round(seq_s[2] / n, 4),
                "cli_s_per_image": round(cli_s / n, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"bench": "cli", **gpu_identity(), "kernels": kernels(a.iters), "end_to_end": end_to_end(a.images)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
