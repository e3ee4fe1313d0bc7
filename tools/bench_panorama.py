"""Panorama inference on the H100: per-stage device times of infer_panorama and the host comparator (the reference's cv2 split
and SciPy-LSMR merge on the same engine views), with output agreement.  Prints one JSON line (profiles/h100_bench_panorama.json).

    python tools/bench_panorama.py [--steps 3] [--out FILE]

Workloads: 2048 x 1024 and 4096 x 2048 synthetic panoramas through a synthetic-weight ViT-L MoGe-1 at resolution level 9, and
the merge alone at 1920 x 960 on the distance maps of an analytic box room (synthetic weights give views with no geometry, so
their LSMR iteration counts say little; the room's do).  The comparator runs when build() compiled the reference module into
oracle/_ref/ and cv2 / SciPy are installed; otherwise its numbers are "not measured".
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_panorama_batch import merge_levels  # noqa: E402
from measure import cuda_samples, gpu_identity  # noqa: E402
from moge_b200 import panorama as P  # noqa: E402
from moge_b200.synthetic import synthetic_panorama, synthetic_room_views  # noqa: E402

DEV = "cuda:0"


class Timer:
    def __init__(self):
        self.ev = []

    def mark(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.ev.append((name, e))

    def result(self):
        torch.cuda.synchronize()
        return {self.ev[k][0]: self.ev[k - 1][1].elapsed_time(self.ev[k][1]) for k in range(1, len(self.ev))}


def staged(model, image):
    """infer_panorama's stages with events between them: (stage ms, merge per-level ms, outputs)."""
    H, W = image.shape[:2]
    extr, intr = P._default_cameras()
    t = Timer()
    t.mark("start")
    views = P.split_panorama(image, extr, intr)
    t.mark("split")
    out = model.infer(views, fov_x=P._fov_x(intr, image.device), apply_mask=False)
    t.mark("infer")
    depth, mask, levels = P.merge_panorama(min(1920, W), min(960, H), out["points"], out["mask"], extr, intr, return_levels=True)
    t.mark("merge")
    d, m, pts = P.finish_panorama(depth, mask, H, W)
    t.mark("finish")
    return t.result(), (d, m, pts), out


def merge_levels_ms(src, mask, width, height, extr, intr):
    """The merge of one panorama alone, src (N, vh, vw[, 3]) and mask (N, vh, vw): per level its size, the ms of its right-hand
    side and of its LSMR solve, its iteration count and istop."""
    return [{**lv, "rhs_ms": round(lv["rhs_ms"], 3), "lsmr_ms": round(lv["lsmr_ms"], 3), "iterations": lv["iterations"][0],
             "istop": lv["istop"][0]} for lv in merge_levels(src[None], mask[None], width, height, extr, intr)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    gpu = gpu_identity()
    from oracle.compile_reference import load_panorama
    ref = None if args.no_reference else load_panorama()
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vitl")
    model = MoGeModel(**cfg)
    model.load_state_dict(make_v1_state_dict(cfg, 30, well_posed=True))
    model = model.to(DEV).eval()
    result = {**gpu, "model": "MoGe-1 ViT-L (synthetic weights), resolution level 9", "workloads": []}
    for H, W in ((1024, 2048), (2048, 4096)):
        img = torch.from_numpy(synthetic_panorama(H, W, 1))
        dimg = img.to(DEV)
        P.infer_panorama(model, dimg)                     # warm-up: tables, engine plans
        torch.cuda.synchronize()
        runs = []
        for _ in range(args.steps):
            runs.append(staged(model, dimg)[0])
        stage = {k: round(float(np.median([r[k] for r in runs])), 3) for k in runs[0]}
        e2e = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            o = P.infer_panorama(model, dimg)
            host = {k: v.cpu() for k, v in o.items()}
            e2e.append((time.perf_counter() - t0) * 1e3)
        _, (d, m, pts), views_out = staged(model, dimg)
        levels = merge_levels_ms(views_out["points"], views_out["mask"], min(1920, W), min(960, H), *P._default_cameras())
        wl = {"panorama": f"{W}x{H}", "stage_ms": stage, "merge_levels": levels, "end_to_end_ms_host_results": round(float(np.median(e2e)), 2)}
        if ref is not None and W == 2048:
            import cv2
            extr, intr = ref.get_panorama_cameras()
            t0 = time.perf_counter()
            views = ref.split_panorama_image(img.numpy(), extr, intr, 512)
            t1 = time.perf_counter()
            tv = torch.tensor(np.stack(views) / 255, dtype=torch.float32, device=DEV).permute(0, 3, 1, 2)
            o = model.infer(tv, fov_x=P._fov_x(intr, DEV), apply_mask=False)
            dist, msk = o["points"].norm(dim=-1).cpu().numpy(), o["mask"].cpu().numpy()
            t2 = time.perf_counter()
            rd, rm = ref.merge_panorama_depth(min(1920, W), min(960, H), list(dist), list(msk), extr, intr)
            t3 = time.perf_counter()
            rd = cv2.resize(rd.astype(np.float32), (W, H), cv2.INTER_LINEAR)
            rm = cv2.resize(rm.astype(np.uint8), (W, H), cv2.INTER_NEAREST) > 0
            t4 = time.perf_counter()
            split_eq = bool(np.array_equal(np.stack(views), P.split_panorama(dimg, return_uint8=True)[1].cpu().numpy()))
            rel = np.abs(host["depth"].numpy().astype(np.float64) / rd - 1)
            wl["reference_host_ms"] = {"split": round((t1 - t0) * 1e3, 1), "merge": round((t3 - t2) * 1e3, 1),
                                       "finish": round((t4 - t3) * 1e3, 1)}
            wl["agreement"] = {"split_bitwise": split_eq, "depth_rel_median": float(np.median(rel)), "depth_rel_max": float(rel.max()),
                               "mask_mismatch": int((host["mask"].numpy() != rm).sum())}
        else:
            wl["reference_host_ms"] = "not measured"
        result["workloads"].append(wl)
        print(json.dumps(wl), flush=True)
    dist, masks = synthetic_room_views(512)
    extr, intr = P.get_panorama_cameras()
    src, msk = torch.from_numpy(dist).to(DEV), torch.from_numpy(masks).to(DEV)
    dep, pm = P.merge_panorama(1920, 960, src, msk, extr, intr)        # warm-up; the merge is repeatable, so also the result
    room = {"merge": "room 1920x960 from 12 x 512^2 distance maps", "levels": merge_levels_ms(src, msk, 1920, 960, extr, intr)}
    t = cuda_samples(lambda: P.merge_panorama(1920, 960, src, msk, extr, intr), args.steps, warmup=0)
    room["merge_ms"] = round(float(np.median(t)), 2)
    if ref is not None:
        t0 = time.perf_counter()
        rd, rmask = ref.merge_panorama_depth(1920, 960, list(dist), list(masks), extr, intr)
        room["reference_host_merge_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        rel = np.abs(dep.cpu().numpy().astype(np.float64) / rd - 1)
        room["agreement"] = {"depth_rel_median": float(np.median(rel)), "depth_rel_max": float(rel.max()),
                             "mask_equal": bool(np.array_equal(pm.cpu().numpy(), rmask))}
    else:
        room["reference_host_merge_ms"] = "not measured"
    result["workloads"].append(room)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
