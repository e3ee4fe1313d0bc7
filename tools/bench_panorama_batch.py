"""Batched panorama inference on the H100: infer_panoramas over P panoramas against P infer_panorama calls, per-panorama stage
times, and the merge's per-level solve times and LSMR iterations.  Prints one JSON line (profiles/h100_bench_panorama_batch.json).

    python tools/bench_panorama_batch.py [--steps 5] [--batches 1 2 4 8] [--out FILE]

Workload: 2048 x 1024 synthetic panoramas (seeds 1..P) through a synthetic-weight ViT-L MoGe-1 at resolution level 9, as
tools/bench_panorama.py.  Per P: the stages between CUDA events (split, the 12P views' infer, merge, finish), each level's
solve (one event pair around its right-hand side and one around its cooperative LSMR launch), and the end-to-end time with the
results copied to the host, infer_panoramas alternated with P infer_panorama calls.  Times are the median, min and max of
--steps runs.
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

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import capi  # noqa: E402
from moge_b200 import panorama as P  # noqa: E402
from moge_b200.synthetic import synthetic_panorama  # noqa: E402

DEV = "cuda:0"


def events(n):
    return [torch.cuda.Event(enable_timing=True) for _ in range(n)]


def staged(model, images):
    """infer_panoramas' stages between events: ({stage: ms for the whole batch}, the views' points and mask, last_merge_stats())."""
    ev = events(5)
    extr, intr = P._default_cameras()
    B, H, W = images.shape[:3]
    ev[0].record()
    views = P.split_panoramas(images, extr, intr)
    ev[1].record()
    out = model.infer(views.view(-1, *views.shape[2:]), fov_x=P._fov_x(intr, images.device).repeat(B), apply_mask=False)
    ev[2].record()
    pts, msk = out["points"].view(B, 12, *out["points"].shape[1:]), out["mask"].view(B, 12, *out["mask"].shape[1:])
    merged, merged_mask = P.merge_panoramas(min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H), pts, msk, extr, intr)
    ev[3].record()
    P.finish_panoramas(merged, merged_mask, H, W)
    ev[4].record()
    torch.cuda.synchronize()
    names = ("split", "views", "merge", "finish")
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}, (pts, msk), P.last_merge_stats()


def merge_levels(src, mask, width, height, extr, intr):
    """The merge of P same-size panoramas, src (P, N, vh, vw) distances or (P, N, vh, vw, 3) points and mask (P, N, vh, vw), as
    merge_panoramas launches it, with an event pair around each level's right-hand side and one around its LSMR solve: per level
    its size, the ms of both for the whole batch, and each panorama's iteration count and istop."""
    L = capi.lib()
    cams, n = P._cameras(extr, intr)
    B, _, vh, vw = src.shape[:4]
    ch = 1 if src.dim() == 4 else 3
    s, m = src.contiguous(), capi.mask_u8(mask)
    sizes = P._levels(width, height)
    finest = (capi.PanoramaLevel * B)()
    for e in finest:
        e.h, e.w = height, width
    ws = capi.workspace(L.moge_panorama_workspace_bytes_groups, finest, B, n, device=src.device)
    stats = torch.zeros(len(sizes), B, 2, dtype=torch.int32, device=DEV)
    st = capi.current_stream()
    init, marks = None, []
    for lv, (w, h) in enumerate(sizes):
        b = torch.empty(B, P.num_rows(h, w), dtype=torch.float64, device=DEV)
        rm = torch.empty_like(b, dtype=torch.uint8)
        pm = torch.empty(B, h, w, dtype=torch.uint8, device=DEV)
        depth = torch.empty(B, h, w, dtype=torch.float32, device=DEV)
        dirs = P._table("dirs", (h, w), torch.device(DEV))
        levels = (capi.PanoramaLevel * B)()
        for k, e in enumerate(levels):
            e.h, e.w, e.view0, e.directions = h, w, k * n, dirs.data_ptr()
            e.b, e.row_mask, e.pano_mask, e.depth = b[k].data_ptr(), rm[k].data_ptr(), pm[k].data_ptr(), depth[k].data_ptr()
            e.init, e.stats = None if init is None else init[k].data_ptr(), stats[lv, k].data_ptr()
        ev = events(3)
        ev[0].record()
        capi.check(L.moge_panorama_rhs_groups(s.data_ptr(), ch, m.data_ptr(), n, vh, vw, cams, levels, B, ws.data_ptr(), ws.numel(),
                                              st))
        ev[1].record()
        capi.check(L.moge_panorama_lsmr_groups(levels, B, ws.data_ptr(), ws.numel(), st))
        ev[2].record()
        marks.append(ev)
        if lv + 1 < len(sizes):
            W2, H2 = sizes[lv + 1]
            init = torch.empty(B, H2, W2, dtype=torch.float32, device=DEV)
            maps = (capi.PanoramaResize * B)()
            for k, r in enumerate(maps):
                r.src, r.h, r.w, r.dst, r.H, r.W = depth[k].data_ptr(), h, w, init[k].data_ptr(), H2, W2
            capi.check(L.moge_panorama_resize_groups(maps, B, st))
    torch.cuda.synchronize()
    it = stats.cpu().tolist()
    return [{"size": f"{w}x{h}", "rhs_ms": ev[0].elapsed_time(ev[1]), "lsmr_ms": ev[1].elapsed_time(ev[2]),
             "iterations": [i[0] for i in it[lv]], "istop": [i[1] for i in it[lv]]}
            for lv, ((w, h), ev) in enumerate(zip(sizes, marks))]


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    {k: v.cpu() for o in (out if isinstance(out, list) else [out]) for k, v in o.items()}
    return (time.perf_counter() - t0) * 1e3


def ms(samples, per=1):
    return {k: round(v, 3) if isinstance(v, float) else v for k, v in summary(samples, per).items()}


def level_table(runs):
    """Per level of several merge_levels results: the rhs and LSMR ms for the whole batch, the iterations and the LSMR µs per
    iteration of the longest system (from the median)."""
    table = []
    for lv in zip(*runs):
        its = lv[0]["iterations"]
        lsmr = ms([r["lsmr_ms"] for r in lv])
        table.append({"size": lv[0]["size"], "rhs_ms": ms([r["rhs_ms"] for r in lv]), "lsmr_ms": lsmr, "iterations": its,
                      "lsmr_us_per_iteration": round(lsmr["median"] * 1e3 / max(1, max(its)), 2)})
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = gpu_identity()
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vitl")
    model = MoGeModel(**cfg)
    model.load_state_dict(make_v1_state_dict(cfg, 30, well_posed=True))
    model = model.to(DEV).eval()
    H, W = 1024, 2048
    result = {**gpu, "model": "MoGe-1 ViT-L (synthetic weights), resolution level 9", "panorama": f"{W}x{H}", "batches": []}
    for B in args.batches:
        imgs = torch.from_numpy(np.stack([synthetic_panorama(H, W, s) for s in range(1, B + 1)])).to(DEV)
        P.infer_panoramas(model, imgs)                                   # warm-up: tables, engine plans
        P.infer_panorama(model, imgs[0])
        stages, levels = [], []
        for _ in range(args.steps):
            t, (pts, msk), stats = staged(model, imgs)
            stages.append(t)
        for _ in range(args.steps):
            levels.append(merge_levels(pts, msk, min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H), *P._default_cameras()))
        e2e = {"batched": lambda: P.infer_panoramas(model, imgs),
               "singles": lambda: [P.infer_panorama(model, imgs[k]) for k in range(B)]}
        host = {k: [] for k in e2e}
        for _ in range(args.steps):                                      # alternated
            for k, fn in e2e.items():
                host[k].append(host_ms(fn))
        entry = {"P": B,
                 "per_panorama_stage_ms": {s: ms([r[s] for r in stages], B) for s in stages[0]},
                 "merge_levels": level_table(levels),
                 "iterations": [[s["iterations"] for s in member] for member in stats],
                 "end_to_end_ms_host_results": {k: ms(v) for k, v in host.items()},
                 "end_to_end_ms_per_panorama": {k: round(float(np.median(v)) / B, 2) for k, v in host.items()}}
        result["batches"].append(entry)
        print(json.dumps(entry), flush=True)
        del imgs, pts, msk
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
