"""Batched panorama inference on the H100: infer_panoramas over P panoramas against P infer_panorama calls, per-panorama stage
times, and the merge's per-level solve times and LSMR iterations.  Prints one JSON line (profiles/h100_bench_panorama_batch.json).

    python tools/bench_panorama_batch.py [--steps 5] [--batches 1 2 4 8] [--parent-lib SO] [--out FILE]

Workload: 2048 x 1024 synthetic panoramas (seeds 1..P) through a synthetic-weight ViT-L MoGe-1 at resolution level 9, as
tools/bench_panorama.py.  Per P: the stages of the batched path between CUDA events (split, the 12P views' infer, merge,
finish), each level's batched solve (one event pair around its right-hand side and one around its cooperative LSMR launch), and
the end-to-end time with the results copied to the host, the batched call alternated with P single calls.  At P = 1,
`merge_panorama` and `merge_panoramas` are alternated on the same views, and with --parent-lib (a libmoge_b200.so built from
another commit, e.g. the parent's, by moge_b200/csrc/build.sh) also `merge_panorama` through that library; outputs and
iteration counts are compared bit for bit and each solve's per-level time is reported.
"""
import argparse
import contextlib
import ctypes as C
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
    """The batched path's stages between events: {stage: ms for the whole batch}, and the views' engine outputs."""
    ev = events(5)
    extr, intr = P._default_cameras()
    B, H, W = images.shape[:3]
    ev[0].record()
    views = P.split_panoramas(images, extr, intr)
    ev[1].record()
    out = model.infer(views.view(-1, *views.shape[2:]), fov_x=P._fov_x(intr, images.device).repeat(B), apply_mask=False)
    ev[2].record()
    pts, msk = out["points"].view(B, 12, *out["points"].shape[1:]), out["mask"].view(B, 12, *out["mask"].shape[1:])
    depth, mask = P.merge_panoramas(min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H), pts, msk, extr, intr)
    ev[3].record()
    P.finish_panoramas(depth, mask, H, W)
    ev[4].record()
    torch.cuda.synchronize()
    names = ("split", "views", "merge", "finish")
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}, (pts, msk)


def merge_levels(pts, msk, width, height):
    """merge_panoramas' launches with an event pair around each level's right-hand side and its LSMR solve: per level the ms of
    both for the whole batch and each panorama's iteration count."""
    L = capi.lib()
    extr, intr = P._default_cameras()
    cams, n = P._cameras(extr, intr)
    B, _, vh, vw = pts.shape[:4]
    levels = P._levels(width, height)
    ws = capi.workspace(L.moge_panorama_workspace_bytes_batch, B, n, height, width, device=pts.device)
    stats = torch.zeros(len(levels), B, 2, dtype=torch.int32, device=DEV)
    s, m = pts.contiguous(), capi.mask_u8(msk)
    st = capi.current_stream()
    init, marks = None, []
    for lv, (w, h) in enumerate(levels):
        b = torch.empty(B, P.num_rows(h, w), dtype=torch.float64, device=DEV)
        rm = torch.empty_like(b, dtype=torch.uint8)
        pm = torch.empty(B, h, w, dtype=torch.uint8, device=DEV)
        depth = torch.empty(B, h, w, dtype=torch.float32, device=DEV)
        dirs = P._table("dirs", (h, w), torch.device(DEV))
        ev = events(3)
        ev[0].record()
        capi.check(L.moge_panorama_rhs_batch(s.data_ptr(), 3, m.data_ptr(), B, n, vh, vw, cams, dirs.data_ptr(), h, w, b.data_ptr(),
                                             rm.data_ptr(), pm.data_ptr(), ws.data_ptr(), ws.numel(), st))
        ev[1].record()
        capi.check(L.moge_panorama_lsmr_batch(b.data_ptr(), rm.data_ptr(), B, h, w, capi.ptr(init), depth.data_ptr(),
                                              stats[lv].data_ptr(), ws.data_ptr(), ws.numel(), st))
        ev[2].record()
        marks.append(ev)
        if lv + 1 < len(levels):
            W2, H2 = levels[lv + 1]
            init = torch.empty(B, H2, W2, dtype=torch.float32, device=DEV)
            capi.check(L.moge_panorama_resize_batch(depth.data_ptr(), B, h, w, H2, W2, init.data_ptr(), st))
    torch.cuda.synchronize()
    it = stats.cpu().tolist()
    return [{"size": f"{w}x{h}", "rhs_ms": round(ev[0].elapsed_time(ev[1]), 3), "lsmr_ms": round(ev[1].elapsed_time(ev[2]), 3),
             "iterations": [i[0] for i in it[lv]],
             "lsmr_us_per_iteration": round(ev[1].elapsed_time(ev[2]) * 1e3 / max(1, max(i[0] for i in it[lv])), 2)}
            for lv, ((w, h), ev) in enumerate(zip(levels, marks))]


@contextlib.contextmanager
def library(path):
    """moge_b200's calls through another build of the library: only the single-panorama merge's entry points are bound."""
    L = C.CDLL(os.path.abspath(path))
    for name in ("moge_last_error", "moge_panorama_workspace_bytes", "moge_panorama_rhs", "moge_panorama_lsmr", "moge_panorama_resize"):
        sig = capi.SIGNATURES[name]
        f = getattr(L, name)
        f.restype, f.argtypes = sig if isinstance(sig, tuple) else (C.c_int, sig)
    saved, capi._lib = capi._lib, L
    try:
        yield
    finally:
        capi._lib = saved


def single_lsmr_levels(pts, msk, width, height):
    """merge_panorama's launches with an event pair around each level's LSMR solve: [ms] per level."""
    L = capi.lib()
    extr, intr = P._default_cameras()
    cams, n = P._cameras(extr, intr)
    levels = P._levels(width, height)
    ws = capi.workspace(L.moge_panorama_workspace_bytes, n, height, width, device=pts.device)
    stats = torch.zeros(len(levels), 2, dtype=torch.int32, device=DEV)
    s, m = pts.contiguous(), capi.mask_u8(msk)
    st = capi.current_stream()
    init, marks = None, []
    for lv, (w, h) in enumerate(levels):
        b = torch.empty(P.num_rows(h, w), dtype=torch.float64, device=DEV)
        rm = torch.empty_like(b, dtype=torch.uint8)
        pm = torch.empty(h, w, dtype=torch.uint8, device=DEV)
        depth = torch.empty(h, w, dtype=torch.float32, device=DEV)
        dirs = P._table("dirs", (h, w), torch.device(DEV))
        capi.check(L.moge_panorama_rhs(s.data_ptr(), 3, m.data_ptr(), n, pts.shape[1], pts.shape[2], cams, dirs.data_ptr(), h, w,
                                       b.data_ptr(), rm.data_ptr(), pm.data_ptr(), ws.data_ptr(), ws.numel(), st))
        ev = events(2)
        ev[0].record()
        capi.check(L.moge_panorama_lsmr(b.data_ptr(), rm.data_ptr(), h, w, capi.ptr(init), depth.data_ptr(), stats[lv].data_ptr(),
                                        ws.data_ptr(), ws.numel(), st))
        ev[1].record()
        marks.append(ev)
        if lv + 1 < len(levels):
            W2, H2 = levels[lv + 1]
            init = torch.empty(H2, W2, dtype=torch.float32, device=DEV)
            capi.check(L.moge_panorama_resize(depth.data_ptr(), h, w, H2, W2, init.data_ptr(), st))
    torch.cuda.synchronize()
    return [round(ev[0].elapsed_time(ev[1]), 3) for ev in marks]


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    {k: v.cpu() for o in (out if isinstance(out, list) else [out]) for k, v in o.items()}
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--parent-lib", default=None, help="a libmoge_b200.so of another commit: its merge_panorama at P = 1 too")
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
        runs = [staged(model, imgs)[0] for _ in range(args.steps)]
        stage = {k: round(float(np.median([r[k] for r in runs])) / B, 3) for k in runs[0]}
        _, (pts, msk) = staged(model, imgs)
        levels = merge_levels(pts, msk, min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H))
        batched, singles = [], []
        for _ in range(args.steps):                                      # alternated
            batched.append(host_ms(lambda: P.infer_panoramas(model, imgs)))
            singles.append(host_ms(lambda: [P.infer_panorama(model, imgs[k]) for k in range(B)]))
        entry = {"P": B, "per_panorama_stage_ms": stage, "merge_levels": levels,
                 "end_to_end_ms_host_results": {"batched": round(float(np.median(batched)), 2),
                                                "singles": round(float(np.median(singles)), 2),
                                                "batched_per_panorama": round(float(np.median(batched)) / B, 2),
                                                "singles_per_panorama": round(float(np.median(singles)) / B, 2)}}
        if B == 1:
            extr, intr = P._default_cameras()
            w, h = min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H)
            arms = {"merge_panorama": lambda: P.merge_panorama(w, h, pts[0], msk[0], extr, intr),
                    "merge_panoramas": lambda: P.merge_panoramas(w, h, pts, msk, extr, intr)}
            if args.parent_lib:
                def parent():
                    with library(args.parent_lib):
                        return P.merge_panorama(w, h, pts[0], msk[0], extr, intr)
                arms["parent_merge_panorama"] = parent
            outs, stats = {}, {}
            for k, fn in arms.items():
                outs[k] = fn()
                st = P.last_merge_stats()
                stats[k] = st[0] if k == "merge_panoramas" else st
            ms = {k: [] for k in arms}
            for _ in range(args.steps):                                  # alternated
                for k, fn in arms.items():
                    ms[k] += cuda_samples(fn, 1, warmup=0)
            lsmr_levels = {"merge_panorama": single_lsmr_levels(pts[0], msk[0], w, h)}
            if args.parent_lib:
                with library(args.parent_lib):
                    lsmr_levels["parent_merge_panorama"] = single_lsmr_levels(pts[0], msk[0], w, h)
            d0, m0 = outs["merge_panorama"]
            entry["p1_merge"] = {
                "ms": {k: summary(v) for k, v in ms.items()}, "lsmr_ms_per_level": lsmr_levels,
                "iterations": [s["iterations"] for s in stats["merge_panorama"]],
                "bitwise_equal_to_merge_panorama": {
                    k: bool(torch.equal(d0, o[0].view_as(d0)) and torch.equal(m0, o[1].view_as(m0)) and stats[k] == stats["merge_panorama"])
                    for k, o in outs.items() if k != "merge_panorama"}}
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
