"""Batched panorama inference on the H100: infer_panoramas over P panoramas against P infer_panorama calls, per-panorama stage
times, and the merge's per-level solve times and LSMR iterations.  Prints one JSON line (profiles/h100_bench_panorama_batch.json).

    python tools/bench_panorama_batch.py [--steps 5] [--batches 1 2 4 8] [--parent-lib SO] [--out FILE]

Workload: 2048 x 1024 synthetic panoramas (seeds 1..P) through a synthetic-weight ViT-L MoGe-1 at resolution level 9, as
tools/bench_panorama.py.  Per P: the stages between CUDA events (split, the 12P views' infer, merge, finish), each level's
solve (one event pair around its right-hand side and one around its cooperative LSMR launch), and the end-to-end time with the
results copied to the host, infer_panoramas alternated with P infer_panorama calls.  Times are the median, min and max of
--steps runs.

With --parent-lib (a libmoge_b200.so built by moge_b200/csrc/build.sh from a commit whose panorama entry points still carried
a _batch suffix, e.g. the parent's), every measurement above is also taken with the panorama calls going through that library,
alternated run by run with this build, and the outputs of every stage and the per-level iteration counts of the two are
compared bit for bit.  The views' engine runs on this build in both arms.
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
    """infer_panoramas' stages between events: ({stage: ms for the whole batch}, {name: output of a stage}, last_merge_stats())."""
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
    depth, mask, points = P.finish_panoramas(merged, merged_mask, H, W)
    ev[4].record()
    torch.cuda.synchronize()
    names = ("split", "views", "merge", "finish")
    outputs = {"views": views, "view_points": pts, "view_mask": msk, "merged_depth": merged, "merged_mask": merged_mask,
               "depth": depth, "mask": mask, "points": points}
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}, outputs, P.last_merge_stats()


def merge_levels(pts, msk, width, height):
    """merge_panoramas' launches with an event pair around each level's right-hand side and its LSMR solve: per level its size,
    the ms of both for the whole batch and each panorama's iteration count."""
    L = capi.lib()
    extr, intr = P._default_cameras()
    cams, n = P._cameras(extr, intr)
    B, _, vh, vw = pts.shape[:4]
    levels = P._levels(width, height)
    ws = capi.workspace(L.moge_panorama_workspace_bytes, B, n, height, width, device=pts.device)
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
        capi.check(L.moge_panorama_rhs(s.data_ptr(), 3, m.data_ptr(), B, n, vh, vw, cams, dirs.data_ptr(), h, w, b.data_ptr(),
                                       rm.data_ptr(), pm.data_ptr(), ws.data_ptr(), ws.numel(), st))
        ev[1].record()
        capi.check(L.moge_panorama_lsmr(b.data_ptr(), rm.data_ptr(), B, h, w, capi.ptr(init), depth.data_ptr(), stats[lv].data_ptr(),
                                        ws.data_ptr(), ws.numel(), st))
        ev[2].record()
        marks.append(ev)
        if lv + 1 < len(levels):
            W2, H2 = levels[lv + 1]
            init = torch.empty(B, H2, W2, dtype=torch.float32, device=DEV)
            capi.check(L.moge_panorama_resize(depth.data_ptr(), B, h, w, H2, W2, init.data_ptr(), st))
    torch.cuda.synchronize()
    it = stats.cpu().tolist()
    return [{"size": f"{w}x{h}", "rhs_ms": ev[0].elapsed_time(ev[1]), "lsmr_ms": ev[1].elapsed_time(ev[2]),
             "iterations": [i[0] for i in it[lv]]} for lv, ((w, h), ev) in enumerate(zip(levels, marks))]


# The panorama entry points of this build and the symbols of a parent build that take the same argument lists.
PARENT_SYMBOLS = {"moge_panorama_split": "moge_panorama_split_batch",
                  "moge_panorama_workspace_bytes": "moge_panorama_workspace_bytes_batch",
                  "moge_panorama_rhs": "moge_panorama_rhs_batch", "moge_panorama_lsmr": "moge_panorama_lsmr_batch",
                  "moge_panorama_resize": "moge_panorama_resize_batch", "moge_panorama_finish": "moge_panorama_finish_batch",
                  "moge_last_error": "moge_last_error"}


def parent_functions(path):
    """{name in this build: the parent build's function, bound with this build's signature}.  Exits when the library lacks one
    of PARENT_SYMBOLS, so that no call reaches a function whose argument list differs."""
    L = C.CDLL(os.path.abspath(path))
    missing = [sym for sym in PARENT_SYMBOLS.values() if not hasattr(L, sym)]
    if missing:
        sys.exit(f"{path} lacks {', '.join(missing)}: --parent-lib takes a build whose panorama entry points end in _batch")
    fns = {}
    for name, sym in PARENT_SYMBOLS.items():
        sig = capi.SIGNATURES[name]
        f = getattr(L, sym)
        f.restype, f.argtypes = sig if isinstance(sig, tuple) else (C.c_int, sig)
        fns[name] = f
    return fns


@contextlib.contextmanager
def through(fns):
    """moge_b200's calls with capi.lib() answering the names in `fns` from them and every other name from this build."""
    own = capi.lib()

    class Lib:
        def __getattr__(self, name):
            return fns[name] if name in fns else getattr(own, name)
    capi._lib = Lib()
    try:
        yield
    finally:
        capi._lib = own


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
    ap.add_argument("--parent-lib", default=None, help="a libmoge_b200.so whose panorama entry points end in _batch: every "
                                                       "measurement also through it, alternated, with the outputs compared")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = gpu_identity()
    arms = {"new": contextlib.nullcontext}
    if args.parent_lib:
        fns = parent_functions(args.parent_lib)
        arms["parent"] = lambda: through(fns)
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vitl")
    model = MoGeModel(**cfg)
    model.load_state_dict(make_v1_state_dict(cfg, 30, well_posed=True))
    model = model.to(DEV).eval()
    H, W = 1024, 2048
    result = {**gpu, "model": "MoGe-1 ViT-L (synthetic weights), resolution level 9", "panorama": f"{W}x{H}",
              "arms": list(arms), "batches": []}
    for B in args.batches:
        imgs = torch.from_numpy(np.stack([synthetic_panorama(H, W, s) for s in range(1, B + 1)])).to(DEV)
        for arm in arms.values():                                        # warm-up: tables, engine plans
            with arm():
                P.infer_panoramas(model, imgs)
                P.infer_panorama(model, imgs[0])
        stages, outputs, stats, levels = ({k: [] for k in arms} for _ in range(4))
        for _ in range(args.steps):                                      # alternated
            for k, arm in arms.items():
                with arm():
                    t, outputs[k], stats[k] = staged(model, imgs)
                stages[k].append(t)
        pts, msk = outputs["new"]["view_points"], outputs["new"]["view_mask"]
        for _ in range(args.steps):                                      # alternated
            for k, arm in arms.items():
                with arm():
                    levels[k].append(merge_levels(pts, msk, min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H)))
        e2e = {"batched": lambda: P.infer_panoramas(model, imgs),
               "singles": lambda: [P.infer_panorama(model, imgs[k]) for k in range(B)]}
        if args.parent_lib:
            def parent_batched():
                with through(fns):
                    return P.infer_panoramas(model, imgs)
            e2e["parent_batched"] = parent_batched
        host = {k: [] for k in e2e}
        for _ in range(args.steps):                                      # alternated
            for k, fn in e2e.items():
                host[k].append(host_ms(fn))
        entry = {"P": B,
                 "per_panorama_stage_ms": {k: {s: ms([r[s] for r in runs], B) for s in runs[0]} for k, runs in stages.items()},
                 "merge_levels": {k: level_table(runs) for k, runs in levels.items()},
                 "iterations": [[s["iterations"] for s in member] for member in stats["new"]],
                 "end_to_end_ms_host_results": {k: ms(v) for k, v in host.items()},
                 "end_to_end_ms_per_panorama": {k: round(float(np.median(v)) / B, 2) for k, v in host.items()}}
        if args.parent_lib:
            new, parent = outputs["new"], outputs["parent"]
            entry["bitwise_equal_to_parent"] = {
                **{k: bool(torch.equal(new[k], parent[k])) for k in new},
                "merge_stats": stats["new"] == stats["parent"],
                "level_iterations": [lv["iterations"] for lv in levels["new"][0]] == [lv["iterations"] for lv in levels["parent"][0]]}
        result["batches"].append(entry)
        print(json.dumps(entry), flush=True)
        del imgs, pts, msk, outputs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
