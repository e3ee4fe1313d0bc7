"""Geometry utilities on the GPU (moge_b200.geometry) against the reference's `moge/utils/geometry_torch.py` on the same GPU:
`refine_depth_with_normal` (10 sweeps, kernel 5) and `dilate_with_mask` (mean and median, 1 iteration) at 518x518, 1024x768
and 2048x1365, batch 1 and 8, on synthetic_geometry_case inputs (piecewise-planar depth, its noisy normals, the scene's mask).
Prints one JSON line with the GPU name and power limit read in the same run.

    python tools/bench_geometry.py [--iters 20] [--ref-iters 3]

Per row, in ms per call (median, min and max of separately timed calls after a warm-up call, CUDA events around each call):
  - engine: the drop-in's call (workspace and output allocation included);
  - reference: the reference module compiled by oracle/compile_reference.py (utils3d from the stand-in in
    oracle/utils3d_geometry.py), on the same CUDA tensors; "not measured" when it was not built;
  - peak_extra_mb: the largest device memory allocated during one call above what was allocated before it;
  - max_rel_diff: the largest |engine - reference| / |reference| over the outputs (refine), or whether the outputs agree
    bitwise (dilate median) or the largest relative difference (dilate mean).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import geometry as G  # noqa: E402
from moge_b200.synthetic import synthetic_geometry_case  # noqa: E402
from oracle.utils3d_geometry import load_geometry  # noqa: E402

WORKLOADS = [(518, 518), (768, 1024), (1365, 2048)]
BATCHES = (1, 8)


def peak_extra_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    extra = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    del out
    return extra


def timed(fn, iters):
    return {"ms": summary(cuda_samples(fn, iters)), "peak_extra_mb": peak_extra_mb(fn)}


def rel_diff(a, b):
    a, b = a.double(), b.double()
    fin = torch.isfinite(b)
    return float(((a - b).abs()[fin] / b.abs()[fin].clamp_min(1e-30)).max()) if fin.any() else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=3)
    a = ap.parse_args()
    ref = load_geometry()
    result = {"metric": "geometry_utils_ms_per_call", **gpu_identity(),
              "reference": "moge/utils/geometry_torch.py on the same GPU" if ref else "not measured (reference not built)", "rows": []}
    for H, W in WORKLOADS:
        case = synthetic_geometry_case(0, (max(BATCHES),), H, W, "scene")
        for B in BATCHES:
            d, n = case["depth"][:B].cuda(), case["normal"][:B].cuda()
            K, m = case["intrinsics"][:B].cuda(), case["mask"][:B].cuda()
            ours = G.refine_depth_with_normal(d, n, K)
            row = {"fn": "refine_depth_with_normal", "H": H, "W": W, "batch": B,
                   "engine": timed(lambda: G.refine_depth_with_normal(d, n, K), a.iters)}
            if ref:
                want = ref.refine_depth_with_normal(d, n, K)
                row["reference"] = timed(lambda: ref.refine_depth_with_normal(d, n, K), a.ref_iters)
                row["max_rel_diff"] = rel_diff(ours, want)
                row["speedup"] = row["reference"]["ms"]["median"] / row["engine"]["ms"]["median"]
                del want
            result["rows"].append(row)
            print(json.dumps(row), file=sys.stderr)
            for filt in ("mean", "median"):
                ov, om = G.dilate_with_mask(d, m, filt)
                row = {"fn": f"dilate_with_mask[{filt}]", "H": H, "W": W, "batch": B,
                       "engine": timed(lambda: G.dilate_with_mask(d, m, filt), a.iters)}
                if ref:
                    rv, rm = ref.dilate_with_mask(d, m, filt)
                    row["reference"] = timed(lambda: ref.dilate_with_mask(d, m, filt), a.ref_iters)
                    row["mask_equal"] = bool(torch.equal(om, rm))
                    if filt == "median":
                        row["bitwise_equal"] = bool(torch.equal(ov.nan_to_num(), rv.nan_to_num())
                                                    and torch.equal(ov.isnan(), rv.isnan()))
                    else:
                        row["max_rel_diff"] = rel_diff(ov, rv)
                    row["speedup"] = row["reference"]["ms"]["median"] / row["engine"]["ms"]["median"]
                result["rows"].append(row)
                print(json.dumps(row), file=sys.stderr)
            del d, n, K, m
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
