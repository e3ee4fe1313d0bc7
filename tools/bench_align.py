"""Per-image time of the alignment solvers at the sizes their callers use (n = 4096 points, the 64x64 grid), engine vs the
reference's own alignment.py on the same GPU.  Prints one JSON line.

    python tools/bench_align.py [--batches 1 32] [--iters 10] [--ref-iters 5]

Each time is the median of `iters` separately timed calls after a warm-up call, with the fastest and slowest beside it.

Workloads: "eval" = the four point and depth alignments of the reference's compute_metrics (align_depth_scale, align_depth_affine,
align_points_scale, align_points_scale_xyz_shift, untruncated, weights 1/|gt|); "train" = align_points_scale_z_shift(trunc=1.0)
as the training loss calls it.  The comparator is loaded from oracle/_ref/ (built by __graft_entry__.build() when MOGE_REFERENCE
is set) and is "not measured" without it; when present, the engine's outputs are checked against it at the timed sizes.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import alignment as engine  # noqa: E402
from oracle.compile_reference import load_alignment  # noqa: E402


def inputs(batch, n, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.randn(batch, n, 3, generator=g)
    gt[..., 2] = 2.0 + 2.0 * torch.rand(batch, n, generator=g)           # positive depth: weights 1/depth, 1/|p| are positive
    pred = (gt - torch.tensor([0.1, -0.2, 0.3])) / 1.3 + 0.01 * torch.randn(batch, n, 3, generator=g)
    outlier = torch.rand(batch, n, 1, generator=g) < 0.1
    pred = torch.where(outlier, pred + torch.randn(batch, n, 3, generator=g), pred)
    return pred.cuda(), gt.cuda()


def workload(mod, name, pred, gt):
    if name == "eval":
        d, dg = pred[..., 2], gt[..., 2]
        wd, wp = 1 / dg, 1 / gt.norm(dim=-1)
        return (mod.align_depth_scale(d, dg, wd), *mod.align_depth_affine(d, dg, wd), mod.align_points_scale(pred, gt, wp),
                *mod.align_points_scale_xyz_shift(pred, gt, wp))
    return mod.align_points_scale_z_shift(pred, gt, 1 / gt.norm(dim=-1), trunc=1.0)


def element_evaluations(name, n):
    """anchors x elements x sorted passes per image (pass A untruncated; A, B and C truncated), summed over the workload's
    solvers; every weight is positive, so every point is an anchor"""
    if name == "eval":
        return n * n + n * 3 * n + 3 * n + n          # depth affine, points scale + xyz shift, points scale, depth scale
    return n * 3 * n * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=5)
    a = ap.parse_args()
    result = {"metric": "alignment_ms_per_image", **gpu_identity(), "n": a.n, "rows": []}
    ref = load_alignment()
    for name in ("eval", "train"):
        for batch in a.batches:
            pred, gt = inputs(batch, a.n, 0)
            row = {"workload": name, "batch": batch, "element_evaluations_per_image": element_evaluations(name, a.n)}
            row["engine_ms_per_image"] = summary(cuda_samples(lambda: workload(engine, name, pred, gt), a.iters), batch)
            if ref is None:
                row["reference_ms_per_image"] = "not measured"
            else:
                # the reference's chunked solvers allocate anchors x 3n tensors per chunk; one image at a time bounds their memory
                def run_ref():
                    return [workload(ref, name, pred[i:i + 1], gt[i:i + 1]) for i in range(min(batch, 2))]
                row["reference_ms_per_image"] = summary(cuda_samples(run_ref, a.ref_iters), min(batch, 2))
                got, want = workload(engine, name, pred[:2], gt[:2]), run_ref()
                got = got if isinstance(got, tuple) else (got,)
                worst = 0.0
                for i, w in enumerate(want):
                    w = w if isinstance(w, tuple) else (w,)
                    for g_, w_ in zip(got, w):
                        worst = max(worst, float(((g_[i:i + 1] - w_).abs() / w_.abs().clamp_min(1e-6)).max()))
                row["max_rel_diff_vs_reference"] = worst
            result["rows"].append(row)
            print(json.dumps(row), file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
