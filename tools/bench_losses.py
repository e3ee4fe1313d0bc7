"""Time of the training losses, forward and backward, on one image: the engine (moge_b200.losses, moge_b200.local_loss) against the
reference's own moge/train/losses.py on the same GPU, with the peak memory each adds.  Prints one JSON line with the GPU name
and power limit read in the same run.

    python tools/bench_losses.py [--iters 20] [--ref-iters 10]

Losses: affine_invariant_global_loss at align_resolution 48 (the v2 "A" set) and 64 (its default), edge_loss (v2 "A"),
normal_loss, mask_bce_loss (v2 "A") and mask_l2_loss; and the three affine_invariant_local_loss terms of v2 "A" (patch_4,
patch_16, patch_64) at the first two sizes, with focal 0.3 and the global loss's scale as global_scale.  Every call of a local
term starts from torch.cuda.manual_seed(0), so the engine and the reference draw the same anchors.  Each time is the median of separately timed calls after a warm-up call
(CUDA events around loss + loss.sum().backward(), host work included, then a device synchronise), with the fastest and slowest
beside it.  Peak memory is torch.cuda.max_memory_allocated over one such call, less what was allocated before it.  The
comparator is loaded from oracle/_ref/ (built by __graft_entry__.build() when MOGE_REFERENCE is set,
oracle/compile_reference.py) and is "not measured" without it; when present, losses and gradients are compared at every
timed size.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import local_loss as engine_local  # noqa: E402
from moge_b200 import losses as engine  # noqa: E402
from moge_b200.synthetic import synthetic_loss_case  # noqa: E402
from oracle.compile_reference import load_losses  # noqa: E402

SIZES = [(512, 512), (768, 1024), (1000, 1000)]
LOSSES = [
    ("global_ar48", "affine_invariant_global_loss", ("pred_points", "gt_points"), {"align_resolution": 48}),
    ("global_ar64", "affine_invariant_global_loss", ("pred_points", "gt_points"), {}),
    ("edge", "edge_loss", ("pred_points", "gt_points"), {}),
    ("normal", "normal_loss", ("pred_points", "gt_points"), {}),
    ("mask_bce", "mask_bce_loss", ("pred_mask", "gt_mask_pos", "gt_mask_neg"), {}),
    ("mask_l2", "mask_l2_loss", ("pred_mask", "gt_mask_pos", "gt_mask_neg"), {}),
]
LOCAL = [
    ("local_patch_4", {"level": 4, "num_patches": 16, "align_resolution": 24}),
    ("local_patch_16", {"level": 16, "num_patches": 256, "align_resolution": 12}),
    ("local_patch_64", {"level": 64, "num_patches": 4096, "align_resolution": 6}),
]
LOCAL_SIZES = SIZES[:2]
DIFF = ("pred_points", "pred_mask")


def call(module, fn, names, kwargs, inputs):
    if fn == "affine_invariant_local_loss":
        torch.cuda.manual_seed(0)
    args = [inputs[k].detach().requires_grad_(True) if k in DIFF else inputs[k] for k in names]
    loss = getattr(module, fn)(*args, **kwargs)[0]
    loss.sum().backward()
    return loss.detach(), args[0].grad


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=10)
    a = ap.parse_args()
    result = {"metric": "training_loss_ms_forward_backward_per_image", **gpu_identity(), "rows": []}
    ref = load_losses()
    for H, W in SIZES:
        inputs = {k: v.cuda() for k, v in synthetic_loss_case(0, (1,), H, W).items()}
        inputs["focal"] = torch.full((1,), 0.3, device="cuda")
        inputs["global_scale"] = engine.affine_invariant_global_loss(inputs["pred_points"], inputs["gt_points"])[2]
        local = [(name, "affine_invariant_local_loss", ("pred_points", "gt_points", "focal", "global_scale"), kw) for name, kw in LOCAL]
        for name, fn, names, kwargs in LOSSES + (local if (H, W) in LOCAL_SIZES else []):
            row = {"H": H, "W": W, "loss": name}
            mod = engine_local if fn == "affine_invariant_local_loss" else engine
            run_e = lambda: call(mod, fn, names, kwargs, inputs)  # noqa: E731
            row["engine_ms"] = summary(cuda_samples(run_e, a.iters))
            row["engine_peak_mb"] = peak_mb(run_e)
            if ref is None:
                row["reference_ms"] = row["reference_peak_mb"] = "not measured"
            else:
                run_r = lambda: call(ref, fn, names, kwargs, inputs)  # noqa: E731
                row["reference_ms"] = summary(cuda_samples(run_r, a.ref_iters))
                row["reference_peak_mb"] = peak_mb(run_r)
                (le, ge), (lr, gr) = run_e(), run_r()
                row["loss_rel_diff"] = float(((le.double() - lr.double()).abs() / lr.double().abs().clamp_min(1e-30)).max())
                row["grad_max_diff_over_max_grad"] = float((ge.double() - gr.double()).abs().max() / gr.double().abs().max().clamp_min(1e-30))
            result["rows"].append(row)
            print(json.dumps(row), file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
