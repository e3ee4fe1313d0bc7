"""Per-image time of compute_metrics with MoGe-2 keys (points_metric, depth_metric, intrinsics), a sharp-boundary GT and box
segments: the engine at batch 1 and batch 8 against the reference's own moge/test/metrics.py on the same GPU.  Prints one JSON
line with the GPU name and power limit read in the same run.

    python tools/bench_metrics.py [--iters 10] [--ref-iters 3]

Each time is the median of separately timed calls after a warm-up call (CUDA events around the whole call, host work included),
with the fastest and slowest beside it.  The comparator is loaded from oracle/_ref/ (built by __graft_entry__.build() when
MOGE_REFERENCE is set, oracle/compile_reference.py) and is "not measured" without it; when present, the two results are compared at every timed size.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import metrics as engine  # noqa: E402
from moge_b200.synthetic import METRICS_KEYS, synthetic_metrics_case  # noqa: E402
from oracle.compile_reference import load_metrics  # noqa: E402

WORKLOADS = [(480, 640, 50), (436, 872, 50), (1365, 2048, 100)]


def flat(m, prefix=""):
    out = {}
    for k, v in m.items():
        out.update(flat(v, prefix + k + ".") if isinstance(v, dict) else {prefix + k: v})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=3)
    a = ap.parse_args()
    result = {"metric": "compute_metrics_ms_per_image", **gpu_identity(), "keys": list(METRICS_KEYS["moge2"]), "rows": []}
    ref = load_metrics()
    for H, W, segments in WORKLOADS:
        cases = []
        for i in range(8):
            p, g = synthetic_metrics_case(i, H, W, METRICS_KEYS["moge2"], True, True, segments)
            cases.append(({k: v.cuda() for k, v in p.items()}, {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in g.items()}))
        pred = {k: torch.stack([c[0][k] for c in cases]) for k in cases[0][0]}
        gt = {k: (torch.stack([c[1][k] for c in cases]) if isinstance(cases[0][1][k], torch.Tensor) else cases[0][1][k])
              for k in cases[0][1] if k != "segmentation_labels"}
        gt["segmentation_labels"] = [c[1]["segmentation_labels"] for c in cases]
        row = {"H": H, "W": W, "segments": segments + 3}
        row["engine_b1_ms_per_image"] = summary(cuda_samples(lambda: engine.compute_metrics(*cases[0]), a.iters))
        row["engine_b8_ms_per_image"] = summary(cuda_samples(lambda: engine.compute_metrics_batch(pred, gt), a.iters), 8)
        if ref is None:
            row["reference_ms_per_image"] = "not measured"
        else:
            row["reference_ms_per_image"] = summary(cuda_samples(lambda: ref.compute_metrics(*cases[0]), a.ref_iters))
            got, want = flat(engine.compute_metrics(*cases[0])[0]), flat(ref.compute_metrics(*cases[0])[0])
            row["keys_agree"] = got.keys() == want.keys()
            row["max_abs_diff_vs_reference"] = max((abs(got[k] - want[k]) for k in want if k in got and not math.isnan(want[k])), default=None)
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
