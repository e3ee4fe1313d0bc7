"""Generate tests/golden/metrics.pt from the UNMODIFIED reference `moge.test.metrics.compute_metrics` (CPU, fp32).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_metrics_golden.py

utils3d resolves to the stand-in under oracle/utils3d_shim, with the metrics' two functions from oracle/utils3d_metrics.py.  Inputs come from moge_b200.synthetic.synthetic_metrics_case (seeded),
so the file stores each case's recipe, a SHA-256 of its inputs, the reference's metrics and its `misc` maps at a stride of 8.
Each case is also run through oracle/metrics_port.py with the reference's alignment solvers, and the two must agree exactly.
"""
import hashlib
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "utils3d_shim"))
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")
sys.path.insert(1, os.environ["MOGE_REFERENCE"])

import torch  # noqa: E402

from moge_b200.synthetic import METRICS_KEYS, synthetic_metrics_case  # noqa: E402
from oracle import metrics_port  # noqa: E402  (installs the metrics' utils3d functions into the stand-in)

from moge.test import metrics as ref  # noqa: E402  (the real reference)
from moge.utils import alignment as ref_alignment  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "metrics.pt")
STRIDE = 8

# (name, keys, H, W, is_metric, sharp, segments, negative, vis)
CASES = [
    ("moge2_metric_640x480", "moge2", 480, 640, True, True, 50, False, False),
    ("moge2_nonmetric_872x436", "moge2", 436, 872, False, True, 20, False, False),
    ("moge1_1024x768", "moge1", 768, 1024, True, True, 12, False, True),
    ("moge2_plain_640x480", "moge2", 480, 640, True, False, 0, False, False),
    ("depth_affine_vis_640x480", "depth_affine", 480, 640, False, True, 0, True, True),
    ("disparity_872x436", "disparity", 436, 872, False, True, 0, True, False),
    ("points_affine_640x480", "points_affine", 480, 640, False, False, 8, False, True),
    ("moge2_subgrid_50x70", "moge2", 50, 70, True, True, 4, False, True),
]


def input_digest(pred, gt) -> str:
    h = hashlib.sha256()
    for d in (pred, gt):
        for k in sorted(d):
            if isinstance(d[k], torch.Tensor):
                h.update(k.encode())
                h.update(d[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    return a == b or (math.isnan(a) and math.isnan(b))


def main():
    gold = []
    for seed, (name, keys, H, W, is_metric, sharp, segments, negative, vis) in enumerate(CASES):
        pred, gt = synthetic_metrics_case(seed, H, W, METRICS_KEYS[keys], is_metric, sharp, segments, negative)
        t0 = time.time()
        metrics, misc = ref.compute_metrics(pred, gt, vis=vis)
        t1 = time.time()
        pm, pmisc = metrics_port.compute_metrics(pred, gt, vis=vis, alignment=ref_alignment)
        assert same(metrics, pm), (name, metrics, pm)
        assert misc.keys() == pmisc.keys() and all(torch.equal(misc[k], pmisc[k]) for k in misc), name
        gold.append({"name": name, "keys": keys, "H": H, "W": W, "is_metric": is_metric, "sharp": sharp, "segments": segments,
                     "negative": negative, "vis": vis, "seed": seed, "inputs_sha256": input_digest(pred, gt), "metrics": metrics,
                     "misc_stride": STRIDE, "misc": {k: v[::STRIDE, ::STRIDE].clone() for k, v in misc.items()}})
        print(f"{name:28s} reference {t1 - t0:6.2f} s  {metrics}")
    torch.save(gold, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
