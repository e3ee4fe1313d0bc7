"""Generate tests/golden/alignment.pt from the UNMODIFIED reference `moge.utils.alignment` (CPU, fp32).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_alignment_golden.py

Inputs come from moge_b200.synthetic.alignment_arguments (seeded), so the file stores each case's recipe, the reference's outputs
and a SHA-256 of the regenerated inputs (tests/test_gpu_alignment.py checks that the generator still reproduces them).

Regeneration reproduces every output bit for bit except the two weighted align_affine_lstsq cases at n = 4096: the reference's
fp32 torch.linalg.lstsq (LAPACK on the host) returns results that vary by ~1e-6 relative from one run to the next, even on one
thread.  The parity test compares those cases at rtol 1e-4.
"""
import hashlib
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

from moge_b200.synthetic import ALIGNMENT_FUNCTIONS, alignment_arguments  # noqa: E402

from moge.utils import alignment as ref  # noqa: E402  (the real reference)

OUT = os.path.join(ROOT, "tests", "golden", "alignment.pt")
TRUNC = 0.1            # active on the synthetic outliers (residuals ~1) and not on the inliers (~0.01)


def input_digest(args) -> str:
    h = hashlib.sha256()
    for a in args:
        if isinstance(a, torch.Tensor):
            h.update(a.contiguous().numpy().tobytes())
    return h.hexdigest()


def cases():
    """(function, batch_shape, n, seed, trunc, single_positive)"""
    out = []
    seed = 0
    for fn in ALIGNMENT_FUNCTIONS[:-1]:
        for trunc in (None, TRUNC):
            for batch_shape, n in (((2, 2), 37), ((3,), 1024), ((), 4096)):
                out.append((fn, batch_shape, n, seed, trunc, False))
                seed += 1
    for n in (37, 1024):     # one problem: the reference's per-element trunc does not broadcast over a batch of problems
        out.append(("align", (), n, seed, "per_element", False))
        seed += 1
    for fn in ("align_depth_affine", "align_points_scale_z_shift", "align_points_scale_xyz_shift"):   # one image: a single positive weight
        for trunc in (None, TRUNC):
            out.append((fn, (3,), 37, seed, trunc, True))
            seed += 1
    for trunc in (None, "weighted"):
        for batch_shape, n in (((2, 2), 37), ((), 4096)):
            out.append(("align_affine_lstsq", batch_shape, n, seed, trunc, False))
            seed += 1
    return out


def main():
    gold = []
    for fn, batch_shape, n, seed, trunc, single in cases():
        args = alignment_arguments(fn, batch_shape, n, seed, trunc, single)
        t0 = time.time()
        if fn == "align_affine_lstsq":
            res = ref.align_affine_lstsq(*args)
        else:
            res = getattr(ref, fn)(*args)
        res = res if isinstance(res, tuple) else (res,)
        gold.append({"fn": fn, "batch_shape": batch_shape, "n": n, "seed": seed, "trunc": trunc, "single_positive": single,
                     "inputs_sha256": input_digest(args), "outputs": tuple(r.detach().clone() for r in res)})
        print(f"{fn:30s} {str(batch_shape):8s} n={n:5d} trunc={trunc} single={single}  {time.time() - t0:6.2f} s")
    torch.save(gold, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
