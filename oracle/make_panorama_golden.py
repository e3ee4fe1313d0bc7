"""Generate tests/golden/panorama.pt from the UNMODIFIED reference `moge/utils/panorama.py` (numpy, cv2 and SciPy on the host).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_panorama_golden.py

utils3d resolves to the stand-in under oracle/utils3d_shim, with `utils3d.np` from oracle/utils3d_panorama.py.  The module's own
`lsmr` name is wrapped at run time to record what each pyramid level solves; the module's code is not changed.  Inputs come from
the seeded generators in moge_b200.synthetic, so the file stores their recipes and SHA-256 digests rather than the inputs:
- cameras: the reference's get_panorama_cameras();
- split cases: synthetic_panorama images split at 64 and 96; the views of the first case, and the SHA-256 of every case's views;
- merge cases: synthetic_room_views(96) (an analytic box room, 1% noise, mask holes) merged at 200 x 100 (one level), 320 x 160
  (two) and 600 x 300 (three).  Per level: the row masks (packed bits), SciPy's LSMR iteration count and istop, and for the
  160 x 80 level the right-hand side in the reference's row order (float32).  The final depth (at a stride of 1, 2, 3) and mask.
  `sensitivity`: the largest relative change of the final depth when every level's b is rounded once to float32 and back;
- finish case: the 200 x 100 merge's depth and mask resized to 251 x 127 as infer_panorama.py:120-121 does.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")

import importlib.util  # noqa: E402

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from moge_b200.synthetic import array_digest, synthetic_panorama, synthetic_room_views  # noqa: E402
from oracle import utils3d_panorama  # noqa: E402

utils3d_panorama.install()
_spec = importlib.util.spec_from_file_location(
    "reference_panorama", os.path.join(os.environ["MOGE_REFERENCE"], "moge", "utils", "panorama.py"))
ref = importlib.util.module_from_spec(_spec)       # the real reference module, loaded from its file under its own name
_spec.loader.exec_module(ref)

OUT = os.path.join(ROOT, "tests", "golden", "panorama.pt")
SPLIT_CASES = [(128, 256, 64, 0), (150, 301, 96, 1)]              # (H, W, resolution, seed)
MERGE_SIZES = [(200, 100), (320, 160), (600, 300)]                 # (width, height)
FINISH = (100, 200, 127, 251)                                      # merged (h, w) -> (H, W)
B_LEVEL = (320, 160, 160, 80)                                      # the level whose right-hand side is stored
DEPTH_STRIDE = {(200, 100): 1, (320, 160): 2, (600, 300): 3}       # final depths are stored at these strides
VIEW, ROOM_SEED = 96, 7


def decode_rows(A, w, h):
    """Row masks in the reference's uncompressed row order (x-gradient h*w; y-gradient (h-1) x (w+1) on the x-wrapped grid, whose
    column w repeats column 0; Laplacian h*w) and each compressed row's index in that order."""
    A = A.tocsr()
    n = h * w
    lap0 = n + (h - 1) * (w + 1)
    dense = np.empty(A.shape[0], np.int64)
    for r in range(A.shape[0]):
        cols, vals = A.indices[A.indptr[r]:A.indptr[r + 1]], A.data[A.indptr[r]:A.indptr[r + 1]]
        if len(cols) > 2:                                          # Laplacian: -4 at the centre (-3 where an edge tap is summed in)
            dense[r] = lap0 + cols[np.argmin(vals)]
        else:
            p, q = cols[vals == 1][0], cols[vals == -1][0]
            i, j = divmod(p, w)
            if q == i * w + (j + 1) % w:
                dense[r] = p
            else:
                dense[r] = n + i * (w + 1) + j
                if j == 0 and r > 0 and dense[r - 1] >= dense[r] and dense[r - 1] < lap0:
                    dense[r] += w                                   # the repeat of column 0 comes after column w - 1
    mask = np.zeros(lap0 + n, bool)
    mask[dense] = True
    return mask, dense


class Recorder:
    def __init__(self, perturb=False):
        self.levels, self.perturb = [], perturb
        self.lsmr = ref.lsmr

    def __call__(self, A, b, **kw):
        if self.perturb:
            b = b.astype(np.float32).astype(np.float64)
        out = self.lsmr(A, b, **kw)
        self.levels.append({"A": A, "b": b, "istop": int(out[1]), "itn": int(out[2])})
        return out


def merge(width, height, dist, masks, extr, intr, perturb=False):
    rec = Recorder(perturb)
    ref.lsmr = rec
    try:
        depth, mask = ref.merge_panorama_depth(width, height, dist, masks, extr, intr)
    finally:
        ref.lsmr = rec.lsmr
    return depth, mask, rec.levels


def level_sizes(width, height):
    sizes = [(width, height)]
    while max(sizes[-1]) > 256:
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    return sizes[::-1]                                             # coarsest first, the order lsmr runs


def main():
    extr, intr = ref.get_panorama_cameras()
    gold = {"extrinsics": torch.from_numpy(np.asarray(extr)), "intrinsics": torch.from_numpy(np.stack(intr)), "split": [],
            "merge": [], "finish": []}
    for k, (H, W, res, seed) in enumerate(SPLIT_CASES):
        img = synthetic_panorama(H, W, seed)
        views = np.stack(ref.split_panorama_image(img, extr, intr, res))
        case = {"H": H, "W": W, "seed": seed, "resolution": res, "views_sha256": array_digest(views)}
        if k == 0:
            case["views"] = torch.from_numpy(views)
        gold["split"].append(case)
        print(f"split {W}x{H} @ {res}")
    dist, masks = synthetic_room_views(VIEW, ROOM_SEED)
    gold["room"] = {"resolution": VIEW, "seed": ROOM_SEED, "inputs_sha256": array_digest(dist, masks)}
    for width, height in MERGE_SIZES:
        depth, mask, levels = merge(width, height, list(dist), list(masks), extr, intr)
        depth_p, _, _ = merge(width, height, list(dist), list(masks), extr, intr, perturb=True)
        sens = float(np.abs(depth_p.astype(np.float64) / depth - 1).max())
        stride = DEPTH_STRIDE[(width, height)]
        case = {"width": width, "height": height, "depth_stride": stride, "depth": torch.from_numpy(depth[::stride, ::stride].copy()),
                "mask": torch.from_numpy(np.packbits(mask)), "sensitivity": sens, "levels": []}
        for (w, h), lv in zip(level_sizes(width, height), levels):
            row_mask, dense = decode_rows(lv["A"], w, h)
            entry = {"width": w, "height": h, "itn": lv["itn"], "istop": lv["istop"],
                     "row_mask": torch.from_numpy(np.packbits(row_mask)), "rows": int(row_mask.size)}
            if (width, height, w, h) == B_LEVEL:
                assert (np.diff(dense) > 0).all()                  # compressed rows are in dense order
                entry["b"] = torch.from_numpy(lv["b"].astype(np.float32))
            case["levels"].append(entry)
            print(f"merge {width}x{height} level {w}x{h}: itn {lv['itn']} istop {lv['istop']} rows {int(row_mask.sum())}")
        print(f"merge {width}x{height}: sensitivity {sens:.3e}")
        gold["merge"].append(case)
        if (height, width) == FINISH[:2]:
            h, w, H, W = FINISH
            gold["finish"].append({"height": h, "width": w, "H": H, "W": W,
                                   "depth": torch.from_numpy(cv2.resize(depth, (W, H), cv2.INTER_LINEAR)),
                                   "mask": torch.from_numpy(np.packbits(cv2.resize(mask.astype(np.uint8), (W, H), cv2.INTER_NEAREST) > 0))})
    torch.save(gold, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
