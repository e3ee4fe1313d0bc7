"""Mixed-size panorama inference on the H100: infer_panoramas_many over a collection of panoramas of several sizes, against one
infer_panoramas call per size and one infer_panorama call per panorama.  Prints one JSON line (profiles/h100_bench_panorama_many.json).

    python tools/bench_panorama_many.py [--steps 5] [--out FILE]

Workload: eight seeded synthetic panoramas, two each of 2048 x 1024, 4096 x 2048 and 1536 x 768 (below the 1920 x 960 merge
cap) and one each of 3840 x 1920 and 1024 x 512, through a synthetic-weight ViT-L MoGe-1 at resolution level 9.  Three arms,
alternated step by step in one process: the list call, one call per size group, one call per panorama.  Per arm: end to end
(the call between CUDA events, the whole collection) and the merge alone (the same views merged as the arm's calls merge them),
both in ms per panorama, median / min / max of --steps.  The arms' outputs are checked bitwise equal.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import panorama as P  # noqa: E402
from moge_b200.synthetic import synthetic_panorama  # noqa: E402

DEV = "cuda:0"
COLLECTION = [(1024, 2048), (2048, 4096), (768, 1536), (1920, 3840), (1024, 2048), (512, 1024), (2048, 4096), (768, 1536)]


def ms(samples, per):
    return {k: round(v, 3) if isinstance(v, float) else v for k, v in summary(samples, per).items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
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
    images = [torch.from_numpy(synthetic_panorama(H, W, seed)).to(DEV) for seed, (H, W) in enumerate(COLLECTION, 1)]
    groups = {}
    for k, image in enumerate(images):
        groups.setdefault(tuple(image.shape[:2]), []).append(k)
    n = len(images)

    def many():
        return P.infer_panoramas_many(model, images)

    def per_size():
        out = [None] * n
        for members in groups.values():
            res = P.infer_panoramas(model, torch.stack([images[k] for k in members]))
            for j, k in enumerate(members):
                out[k] = {key: v[j] for key, v in res.items()}
        return out

    def per_panorama():
        return [P.infer_panorama(model, image) for image in images]

    # the merge alone, on the views of every panorama: one mixed call, one call per size, one call per panorama
    extr, intr = P._default_cameras()
    views, _ = P._split("bench", images, extr, intr, P.SPLIT_RESOLUTION, False)
    fov = P._fov_x(intr, DEV).repeat(n)
    vo = model.infer(views.view(-1, *views.shape[2:]), fov_x=fov, apply_mask=False)
    pts, msk = vo["points"].view(n, 12, *vo["points"].shape[1:]), vo["mask"].view(n, 12, *vo["mask"].shape[1:])
    sizes = [(min(P.MERGE_WIDTH, W), min(P.MERGE_HEIGHT, H)) for H, W in COLLECTION]

    def merge(members):
        return P._merge("bench", [sizes[k] for k in members], pts[members], msk[members], extr, intr, False)

    arms = {"many": (many, lambda: merge(list(range(n)))),
            "per_size": (per_size, lambda: [merge(m) for m in groups.values()]),
            "per_panorama": (per_panorama, lambda: [merge([k]) for k in range(n)])}
    outputs = {k: fn() for k, (fn, _) in arms.items()}               # warm-up: tables, engine plans
    for k, out in outputs.items():
        for a, b in zip(out, outputs["per_panorama"]):
            assert all(torch.equal(a[key], b[key]) for key in ("depth", "mask", "points")), k
    for _, m in arms.values():
        m()
    e2e, merges = {k: [] for k in arms}, {k: [] for k in arms}
    for _ in range(args.steps):                                      # alternated
        for k, (fn, m) in arms.items():
            e2e[k] += cuda_samples(fn, 1, warmup=0)
            merges[k] += cuda_samples(m, 1, warmup=0)
    result = {**gpu, "model": "MoGe-1 ViT-L (synthetic weights), resolution level 9",
              "collection": [f"{W}x{H}" for H, W in COLLECTION], "steps": args.steps, "bitwise_equal": True,
              "end_to_end_ms_per_panorama": {k: ms(v, n) for k, v in e2e.items()},
              "merge_ms_per_panorama": {k: ms(v, n) for k, v in merges.items()}}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
