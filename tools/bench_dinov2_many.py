"""Mixed-shape lists on the DINOv2 backbone (moge_b200.dinov2): `get_intermediate_layers_many` over a list of images of five aspect
ratios against the two ways a caller gets the same outputs without it, one call per shape bucket and one call per image.
ViT-L/14 and ViT-S/14 with synthetic weights, fp16, get_intermediate_layers(n=4); two sets of 32 images (the five shapes in
turn), about 224^2 and about 518^2 pixels each, all sides multiples of 14.  Prints one JSON line with the GPU name and power limit
read in the same run, and writes it to --out.

    python tools/bench_dinov2_many.py [--iters 20] [--out profiles/h100_bench_dinov2_many.json]

Per (model, set) and method (CUDA events around one pass over the whole list, after warm-up passes; median, min and max):
  - ms and images_per_s (from the median);
  - engine_calls: engine calls per pass; ops_per_call: launches in the engine's list of the last call (`engine_ops()`), the
    same for every call of the per-shape and per-image methods;
  - the three methods' outputs are checked to be bitwise equal, per image.
The per-shape method stacks each bucket inside the timed pass, as the list method does.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import capi, dinov2  # noqa: E402
from moge_b200.synthetic import make_dinov2_state_dict, synthetic_dino_input  # noqa: E402

MODELS = (("vitl", dinov2.dinov2_vitl14), ("vits", dinov2.dinov2_vits14))
SETS = {
    "224": [(224, 224), (182, 280), (280, 182), (196, 252), (252, 196)],
    "518": [(518, 518), (420, 644), (644, 420), (462, 574), (574, 462)],
}
IMAGES = 32
N_LAYERS = 4


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_dinov2_many.json"))
    args = ap.parse_args()
    ident = gpu_identity()
    torch.set_grad_enabled(False)
    rows = []
    for size, ctor in MODELS:
        model = ctor(pretrained=False)
        model.load_state_dict(make_dinov2_state_dict(size, 0))
        model = model.to("cuda").half()
        for set_name, shapes in SETS.items():
            images = [synthetic_dino_input(1, *shapes[i % len(shapes)], i)[0].to("cuda").half() for i in range(IMAGES)]
            buckets = {}
            for i, im in enumerate(images):
                buckets.setdefault(tuple(im.shape[1:]), []).append(i)

            def many():
                return model.get_intermediate_layers_many(images, n=N_LAYERS)

            def per_shape():
                out = [None] * IMAGES
                for idx in buckets.values():
                    res = model.get_intermediate_layers(torch.stack([images[i] for i in idx]), n=N_LAYERS)
                    for j, i in enumerate(idx):
                        out[i] = tuple(t[j] for t in res)
                return out

            def per_image():
                return [tuple(t[0] for t in model.get_intermediate_layers(im[None], n=N_LAYERS)) for im in images]

            ref = many()
            geometry = lambda H, W: (None, (H // 14) * (W // 14) + 1)              # noqa: E731
            calls = {"many": len(model._pack_calls(images, geometry, capi.DINO_MAX_GROUPS)), "per_shape": len(buckets),
                     "per_image": IMAGES}
            row = {"model": size, "set": set_name, "shapes": shapes, "images": IMAGES}
            for name, fn in (("many", many), ("per_shape", per_shape), ("per_image", per_image)):
                out = fn()
                assert all(torch.equal(a, b) for o, r in zip(out, ref) for a, b in zip(o, r)), (size, set_name, name)
                t = summary(cuda_samples(fn, args.iters, warmup=2))
                row[name] = {"ms": t, "images_per_s": IMAGES * 1000.0 / t["median"], "engine_calls": calls[name],
                             "ops_per_call": len(model.engine_ops())}
            print(json.dumps(row), file=sys.stderr)
            rows.append(row)
            del images, ref
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    result = {"tool": "bench_dinov2_many", "models": "ViT-L/14 and ViT-S/14 synthetic weights, fp16",
              "call": "get_intermediate_layers(n=4)", **ident, "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(result) + "\n")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
