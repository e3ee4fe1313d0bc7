"""MoGe-1 throughput and latency on one GPU: ViT-L (configs/train/v1.json) fp16, 518x518 at the default resolution level 9
(2500 tokens: resized to 700x700, 50x50 token grid), seeded synthetic weights and images.

    python tools/bench_v1.py [--batch 32] [--steps 10] [--iters 200]
    python tools/bench_v1.py --many [--steps 10] [--warmup 2]

Prints one JSON line: engine images/s at --batch, engine batch-1 p50 / p90 over --iters calls after warm-up (each call timed with
CUDA events around forward()), the oracle port (oracle/moge_v1_port.py, plain PyTorch) in .half() on the same GPU as the
comparator, the rel-L2 agreement of the two, the engine's per-kernel-class split (engine_profile(), batch 1) and the GPU name
and power limit.  Writes nothing to the tree.

--many measures mixed-shape batches instead: the five aspect ratios of `bench.py --config 3` (W x H 1036x518, 777x518, 518x518,
518x777, 518x1036), as 32 images (7, 7, 6, 6, 6) and as 5 (one each), at resolution levels 9 and 0 (2500 and 1200 tokens).  Each
workload is run three ways: infer_many(all images), a loop of infer() over single images, and one infer() per shape bucket.  The
three are timed in turn, one step each, --steps times (CUDA events around the step), so that clock drift spreads over all three;
images/s is reported as the median and range over the steps.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--many", action="store_true", help="the mixed-shape workloads (infer_many) instead")
    a = ap.parse_args()
    gpu = gpu_identity()
    if a.many:
        return run_many(a, gpu)
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict, synthetic_images
    from oracle import moge_v1_port

    dev = "cuda:0"
    cfg = v1_model_config("vitl")
    sd = make_v1_state_dict(cfg, 0, well_posed=True)
    model = MoGeModel(**cfg)
    model.load_state_dict(sd)
    model = model.to(dev).half()
    tokens = 2500
    img1 = synthetic_images(1, 518, 518, 0).to(dev)
    imgB = synthetic_images(a.batch, 518, 518, 1).to(dev)

    # batch 1 latency
    t1 = cuda_samples(lambda: model.forward(img1, tokens), a.iters, a.warmup)
    # throughput at --batch
    for _ in range(2):
        model.forward(imgB, tokens)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        model.forward(imgB, tokens)
    torch.cuda.synchronize()
    ips = a.batch * a.steps / (time.perf_counter() - t0)

    # per-kernel-class split of one batch-1 forward
    model.forward(img1, tokens)
    torch.cuda.synchronize()
    ops, ms = model.engine_ops(), model.engine_profile()
    split = {}
    for (name, _, _), t in zip(ops, ms):
        cls = name.split(".")[0]
        split[cls] = split.get(cls, 0.0) + t

    # comparator: the oracle port in fp16 on the same GPU
    sd16 = {k: v.to(dev).half() for k, v in sd.items()}
    with torch.inference_mode():
        def port1():
            return moge_v1_port.forward(cfg, sd16, img1.half(), tokens)
        tp = cuda_samples(port1, 20, 3)
        nb = min(a.batch, 8)
        port_b = lambda: moge_v1_port.forward(cfg, sd16, imgB[:nb].half(), tokens)  # noqa: E731
        port_b()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(3):
            port_b()
        torch.cuda.synchronize()
        port_ips = nb * 3 / (time.perf_counter() - t0)
        # agreement: engine fp16 vs the port in fp32 on the same image
        sd32 = {k: v.to(dev) for k, v in sd.items()}
        ref = moge_v1_port.forward(cfg, sd32, img1, tokens)
        out = model.forward(img1, tokens)
        agree = {k: float(((out[k].double() - ref[k].double()).norm() / ref[k].double().norm()).item()) for k in ("points", "mask")}

    q = statistics.quantiles(t1, n=10)
    print(json.dumps({
        "workload": "MoGe-1 ViT-L fp16, 518x518, resolution level 9 (2500 tokens, 700x700, grid 50x50), synthetic weights",
        **gpu,
        "engine": {"images_per_s": round(ips, 2), "batch": a.batch, "steps": a.steps,
                   "batch1_p50_ms": round(statistics.median(t1), 3), "batch1_p90_ms": round(q[8], 3), "batch1_iters": a.iters},
        "port_fp16": {"batch1_p50_ms": round(statistics.median(tp), 3), "images_per_s": round(port_ips, 2), "batch": nb},
        "speedup_batch1": round(statistics.median(tp) / statistics.median(t1), 2),
        "agreement_rel_l2_vs_port_fp32": agree,
        "kernel_class_ms_batch1": {k: round(v, 4) for k, v in sorted(split.items(), key=lambda kv: -kv[1])},
    }))


MANY_SHAPES = [(518, 1036, 7), (518, 777, 7), (518, 518, 6), (777, 518, 6), (1036, 518, 6)]      # (H, W, images), bench.py --config 3


def run_many(a, gpu):
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import default_num_tokens, v1_model_config, v1_resized_size
    from moge_b200.synthetic import make_v1_state_dict

    dev = "cuda:0"
    cfg = v1_model_config("vitl")
    model = MoGeModel(**cfg)
    model.load_state_dict(make_v1_state_dict(cfg, 0, well_posed=True))
    model = model.to(dev).half()
    g = torch.Generator().manual_seed(7)
    workloads = []
    for per_shape in (True, False):
        counts = [n if per_shape else 1 for (_, _, n) in MANY_SHAPES]
        batches = [torch.rand(n, 3, H, W, generator=g).to(dev) for (H, W, _), n in zip(MANY_SHAPES, counts)]
        images = [im for b in batches for im in b]
        for level in (9, 0):
            tokens = default_num_tokens(cfg["num_tokens_range"], level)
            modes = {
                "infer_many": lambda: model.infer_many(images, resolution_level=level),
                "per_image_infer": lambda: [model.infer(im, resolution_level=level) for im in images],
                "per_bucket_infer": lambda: [model.infer(b, resolution_level=level) for b in batches],
            }
            with torch.inference_mode():
                for _ in range(a.warmup):
                    for fn in modes.values():
                        fn()
                ms = {k: [] for k in modes}
                for _ in range(a.steps):
                    for k, fn in modes.items():
                        ms[k] += cuda_samples(fn, 1, 0)
                many = model.infer_many(images, resolution_level=level)
                one = [model.infer(im, resolution_level=level) for im in images]
                agree = max(float(((x["depth"][x["mask"]].double() - y["depth"][x["mask"]].double()).norm()
                                   / y["depth"][x["mask"]].double().norm()).item()) for x, y in zip(many, one))
            nimg = len(images)
            rates = {k: sorted(nimg / (t / 1e3) for t in v) for k, v in ms.items()}
            workloads.append({
                "images": nimg, "resolution_level": level, "num_tokens": tokens,
                "shapes": [f"{n} x {W}x{H} -> {'x'.join(map(str, v1_resized_size(H, W, tokens)[::-1]))}"
                           for (H, W, _), n in zip(MANY_SHAPES, counts)],
                **{k: {"images_per_s_median": round(r[len(r) // 2], 2), "images_per_s_min": round(r[0], 2),
                       "images_per_s_max": round(r[-1], 2), "steps": len(r)} for k, r in rates.items()},
                "infer_many_vs_per_image_depth_rel_l2_max": agree,
            })
    print(json.dumps({
        "workload": "MoGe-1 ViT-L fp16, synthetic weights and images; mixed-aspect batches (bench.py --config 3 aspects): "
                    "infer_many vs a loop of per-image infer() vs one infer() per shape bucket (W x H -> resized W x H)",
        **gpu, "steps": a.steps, "warmup": a.warmup, "workloads": workloads,
    }))


if __name__ == "__main__":
    main()
