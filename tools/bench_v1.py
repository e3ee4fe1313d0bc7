"""MoGe-1 throughput and latency on one GPU: ViT-L (configs/train/v1.json) fp16, 518x518 at the default resolution level 9
(2500 tokens: resized to 700x700, 50x50 token grid), seeded synthetic weights and images.

    python tools/bench_v1.py [--batch 32] [--steps 10] [--iters 200]

Prints one JSON line: engine images/s at --batch, engine batch-1 p50 / p90 over --iters calls after warm-up (each call timed with
CUDA events around forward()), the oracle port (oracle/moge_v1_port.py, plain PyTorch) in .half() on the same GPU as the
comparator, the rel-L2 agreement of the two, the engine's per-kernel-class split (engine_profile(), batch 1) and the GPU name
and power limit.  Writes nothing to the tree.
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
    a = ap.parse_args()
    gpu = gpu_identity()
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


if __name__ == "__main__":
    main()
