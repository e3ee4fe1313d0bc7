"""The DINOv2 backbone on the engine (moge_b200.dinov2) against the oracle's PyTorch restatement of the same encoder
(oracle/dinov2_port.py over oracle/moge_port.py: F.linear, SDPA, F.layer_norm) run in half precision on the same GPU:
ViT-L/14 with synthetic weights, get_intermediate_layers(n=4) at 224 x 224 and 518 x 518, batch 1 and 32.  Prints one JSON line
with the GPU name, power limit and SM clocks read in the same run, and writes it to --out.

    python tools/bench_dinov2.py [--iters 20] [--out profiles/h100_bench_dinov2.json]

Per row (CUDA events around each call, after a warm-up call; median, min and max of the timed calls):
  - engine_ms / port_ms: one call (outputs allocated inside it), engine_images_per_s / port_images_per_s from the medians;
  - max_rel_err: the largest |engine - port| over the port's largest |value|, over the four outputs (16-bit both sides).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200.dinov2 import dinov2_vitl14  # noqa: E402
from moge_b200.synthetic import make_dinov2_state_dict, synthetic_dino_input  # noqa: E402
from oracle.dinov2_port import intermediate_layers  # noqa: E402

SIZES = (224, 518)
BATCHES = (1, 32)


def clocks():
    try:
        q = subprocess.run(["nvidia-smi", "--id=" + os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                            "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        sm, mx = (float(v) for v in q.stdout.strip().split(","))
        return {"sm_clock_mhz": sm, "max_sm_clock_mhz": mx}
    except (OSError, subprocess.SubprocessError, ValueError):
        return {"sm_clock_mhz": None, "max_sm_clock_mhz": None}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_dinov2.json"))
    args = ap.parse_args()
    ident = gpu_identity()
    torch.set_grad_enabled(False)
    sd = make_dinov2_state_dict("vitl", 0)
    model = dinov2_vitl14(pretrained=False)
    model.load_state_dict(sd)
    model = model.to("cuda").half()
    sd16 = {k: v.to("cuda").half() for k, v in sd.items()}
    rows = []
    for S in SIZES:
        for B in BATCHES:
            x = synthetic_dino_input(B, S, S, 0).to("cuda").half()
            eng = lambda: model.get_intermediate_layers(x, n=4)            # noqa: E731
            port = lambda: intermediate_layers(sd16, x, [20, 21, 22, 23], 16)  # noqa: E731
            e, p = eng(), port()
            err = max(float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(e, p))
            te = summary(cuda_samples(eng, args.iters))
            tp = summary(cuda_samples(port, args.iters))
            row = {"size": S, "batch": B, "engine_ms": te, "port_ms": tp, "engine_images_per_s": B * 1000.0 / te["median"],
                   "port_images_per_s": B * 1000.0 / tp["median"], "max_rel_err": err}
            print(json.dumps(row), file=sys.stderr)
            rows.append(row)
            del x, e, p
            torch.cuda.empty_cache()
    result = {"tool": "bench_dinov2", "model": "ViT-L/14 synthetic weights, fp16", "call": "get_intermediate_layers(n=4)", **ident,
              **clocks(), "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(result) + "\n")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
