"""Same-box A/B of library build variants (GPU box).  Each variant is a libmoge_b200_<name>.so built with
`MG_VARIANT=<name> MG_EXTRA_FLAGS=... bash moge_b200/csrc/build.sh`; every measurement runs in its own process (the library is
loaded once per process) and the variants are interleaved `--rounds` times to average out clock / thermal drift.

    python tools/ab_variants.py base polyA polyB [--rounds 3] [--batch 32] [--size vitl] [--tokens 1369] [--res 518]
        ("base" = the product library)  -> per variant: step ms (CUDA events over 5 infer() calls) and per-class ms from the
        engine's own per-launch profile (gemm / attention / conv / other)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r'''
import json, os, sys
sys.path.insert(0, %(root)r)
import torch
from moge.model.v2 import MoGeModel
from moge_b200.configs import model_config
from moge_b200.synthetic import make_state_dict
cfg = model_config(%(size)r, True)
m = MoGeModel(**cfg); m.load_state_dict(make_state_dict(cfg, 0)); m = m.to("cuda").eval()
if %(dtype)r == "bf16": m = m.bfloat16()
x = torch.rand(%(batch)d, 3, %(res)d, %(res)d, generator=torch.Generator().manual_seed(1)).cuda()
for _ in range(3): m.infer(x, num_tokens=%(tokens)d)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5): m.infer(x, num_tokens=%(tokens)d)
e1.record(); torch.cuda.synchronize()
ops = m.engine_ops()
prof = [m.engine_profile() for _ in range(3)]
ms = [min(p[i] for p in prof) for i in range(len(ops))]
cls = {}
for (n, f, b), t in zip(ops, ms):
    k = "gemm" if n.startswith("gemm.") else "attention" if n.startswith("attention") else "conv" if n.startswith("conv") else "other"
    cls[k] = cls.get(k, 0.0) + t
byname = {}
for (n, f, b), t in zip(ops, ms):
    byname[n] = byname.get(n, 0.0) + t
print(json.dumps({"step_ms": e0.elapsed_time(e1) / 5, "classes": cls, "byname": byname}))
'''


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("variants", nargs="+")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", default="vitl")
    ap.add_argument("--tokens", type=int, default=1369)
    ap.add_argument("--res", type=int, default=518)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--names", default="", help="comma-separated op-name prefixes to print per variant")
    a = ap.parse_args()
    res = {v: [] for v in a.variants}
    code = CHILD % dict(root=ROOT, size=a.size, batch=a.batch, res=a.res, tokens=a.tokens, dtype=a.dtype)
    for r in range(a.rounds):
        for v in a.variants:
            env = dict(os.environ)
            env.pop("MOGE_B200_LIB", None)
            if v != "base":
                env["MOGE_B200_LIB"] = os.path.join(ROOT, "moge_b200", "_lib", f"libmoge_b200_{v}.so")
            try:
                out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=240)
            except subprocess.TimeoutExpired:
                print(v, "TIMEOUT")
                continue
            if out.returncode != 0:
                print(v, "FAILED", out.stderr[-800:])
                continue
            res[v].append(json.loads(out.stdout.strip().splitlines()[-1]))
    prefixes = [p for p in a.names.split(",") if p]
    for v, rows in res.items():
        if not rows:
            continue
        step = sorted(r["step_ms"] for r in rows)
        line = f"{v:12s} step_ms min {step[0]:.3f} med {step[len(step) // 2]:.3f} |"
        for k in ("gemm", "attention", "conv", "other"):
            vals = sorted(r["classes"].get(k, 0.0) for r in rows)
            line += f" {k} {vals[0]:.3f}"
        print(line)
        for p in prefixes:
            vals = sorted(sum(t for n, t in r["byname"].items() if n.startswith(p)) for r in rows)
            print(f"    {p:40s} min {vals[0]:.4f} med {vals[len(vals) // 2]:.4f}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
