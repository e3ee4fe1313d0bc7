"""Per-kind table of the encoder from `bench.py --dump-ops` files: the `gemm.*` launches of one step summed by kind (patch
embed, qkv, proj, fc1, fc2, taps projection) and the `attention` launches, with the engine's own flops and bytes, the lower bound they imply (the larger of flops
at the tensor peak and bytes at the HBM peak) and the fraction of it each kind reaches.  With two files (parent, new) it adds the
new time and the change per kind.

    python tools/encoder_table.py ops_base.json [ops_new.json] [--peak-tflops 989] [--hbm-gbs 3350]"""
import argparse
import json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("ops", nargs="+")
    ap.add_argument("--peak-tflops", type=float, default=989.0)
    ap.add_argument("--hbm-gbs", type=float, default=3350.0)
    a = ap.parse_args()
    runs = []
    for f in a.ops:
        kinds = {}
        for o in json.load(open(f)):
            if o["name"].startswith("gemm."):
                name = o["name"][len("gemm."):]
            elif o["name"].startswith("attention"):
                name = "attention"
            else:
                continue
            k = kinds.setdefault(name, {"n": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            k["n"] += 1
            k["ms"] += o["ms"]
            k["flops"] += o["flops"]
            k["bytes"] += o["bytes"]
        runs.append(kinds)
    head = "| kind | launches | GFLOP | MB | bound ms | parent ms | frac |"
    if len(runs) > 1:
        head += " new ms | frac | change |"
    print(head)
    print("|" + "---|" * (head.count("|") - 1))
    tot = [0.0] * len(runs)
    for name, k in runs[0].items():
        bound = max(k["flops"] / (a.peak_tflops * 1e9), k["bytes"] / (a.hbm_gbs * 1e6))
        row = f"| {name} | {k['n']} | {k['flops'] / 1e9:.0f} | {k['bytes'] / 1e6:.0f} | {bound:.3f} |"
        for r, run in enumerate(runs):
            t = run[name]["ms"]
            tot[r] += t
            row += f" {t:.3f} | {bound / t:.2f} |"
        if len(runs) > 1:
            row += f" {100 * (runs[1][name]['ms'] / k['ms'] - 1):+.0f} % |"
        print(row)
    print(f"| all | {sum(k['n'] for k in runs[0].values())} | | | |" + "".join(f" {t:.3f} | |" for t in tot) +
          (f" {100 * (tot[1] / tot[0] - 1):+.0f} % |" if len(runs) > 1 else ""))


if __name__ == "__main__":
    main()
