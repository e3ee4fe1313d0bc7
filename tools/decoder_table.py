"""Per-launch table of the MoGe-2 decoder from `bench.py --dump-ops` files: every conv launch by level and main-loop mode, with the
engine's own flops and bytes, the lower bound they imply (the larger of flops at the tensor peak and bytes at the HBM peak) and the
fraction of it each launch reaches.  With two files (parent, new) it adds the new time and the change per launch.

    python tools/decoder_table.py ops_base.json [ops_new.json] [--peak-tflops 989] [--hbm-gbs 3350]

Modes follow gemm_conv's choice for the ViT-L decoder: 3x3 convs at levels 1-2 (C_in 256 / 128) run CONVH, at level 3
(C_in = 64) CONV64; the folded last-level output convs run CONV64 with the HEADOUT / NECKOUT epilogues; ConvTranspose2d and the
1x1 input blocks run the per-tap GEMM."""
import argparse
import json
import re


def mode_of(name):
    if ".headout." in name:
        return "CONV64 HEADOUT"
    if ".neckout." in name:
        return "CONV64 NECKOUT"
    if name.startswith("conv3x3."):
        return "CONV64" if name.endswith(".l3") else "CONVH"
    return "GEMM (per tap)"


def level_of(name):
    m = re.search(r"\.l(\d)$", name)
    return int(m.group(1)) if m else -1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("ops", nargs="+")
    ap.add_argument("--peak-tflops", type=float, default=989.0)
    ap.add_argument("--hbm-gbs", type=float, default=3350.0)
    a = ap.parse_args()
    runs = [[o for o in json.load(open(f)) if o["name"].startswith("conv")] for f in a.ops]
    head = f"| launch | level | mode | GFLOP | MB | bound ms | parent ms | frac |"
    if len(runs) > 1:
        head += " new ms | frac | change |"
    print(head)
    print("|" + "---|" * (head.count("|") - 1))
    tot = [0.0] * len(runs)
    by_mode = {}
    for i, o in enumerate(runs[0]):
        bound = max(o["flops"] / (a.peak_tflops * 1e9), o["bytes"] / (a.hbm_gbs * 1e6))
        mode = mode_of(o["name"])
        row = f"| {o['name']} | {level_of(o['name'])} | {mode} | {o['flops'] / 1e9:.1f} | {o['bytes'] / 1e6:.0f} | {bound:.3f} |"
        for r, run in enumerate(runs):
            t = run[i]["ms"]
            tot[r] += t
            k = (level_of(o["name"]), mode)
            by_mode.setdefault(k, [0.0] * len(runs))[r] += t
            row += f" {t:.3f} | {bound / t:.2f} |"
        if len(runs) > 1:
            row += f" {100 * (runs[1][i]['ms'] / runs[0][i]['ms'] - 1):+.0f} % |"
        print(row)
    print()
    print("| level | mode | " + " | ".join(f"ms ({f})" for f in a.ops) + " |")
    print("|---|---|" + "---|" * len(runs))
    for (lv, mode), ts in sorted(by_mode.items()):
        print(f"| {lv} | {mode} | " + " | ".join(f"{t:.3f}" for t in ts) + " |")
    print(f"| all | | " + " | ".join(f"{t:.3f}" for t in tot) + " |")


if __name__ == "__main__":
    main()
