"""Generate tests/golden/v1_*.pt from the UNMODIFIED reference MoGe-1 (CPU only).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_v1_golden.py [--only name,...]

For every case the script builds the reference `moge.model.v1.MoGeModel(**cfg)`, loads the seeded synthetic state dict from
moge_b200.synthetic with strict=True (pins key names and shapes), runs the reference `forward()` / `infer()` in fp32, asserts that
oracle/moge_v1_port.py reproduces both, and stores the reference's outputs (at a pixel stride for large shapes) together with its
own fp16 / bf16 autocast deviation.  Inputs are regenerated from the seed by the tests.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "utils3d_shim"))
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")
sys.path.insert(1, os.environ["MOGE_REFERENCE"])

import torch  # noqa: E402

from moge_b200.configs import v1_model_config  # noqa: E402
from moge_b200.synthetic import make_v1_state_dict, synthetic_images  # noqa: E402
from oracle import moge_v1_port  # noqa: E402

from moge.model.v1 import MoGeModel as RefModel  # noqa: E402  (the real reference)

OUT = os.path.join(ROOT, "tests", "golden")

# name, size, seed, (B,H,W), num_tokens (None = resolution level 9), store stride, options
#   options: remap (overrides remap_output), autocast (store the reference's own 16-bit deviation), infer (extra infer() calls:
#   list of kwargs dicts beyond the default one)
CASES = [
    ("v1_vitl_b1_518x518_default_wp", "vitl", 20, (1, 518, 518), None, 4, {"autocast": True}),
    ("v1_vitl_b1_518x1036_default_wp", "vitl", 21, (1, 518, 1036), None, 8, {}),       # 494x989, grid 35x70
    ("v1_vitl_b1_1036x518_default_wp", "vitl", 22, (1, 1036, 518), None, 8, {}),
    ("v1_vitl_b1_1024x768_default_wp", "vitl", 23, (1, 1024, 768), None, 8, {}),       # bicubic DOWN-sampling to 808x606
    ("v1_vits_b2_126x168_t192_wp", "vits", 24, (2, 126, 168), 192, 3,
     {"autocast": True, "infer": [{"fov_x": 60.0}, {"apply_mask": False}, {"force_projection": False}]}),
    ("v1_vits_b1_98x126_t120_linear", "vits", 25, (1, 98, 126), 120, 1, {"remap": "linear"}),
    ("v1_vits_b1_98x126_t120_sinh", "vits", 26, (1, 98, 126), 120, 1, {"remap": "sinh"}),
    ("v1_vits_b1_98x126_t120_sinh_exp", "vits", 27, (1, 98, 126), 120, 1, {"remap": "sinh_exp"}),
]


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def infer_key(kw):
    return ",".join(f"{k}={v}" for k, v in sorted(kw.items())) or "default"


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, help="comma-separated substrings of the case names to generate")
    a = ap.parse_args()
    only = a.only.split(",") if a.only else None
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    for name, size, seed, (B, H, W), tokens, stride, opt in CASES:
        if only and not any(o in name for o in only):
            continue
        cfg = v1_model_config(size)
        if "remap" in opt:
            cfg["remap_output"] = opt["remap"]
        well_posed = name.endswith("_wp")
        sd = make_v1_state_dict(cfg, seed, well_posed=well_posed)
        ref = RefModel(**cfg).eval()
        ref.load_state_dict(sd, strict=True)
        img = synthetic_images(B, H, W, seed)
        lo, hi = cfg["num_tokens_range"]
        nt = tokens if tokens is not None else int(lo + (9 / 9) * (hi - lo))
        report, dev16, infers = {}, {}, {}
        with torch.no_grad():
            fwd = ref.forward(img, nt)
            for tag, dt_ in ((("fp16", torch.float16), ("bf16", torch.bfloat16)) if opt.get("autocast") else ()):
                with torch.autocast("cpu", dtype=dt_):
                    f16 = ref.forward(img, nt)
                dev16[tag] = {k: rel_l2(f16[k].float(), fwd[k]) for k in fwd}
            pf = moge_v1_port.forward(cfg, sd, img, nt)
            for k in fwd:
                report["fwd." + k] = rel_l2(pf[k], fwd[k])
                assert report["fwd." + k] < 2e-5, (name, k, report)
            for kw in [{}] + opt.get("infer", []):
                inf = ref.infer(img, num_tokens=tokens, use_fp16=False, **kw)
                pi = moge_v1_port.infer(cfg, sd, img, num_tokens=tokens, **kw)
                m = inf["mask"]
                assert bool((pi["mask"] == m).float().mean() > 0.9999), name
                both = m & pi["mask"]
                key = infer_key(kw)
                for k in ("points", "depth"):
                    report[f"inf[{key}].{k}"] = rel_l2(pi[k][both], inf[k][both])
                    assert report[f"inf[{key}].{k}"] < 1e-4, (name, key, k, report)
                report[f"inf[{key}].intrinsics"] = rel_l2(pi["intrinsics"], inf["intrinsics"])
                assert report[f"inf[{key}].intrinsics"] < 1e-4, (name, report)
                sl = (slice(None), slice(None, None, stride), slice(None, None, stride))
                infers[key] = {"kwargs": kw, **{k: (v[sl].contiguous() if k != "intrinsics" else v) for k, v in inf.items()}}
        print(name, {k: f"{v:.2e}" for k, v in report.items()}, "mask_frac", float(fwd["mask"].gt(0.5).float().mean()))
        print("   reference autocast deviation:", {t: {k: f"{v:.1e}" for k, v in d.items()} for t, d in dev16.items()})
        sl = (slice(None), slice(None, None, stride), slice(None, None, stride))
        gold = {
            "meta": {"size": size, "seed": seed, "shape": (B, H, W), "num_tokens": tokens, "stride": stride, "options": dict(opt),
                     "remap_output": cfg["remap_output"], "well_posed": well_posed, "port_vs_reference": report,
                     "reference_autocast_deviation": dev16},
            "forward": {k: v[sl].contiguous() for k, v in fwd.items()},
            "infer": infers,
        }
        path = os.path.join(OUT, name + ".pt")
        torch.save(gold, path)
        assert os.path.getsize(path) <= 1_000_000, (path, os.path.getsize(path))


if __name__ == "__main__":
    main()
