"""Where the engine's fp16 deviation from the fp32 reference is born (DESIGN.md section 2, "normal tolerance").

Runs on the GPU:  python tools/error_attribution.py [--out error_attribution.json]

Three measurements on the benchmarked shape (ViT-L, 518x518, 37x37 grid), for a plain random-init checkpoint and for the
`well_posed` one (near-unit raw normals, like a trained model):

 1. engine (fp16) vs the oracle port in fp32 on the same GPU (TF32 off): rel-L2 per forward() output;
 2. the F.normalize amplification: statistics of the RAW (pre-normalize) normal-head output |n| of the oracle,
    sqrt(E[1/|n|^2] E[|n|^2]) (= the factor by which a uniform relative error of the raw vector grows through v2.py:178), and the
    engine's normal error split by |n| quantile;
 3. rounding-site sensitivity: the oracle with 16-bit rounding of operands / stored activations switched on at ONE site class at
    a time (encoder linears, attention operands, decoder level l convs, head output conv), everything else fp32 -- the error
    each site class alone produces -- and with all of them on (the arithmetic model of the engine and of the reference's .half()).

TEST INFRASTRUCTURE: imports oracle/ (the checker), never imported by the product path.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from moge.model.v2 import MoGeModel  # noqa: E402
from moge_b200.configs import model_config, token_grid  # noqa: E402
from moge_b200.synthetic import make_state_dict, synthetic_images  # noqa: E402
from oracle import moge_port  # noqa: E402

DEV = "cuda"


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def r16(t):
    return t.half().float()


class Sites:
    """Monkeypatches the torch.nn.functional entry points the oracle calls so that selected site classes round like a 16-bit path:
    operands (activation + weight) to fp16, fp32 accumulation, result rounded to fp16 where the engine stores it in 16 bit."""

    def __init__(self, h, w):
        self.h, self.w, self.on = h, w, set()
        self.orig = {k: getattr(F, k) for k in ("linear", "conv2d", "conv_transpose2d", "scaled_dot_product_attention")}

    def level(self, x):
        hh = x.shape[-2]
        for l in range(5):
            if hh in (self.h << l, (self.h << l) + 2):          # (+2: replicate-padded input of a 3x3 conv)
                return l
        return -1

    def __enter__(self):
        S = self

        def linear(x, w, b=None):
            if "enc.linear" in S.on and x.dim() == 3:
                return r16(S.orig["linear"](r16(x), r16(w), b))
            return S.orig["linear"](x, w, b)

        def sdpa(q, k, v, *a, **kw):
            if "enc.attention" in S.on:
                return r16(S.orig["scaled_dot_product_attention"](r16(q), r16(k), r16(v), *a, **kw))
            return S.orig["scaled_dot_product_attention"](q, k, v, *a, **kw)

        def conv2d(x, w, b=None, *a, **kw):
            if x.shape[1] == 3 and w.shape[-1] == 14:           # patch embed
                if "enc.linear" in S.on:
                    return S.orig["conv2d"](r16(x), r16(w), b, *a, **kw)
                return S.orig["conv2d"](x, w, b, *a, **kw)
            l = S.level(x)
            key = "dec.l%d" % l
            if w.shape[0] <= 3 and w.shape[-1] == 1:            # head output block (folded into the last conv in the engine: fp32 out)
                key = "dec.headout"
            if key in S.on:
                y = S.orig["conv2d"](r16(x), r16(w), b, *a, **kw)
                return y if key == "dec.headout" else r16(y)
            return S.orig["conv2d"](x, w, b, *a, **kw)

        def convT(x, w, b=None, *a, **kw):
            key = "dec.l%d" % S.level(x)
            if key in S.on:
                return r16(S.orig["conv_transpose2d"](r16(x), r16(w), b, *a, **kw))
            return S.orig["conv_transpose2d"](x, w, b, *a, **kw)

        F.linear, F.conv2d, F.conv_transpose2d, F.scaled_dot_product_attention = linear, conv2d, convT, sdpa
        return self

    def __exit__(self, *exc):
        for k, v in self.orig.items():
            setattr(F, k, v)


def oracle_fwd(cfg, sdd, img, nt, capture_raw=None):
    orig = F.normalize
    if capture_raw is not None:
        def fake(x, dim=-1, **kw):
            capture_raw["n"] = x.detach().clone()
            return orig(x, dim=dim, **kw)
        F.normalize = fake
    try:
        return moge_port.forward(cfg, sdd, img, nt)
    finally:
        F.normalize = orig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="error_attribution.json")
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = model_config("vitl", True)
    H = W = 518
    nt = 1369
    h, w = token_grid(H, W, nt)
    report = {"shape": "ViT-L, 1 x 518x518, 37x37 grid, fp16 engine vs fp32 oracle on the same GPU (TF32 off)", "cases": []}
    for label, seed, wp in (("plain random init", 5, False), ("well_posed (near-unit raw normals)", 10, True)):
        sd = make_state_dict(cfg, seed, well_posed=wp)
        sdd = {k: v.to(DEV) for k, v in sd.items()}
        img = synthetic_images(1, H, W, seed).to(DEV)
        raw = {}
        ref = oracle_fwd(cfg, sdd, img, nt, raw)
        model = MoGeModel(**cfg)
        model.load_state_dict(sd)
        model = model.to(DEV).eval()
        out = model.forward(img, nt)
        torch.cuda.synchronize()
        case = {"checkpoint": label, "seed": seed, "engine_vs_fp32": {k: rel(out[k], ref[k]) for k in ref}}
        n = raw["n"][0].norm(dim=-1)                                   # (Hl, Wl) raw |n| at the head's own resolution
        amp = float(((1 / n ** 2).mean() * (n ** 2).mean()).sqrt())
        case["raw_normal"] = {"norm_quantiles_1_10_50_90": [float(q) for q in torch.quantile(n.flatten().float(), torch.tensor([0.01, 0.1, 0.5, 0.9], device=n.device))],
                              "normalize_amplification_sqrt(E[1/n^2]E[n^2])": amp}
        # engine normal error by |n| of the reference at the output resolution
        nref = F.interpolate(raw["n"].permute(0, 3, 1, 2), (H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)[0].norm(dim=-1)
        err = (out["normal"][0] - ref["normal"][0]).norm(dim=-1)
        qs = torch.quantile(nref.flatten(), torch.tensor([0.25, 0.5, 0.75], device=nref.device))
        bins = [(None, qs[0]), (qs[0], qs[1]), (qs[1], qs[2]), (qs[2], None)]
        split = []
        for lo, hi in bins:
            m = torch.ones_like(nref, dtype=torch.bool)
            if lo is not None:
                m &= nref >= lo
            if hi is not None:
                m &= nref < hi
            split.append(float((err[m] ** 2).mean().sqrt()))
        case["engine_normal_rms_error_by_raw_norm_quartile(low..high)"] = split
        # rounding-site sensitivity in the oracle
        sites = ["enc.linear", "enc.attention", "dec.l0", "dec.l1", "dec.l2", "dec.l3", "dec.l4", "dec.headout"]
        table = {}
        with Sites(h, w) as S:
            for s in sites + ["ALL"]:
                S.on = set(sites) if s == "ALL" else {s}
                o = oracle_fwd(cfg, sdd, img, nt)
                table[s] = {k: rel(o[k], ref[k]) for k in ("points", "normal", "mask")}
        case["oracle_rounding_site_sensitivity"] = table
        case["quadrature_sum_of_single_sites"] = {k: float(sum(table[s][k] ** 2 for s in sites) ** 0.5) for k in ("points", "normal", "mask")}
        report["cases"].append(case)
        print(json.dumps(case, indent=1))
        del model
    with open(a.out, "w") as fh:
        json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
