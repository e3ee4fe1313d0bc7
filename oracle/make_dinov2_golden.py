"""Generate tests/golden/dinov2.pt from the UNMODIFIED reference DINOv2 backbone (moge/model/dinov2, CPU, fp32).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_dinov2_golden.py

The backbones are built by the reference's hub constructors (hub/backbones.py, pretrained=False) and loaded, strictly, with the
seeded synthetic state dicts of moge_b200.synthetic.make_dinov2_state_dict; the inputs come from synthetic_dino_input.  So the
file stores each case's recipe (size, seed, batch, H, W, the call and its arguments) and the reference's outputs, not the inputs.
Of each patch-token output it keeps 16 tokens (the first, the last and a seeded sample; all of a grid of 16 or fewer) and their
indices, which keeps the file small; class tokens are kept whole.  The maker also checks oracle/dinov2_port.py against the
reference on the full outputs of every get_intermediate_layers case, so that the GPU tests can compare every token with the port
and the kept ones with the reference.  The cases:
- ViT-S/14 at 224 x 224, 98 x 126, 126 x 98 and 14 x 518 (a 1 x 37 grid), and ViT-B/14 at 98 x 126;
- get_intermediate_layers with an int n and with a list of blocks, norm on and off, reshape on and off, return_class_token;
- forward_features (its tensors) and forward (the class token).
The key list of the reference's state dict is stored too, for the alias's load_state_dict.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")
sys.path.insert(0, os.environ["MOGE_REFERENCE"])      # `moge` is the reference's, `moge_b200` this tree's

import torch  # noqa: E402

from moge_b200.synthetic import make_dinov2_state_dict, synthetic_dino_input  # noqa: E402
from oracle.dinov2_port import intermediate_layers  # noqa: E402

from moge.model.dinov2.hub import backbones as ref_hub  # noqa: E402  (the real reference)

assert ref_hub.__file__.startswith(os.path.abspath(os.environ["MOGE_REFERENCE"])), ref_hub.__file__
OUT = os.path.join(ROOT, "tests", "golden", "dinov2.pt")
CTORS = {"vits": ref_hub.dinov2_vits14, "vitb": ref_hub.dinov2_vitb14}

# (size, seed, B, H, W, [(call, kwargs)])
CASES = [
    ("vits", 0, 1, 224, 224, [("gil", dict(n=1, return_class_token=True)),
                              ("gil", dict(n=[7], reshape=True, norm=False)),
                              ("forward", {})]),
    ("vits", 1, 2, 98, 126, [("gil", dict(n=2, reshape=True, return_class_token=True)),
                             ("gil", dict(n=[0, 7], norm=False, return_class_token=True)),
                             ("forward_features", {})]),
    ("vits", 2, 1, 126, 98, [("gil", dict(n=1)),
                             ("gil", dict(n=[3, 11], reshape=True, norm=False, return_class_token=True))]),
    ("vits", 3, 1, 14, 518, [("gil", dict(n=4, reshape=True, return_class_token=True)),
                             ("forward_features", {})]),
    ("vitb", 4, 1, 98, 126, [("gil", dict(n=[5, 11], return_class_token=True)),
                             ("gil", dict(n=2, reshape=True, norm=False)),
                             ("forward", {})]),
]


KEEP_TOKENS = 16         # patch tokens kept per output: the first, the last and a seeded sample between them


def token_sample(T: int, seed: int) -> torch.Tensor:
    """Sorted patch-token indices kept of a T-token grid: all of them when T <= KEEP_TOKENS."""
    if T <= KEEP_TOKENS:
        return torch.arange(T)
    g = torch.Generator().manual_seed(1000 + seed)
    inner = torch.randperm(T - 2, generator=g)[:KEEP_TOKENS - 2] + 1
    return torch.cat([torch.tensor([0, T - 1]), inner]).sort().values


def pick(t: torch.Tensor, idx: torch.Tensor, channel_major: bool) -> torch.Tensor:
    """The kept tokens of a (B, T, D) or (B, D, h, w) output: (B, k, D) or (B, D, k), as a compact copy."""
    return (t.flatten(2)[:, :, idx] if channel_major else t[:, idx]).clone()


def run(model, call, kw, x, idx):
    """The call's outputs with the patch tokens (and the pre-norm stream's rows: the class row, then the kept tokens) reduced to
    the kept ones; class tokens whole."""
    chw = bool(kw.get("reshape"))
    if call == "gil":
        out = model.get_intermediate_layers(x, **kw)
        return [(pick(o[0], idx, chw), o[1].clone()) if isinstance(o, tuple) else pick(o, idx, chw) for o in out]
    if call == "forward_features":
        d = model.forward_features(x)
        rows = torch.cat([torch.tensor([0]), idx + 1])
        return {"x_norm_clstoken": d["x_norm_clstoken"].clone(), "x_norm_regtokens": d["x_norm_regtokens"].clone(),
                "x_norm_patchtokens": pick(d["x_norm_patchtokens"], idx, False), "x_prenorm": pick(d["x_prenorm"], rows, False)}
    return model(x).clone()


def check_port(model, sd, x, kw):
    """oracle/dinov2_port.py, which the GPU tests use to check every token, against the reference on the full outputs."""
    ref = model.get_intermediate_layers(x, n=kw["n"], norm=kw.get("norm", True))
    layers = [i for i in range(model.n_blocks) if i in (range(model.n_blocks - kw["n"], model.n_blocks) if isinstance(kw["n"], int)
                                                       else kw["n"])]
    port = intermediate_layers(sd, x, layers, model.num_heads, norm=kw.get("norm", True))
    for r, p in zip(ref, port):
        err = float((r - p).abs().max() / r.abs().max())
        assert err < 1e-5, err


def main():
    torch.set_grad_enabled(False)
    cases, keys = [], {}
    for size, seed, B, H, W, calls in CASES:
        model = CTORS[size](pretrained=False).eval()
        sd = make_dinov2_state_dict(size, seed)
        model.load_state_dict(sd, strict=True)
        keys[size] = list(model.state_dict().keys())
        x = synthetic_dino_input(B, H, W, seed)
        idx = token_sample((H // 14) * (W // 14), seed)
        for call, kw in calls:
            if call == "gil":
                check_port(model, sd, x, kw)
            cases.append({"size": size, "seed": seed, "shape": (B, H, W), "call": call, "kwargs": kw, "tokens": idx,
                          "out": run(model, call, kw, x, idx)})
            print(size, seed, (B, H, W), call, kw)
    torch.save({"cases": cases, "keys": keys}, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
