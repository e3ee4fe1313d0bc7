"""CPU: the oracle port (oracle/moge_port.py) against the golden vectors produced by the unmodified
reference (oracle/make_golden.py).  Pins the oracle before it is trusted as the GPU checker."""
import os

import pytest
import torch

from moge_b200.configs import model_config, token_grid, default_num_tokens
from moge_b200.synthetic import make_state_dict, synthetic_images, synthetic_point_map
from oracle import moge_port
from golden_io import load_golden

FAST_CASES = ["vits_b1_126x168_t192", "vits_b2_140x98_t117", "vitb_b1_98x154_t150_nonormal", "vits_b2_126x168_t192_wp",
              "vits_b1_98x126_t120_linear", "vits_b1_98x126_t120_sinh", "vits_b1_98x126_t120_sinh_exp"]


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("name", FAST_CASES)
def test_port_matches_reference_golden(name, golden_dir):
    gold = load_golden(golden_dir, name)
    meta = gold["meta"]
    opt = meta.get("options", {})
    cfg = model_config(meta["size"], meta["with_normal"])
    if "remap" in opt:
        cfg["remap_output"] = opt["remap"]
    sd = make_state_dict(cfg, meta["seed"], well_posed=opt.get("well_posed", False))
    B, H, W = meta["shape"]
    img = synthetic_images(B, H, W, meta["seed"])
    s = meta["stride"]
    nt = meta["num_tokens"] or default_num_tokens(cfg["num_tokens_range"])
    fwd = moge_port.forward(cfg, sd, img, nt)
    for k, ref in gold["forward"].items():
        got = fwd[k][:, ::s, ::s] if fwd[k].dim() >= 3 else fwd[k]
        assert rel_l2(got, ref) < 2e-5, k
    inf = moge_port.infer(cfg, sd, img, num_tokens=meta["num_tokens"])
    m = gold["infer"]["mask"]
    assert (inf["mask"][:, ::s, ::s] == m).float().mean() > 0.9999
    for k in ("points", "depth", "normal"):
        if k in gold["infer"]:
            got = inf[k][:, ::s, ::s]
            assert rel_l2(got[m], gold["infer"][k][m]) < 1e-4, k
    assert rel_l2(inf["intrinsics"], gold["infer"]["intrinsics"]) < 1e-5


def test_port_focal_shift_golden(golden_dir):
    cases = torch.load(os.path.join(golden_dir, "recover_focal_shift.pt"), weights_only=False)
    for c in cases:
        pts, mask = synthetic_point_map(*c["args"][:7], seed=c["args"][7])
        f, s = moge_port.recover_focal_shift(pts, mask, focal=c["focal_in"])
        assert torch.allclose(f, c["focal"], rtol=1e-5, atol=1e-6)
        assert torch.allclose(s, c["shift"], rtol=1e-5, atol=1e-6)


def test_token_grid_matches_reference_rounding():
    # v2.py:142-147, Python round (half-to-even); values from SURVEY.md section 8 preamble
    assert token_grid(518, 518, 1369) == (37, 37)
    assert token_grid(518, 518, 3600) == (60, 60)
    assert token_grid(518, 1036, 700) == (19, 37)
    assert token_grid(518, 777, 700) == (22, 32)
    assert token_grid(1036, 518, 700) == (37, 19)
    assert default_num_tokens([1200, 3600], 9) == 3600
    assert default_num_tokens([1200, 3600], 0) == 1200
    assert default_num_tokens([1200, 3600], 5) == 2533
