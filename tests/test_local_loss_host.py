"""moge_b200.local_loss, the sampled local loss, on the CPU side: the golden's inputs and draws (tests/golden/local_loss.pt,
oracle/make_local_loss_golden.py), the plain-torch port against the golden, the public names, and CPU tensors rejected before
any launch."""
import math
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from moge_b200 import local_loss as L  # noqa: E402
from moge_b200.capi import MogeError  # noqa: E402
from moge_b200.synthetic import array_digest, synthetic_loss_case  # noqa: E402
from oracle.utils3d_metrics import install  # noqa: E402

install()
from oracle import local_loss_port as port  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "local_loss.pt")
CASES = torch.load(GOLDEN, weights_only=False)


def case_inputs(c):
    inputs = synthetic_loss_case(c["seed"], c["batch_shape"], c["H"], c["W"], empty_image=c["empty_image"])
    g = torch.Generator().manual_seed(6000 + c["seed"])
    focal = 0.15 + 0.15 * torch.rand(c["batch_shape"], generator=g)
    return inputs["pred_points"], inputs["gt_points"], focal


def case_draws(c):
    """The two offset tensors regenerated from the case's seed, and the recorded selection."""
    H, W = c["H"], c["W"]
    r = math.ceil(0.5 / c["kwargs"]["level"] * (H ** 2 + W ** 2) ** 0.5)
    torch.manual_seed(c["draw_seed"])
    di = torch.randint(-r, r + 1, (H, W, 64))
    dj = torch.randint(-r, r + 1, (H, W, 64))
    return {"delta_i": di, "delta_j": dj, "selection": c["selection"]}


def test_golden_covers_the_cases():
    assert os.path.getsize(GOLDEN) < 512 << 10
    levels = {(c["kwargs"]["level"], c["H"], c["W"]) for c in CASES}
    assert {(4, 48, 64), (16, 48, 64), (4, 61, 83), (16, 61, 83), (64, 144, 224), (64, 48, 64)} <= levels
    for c in CASES:
        assert (c["kwargs"]["num_patches"], c["kwargs"]["align_resolution"]) == {4: (16, 24), 16: (256, 12), 64: (4096, 6)}[c["kwargs"]["level"]]
    assert {c["batch_shape"] for c in CASES} == {(), (2,)}
    assert any(c["global_scale"] is None for c in CASES) and any(c["kwargs"].get("beta", 0) > 0 for c in CASES)
    assert any(c["kwargs"].get("sparsity_aware") for c in CASES) and any(c["kwargs"].get("trunc", 1.0) < 1.0 for c in CASES)
    assert any(c["empty_image"] for c in CASES) and any(c["kept"].numel() == 0 for c in CASES)
    assert all(c["reference"] for c in CASES if c["batch_shape"] == ())
    # a global scale that rejects some patches: the recorded scale of some kept patch is outside (0.1, 10) times it
    rejecting = [c for c in CASES if c["global_scale"] is not None and c["scale"] is not None
                 and not bool(((c["scale"] / c["global_scale"].reshape(-1)[0] > 0.1) & (c["scale"] / c["global_scale"].reshape(-1)[0] < 10)).all())]
    assert rejecting


@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_golden_inputs_and_draws_are_reproduced(c):
    pred, gt, focal = case_inputs(c)
    assert array_digest(pred.numpy(), gt.numpy(), focal.numpy()) == c["inputs_sha256"]
    d = case_draws(c)
    assert array_digest(d["delta_i"].numpy(), d["delta_j"].numpy()) == c["draws_sha256"]


@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_port_reproduces_the_golden(c):
    """Bitwise on the CPU, from the recorded draws.  The reference's alignment solver is not importable here, so the port takes
    the scale and shift the golden recorded: the loss, misc, selection and kept patches are checked, and the gradient (which
    also flows through the solver's gathers) is checked on the GPU."""
    pred, gt, focal = case_inputs(c)
    record = {}
    loss, misc = port.affine_invariant_local_loss(pred, gt, focal, c["global_scale"], align=lambda *_: (c["scale"], c["shift"]),
                                                  draws=case_draws(c), record=record, **c["kwargs"])
    assert torch.equal(loss.detach(), c["loss"]) and misc == c["misc"]
    assert torch.equal(record["selection"], c["selection"]) and torch.equal(record["kept"], c["kept"])


def test_port_draws_as_the_reference():
    """Without explicit draws, the port makes the reference's calls: from the same seed it draws the recorded offsets and
    selection."""
    c = CASES[0]
    pred, gt, focal = case_inputs(c)
    record = {}
    torch.manual_seed(c["draw_seed"])
    port.affine_invariant_local_loss(pred, gt, focal, c["global_scale"], align=lambda *_: (c["scale"], c["shift"]),
                                     record=record, **c["kwargs"])
    assert array_digest(record["delta_i"].numpy(), record["delta_j"].numpy()) == c["draws_sha256"]
    assert torch.equal(record["selection"], c["selection"])


def test_exports():
    assert set(L.__all__) == {"compute_anchor_sampling_weight", "affine_invariant_local_loss"}
    assert all(callable(getattr(L, name)) for name in L.__all__)


@pytest.mark.parametrize("fn", ["compute_anchor_sampling_weight", "affine_invariant_local_loss"])
def test_cpu_inputs_are_rejected(fn):
    inputs = synthetic_loss_case(0, (), 8, 8)
    pred, gt = inputs["pred_points"], inputs["gt_points"]
    with pytest.raises(MogeError, match="CUDA tensors only"):
        if fn == "compute_anchor_sampling_weight":
            L.compute_anchor_sampling_weight(gt, torch.isfinite(gt).all(-1), 2, torch.ones(8, 8))
        else:
            L.affine_invariant_local_loss(pred, gt, torch.tensor(0.5), None, 4)
