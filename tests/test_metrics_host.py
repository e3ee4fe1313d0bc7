"""moge_b200.metrics on the CPU side: golden inputs, the plain-torch port, the utils3d stand-in, the F1 threshold table and
argument validation (every check fails before any launch, so none needs a GPU)."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from moge_b200 import metrics as M  # noqa: E402
from moge_b200.capi import MogeError  # noqa: E402
from moge_b200.synthetic import METRICS_KEYS, synthetic_metrics_case  # noqa: E402
from oracle.utils3d_metrics import install  # noqa: E402

u3d = install()

GOLDEN = os.path.join(ROOT, "tests", "golden", "metrics.pt")
CASES = torch.load(GOLDEN, weights_only=False)


def case_inputs(c):
    return synthetic_metrics_case(c["seed"], c["H"], c["W"], METRICS_KEYS[c["keys"]], c["is_metric"], c["sharp"], c["segments"],
                                  c["negative"])


def digest(pred, gt):
    h = hashlib.sha256()
    for d in (pred, gt):
        for k in sorted(d):
            if isinstance(d[k], torch.Tensor):
                h.update(k.encode())
                h.update(d[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def test_golden_covers_the_cases():
    names = {c["name"] for c in CASES}
    assert len(CASES) >= 8 and os.path.getsize(GOLDEN) < 1 << 20
    assert {c["keys"] for c in CASES} >= {"moge2", "moge1", "depth_affine", "disparity", "points_affine"}
    assert any(c["H"] < 64 for c in CASES) and any(c["vis"] for c in CASES) and any(c["segments"] for c in CASES), names


@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_golden_inputs_are_reproduced(c):
    assert digest(*case_inputs(c)) == c["inputs_sha256"]


@pytest.mark.parametrize("c", [c for c in CASES if c["H"] * c["W"] <= 640 * 480], ids=lambda c: c["name"])
def test_port_reproduces_the_golden(c):
    """The plain-torch port with the reference's solvers is not importable here; its metric logic is checked with exact solvers
    replaced by the values the golden run found: depth_metric, fov_x and the boundary of raw metric depth need no solver."""
    from oracle import metrics_port
    pred, gt = case_inputs(c)
    want = c["metrics"]
    if "depth_metric" in pred and c["is_metric"]:
        got = {"rel": metrics_port._rel_depth(pred["depth_metric"][gt["depth_mask"]], gt["depth"][gt["depth_mask"]]),
               "delta1": metrics_port._delta_depth(pred["depth_metric"][gt["depth_mask"]], gt["depth"][gt["depth_mask"]])}
        assert got == want["depth_metric"]
        if c["sharp"]:
            for r in (1, 2, 3):
                assert metrics_port.boundary_f1(pred["depth_metric"], gt["depth"], gt["depth_mask"], r) == want["boundary"][f"radius{r}_f1"]
    if "intrinsics" in pred:
        fov = lambda K: 2 * torch.atan(0.5 / K[..., 0, 0])  # noqa: E731
        diff = torch.rad2deg(fov(pred["intrinsics"]) - fov(gt["intrinsics"]))
        assert {"mae": diff.abs().mean().item(), "deviation": diff.item()} == want["fov_x"]


def test_shim_resize_is_identity_at_full_size():
    g = torch.Generator().manual_seed(0)
    for H, W in ((64, 64), (33, 47)):
        mask = torch.ones(H, W, dtype=torch.bool)
        x = torch.randn(H, W, 3, generator=g)
        y, lr_mask, (i, j) = u3d.masked_nearest_resize(x, mask=mask, size=(H, W), return_index=True)
        assert lr_mask.all() and torch.equal(y, x)
        assert torch.equal(i, torch.arange(H)[:, None].expand(H, W)) and torch.equal(j, torch.arange(W)[None].expand(H, W))


def test_shim_resize_takes_the_nearest_valid_pixel():
    mask = torch.zeros(128, 128, dtype=torch.bool)
    mask[5, 7] = True
    lr_mask, (i, j) = u3d.masked_nearest_resize(mask=mask, size=(64, 64), return_index=True)
    assert lr_mask.sum() == 1 and lr_mask[2, 3]
    assert (i[2, 3].item(), j[2, 3].item()) == (5, 7)


def test_shim_sliding_window():
    x = torch.arange(20.0).reshape(4, 5)
    w = u3d.sliding_window_2d(x, 3, 1, dim=(-2, -1))
    assert w.shape == (2, 3, 3, 3)
    assert torch.equal(w[1, 2], x[1:4, 2:5])


def test_threshold_table():
    t = torch.linspace(0.05, 0.25, 10)
    assert M.F1_WEIGHTS == t.tolist()
    assert M.F1_THRESHOLDS.dtype == np.float32
    assert [float(v) for v in M.F1_THRESHOLDS] == [float(np.float32(1 + float(x))) for x in t]
    ratios = torch.tensor([float(v) for v in M.F1_THRESHOLDS])
    for k, tt in enumerate(t.tolist()):      # ratio > 1 + t in fp32 equals ratio > table[k]
        assert torch.equal(ratios > 1 + tt, ratios > ratios[k])
    assert all(np.diff(M.F1_THRESHOLDS) > 0)


def _cpu_case():
    return synthetic_metrics_case(0, 40, 48, METRICS_KEYS["moge2"], segments=2)


def test_cpu_inputs_are_rejected():
    pred, gt = _cpu_case()
    with pytest.raises(MogeError, match="CUDA"):
        M.compute_metrics(pred, gt)
    with pytest.raises(MogeError, match="CUDA"):
        M.masked_nearest_resize(mask=gt["depth_mask"], size=(64, 64))
    with pytest.raises(MogeError, match="CUDA"):
        M.boundary_f1(pred["depth_metric"], gt["depth"], gt["depth_mask"], 1)


def test_bad_radius_is_rejected():
    pred, gt = _cpu_case()
    with pytest.raises(MogeError, match="radius"):
        M.boundary_f1(pred["depth_metric"], gt["depth"], gt["depth_mask"], 4)


def test_abi_rejects_bad_arguments_before_launch():
    from moge_b200 import capi
    import ctypes as C
    L = capi.lib()
    nbytes = C.c_size_t()
    assert L.moge_metrics_workspace_bytes(1, 480, 640, 257, C.byref(nbytes)) != 0
    assert b"segment" in L.moge_last_error()
    assert L.moge_metrics_workspace_bytes(0, 480, 640, 0, C.byref(nbytes)) != 0
    assert L.moge_metrics_workspace_bytes(1, 480, 640, 256, C.byref(nbytes)) == 0 and nbytes.value > 0
    assert L.moge_metrics_resize(None, 1, 8, 8, 4, 4, None, None, None, None, None, None) != 0
    vs = (capi.MetricVariant * 1)()
    assert L.moge_metrics_eval(8, 8, 8, vs, 9, None, None, None, None, 0, None, None, 1, 8, 8, 8, 40, None, 0, None) != 0
    assert b"variants" in L.moge_last_error()
    assert L.moge_metrics_stats(8, 8, 8, None, 0, 8, 8, 8, 300, 1, 8, 8, 8, 8, None, 0, None) != 0
    assert b"segment" in L.moge_last_error()
    thr = (C.c_float * 10)(*reversed([float(t) for t in M.F1_THRESHOLDS]))
    var = capi.MetricVariant(capi.MV_DEPTH, 8, None)
    assert L.moge_metrics_boundary(8, 8, C.byref(var), thr, 1, 8, 8, 8, 90, None) != 0
    assert b"sorted" in L.moge_last_error()


def test_too_many_segments_are_rejected_before_launch(monkeypatch):
    """The segment count is checked on the host labels, before anything touches the device."""
    pred, gt = _cpu_case()
    gt["segmentation_labels"] = {f"s{i}": i for i in range(300)}
    calls = []
    monkeypatch.setattr(M, "_resize", lambda *a: calls.append(a))
    monkeypatch.setattr(M, "_mask_u8", lambda m: m.to(torch.uint8))
    monkeypatch.setattr(M, "_f32", lambda t: t.float())
    with pytest.raises(MogeError, match="at most 256"):
        M._launch({k: v[None] for k, v in pred.items()},
                  {k: (v[None] if isinstance(v, torch.Tensor) else v) for k, v in gt.items() if k != "segmentation_labels"},
                  [gt["segmentation_labels"]], False)
    assert not calls


def test_bad_shapes_are_rejected(monkeypatch):
    pred, gt = _cpu_case()
    monkeypatch.setattr(M, "_mask_u8", lambda m: m.to(torch.uint8))
    monkeypatch.setattr(M, "_f32", lambda t: t.float())
    g = {k: (v[None] if isinstance(v, torch.Tensor) else v) for k, v in gt.items() if k != "segmentation_labels"}
    p = {k: v[None] for k, v in pred.items()}
    p["depth_metric"] = p["depth_metric"][:, :-1]
    with pytest.raises(MogeError, match="shape"):
        M._launch(p, g, [gt["segmentation_labels"]], False)
    with pytest.raises(MogeError, match="depth_mask"):
        M._launch({k: v[None] for k, v in pred.items()}, dict(g, depth_mask=gt["depth_mask"]), None, False)
