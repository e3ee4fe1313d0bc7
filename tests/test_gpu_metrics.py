"""moge_b200.metrics (the reference's moge/test/metrics.py on sm_90a kernels), on the GPU: golden parity with the unmodified
reference (tests/golden/metrics.pt, oracle/make_metrics_golden.py), the resize against the utils3d stand-in, boundary counts
against the plain-torch port, padded against unpadded alignments, batch against single-image calls, determinism, the
single host transfer, vis outputs and an end-to-end check on an infer() output."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from moge_b200 import alignment as A  # noqa: E402
from moge_b200 import metrics as M  # noqa: E402
from moge_b200.synthetic import METRICS_KEYS, synthetic_metrics_case  # noqa: E402
from oracle import metrics_port  # noqa: E402
from oracle.utils3d_metrics import install  # noqa: E402

u3d = install()

GOLDEN = os.path.join(ROOT, "tests", "golden", "metrics.pt")
CASES = torch.load(GOLDEN, weights_only=False)
gpu = pytest.mark.gpu


def cuda(d):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def inputs(c):
    p, g = synthetic_metrics_case(c["seed"], c["H"], c["W"], METRICS_KEYS[c["keys"]], c["is_metric"], c["sharp"], c["segments"],
                                  c["negative"])
    return cuda(p), cuda(g)


def flat(m, prefix=""):
    out = {}
    for k, v in m.items():
        if isinstance(v, dict):
            out.update(flat(v, prefix + k + "."))
        else:
            out[prefix + k] = v
    return out


def assert_metrics_close(got, want, lstsq_downstream=()):
    fg, fw = flat(got), flat(want)
    assert fg.keys() == fw.keys(), (sorted(fg), sorted(fw))
    for k, w in fw.items():
        g = fg[k]
        if math.isnan(w):
            assert math.isnan(g), k
            continue
        if any(k.startswith(p) for p in lstsq_downstream):
            assert abs(g - w) <= 1e-4 * max(1.0, abs(w)), (k, g, w)
        elif k.endswith(".rel"):
            assert abs(g - w) <= 1e-5 * abs(w), (k, g, w)
        else:
            assert abs(g - w) <= 1e-6, (k, g, w)


def lstsq_keys(c):
    """metrics downstream of the disparity least squares: the disparity variant, and the boundary when it is the aligned map"""
    keys = ["disparity_affine_invariant."]
    if c["keys"] == "disparity":
        keys.append("boundary.")
    return keys


# Metrics where the reference's own fp32 arithmetic, not the engine, decides the golden value (DESIGN.md §1, "Evaluation
# metrics"): key prefix -> the bound against the golden (None: not comparable).  These keys are checked at the normal limits
# against the plain-torch port run on CUDA with the engine's solvers instead.
#   - moge1_1024x768: the reference's fp32 LAPACK lstsq over 786k rows returns a disparity fit ~10x worse than the fp64
#     normal equations (rel 0.278 against 0.027);
#   - depth_affine_vis_640x480: the reference picks its depth-affine anchor by an fp32 objective, the engine by fp64; the two
#     near-equal optima move a few boundary label pairs at radius 3.
DIVERGENT = {"moge1_1024x768": {"disparity_affine_invariant.": None}, "depth_affine_vis_640x480": {"boundary.": 1e-5}}
# the vis maps built from that depth-affine alignment: checked against the port at the normal limits, against the golden at
# this relative bound
DIVERGENT_MAPS = {"depth_affine_vis_640x480": 1e-3}


def split(m, prefixes):
    fm = flat(m)
    inside = {k: v for k, v in fm.items() if any(k.startswith(p) for p in prefixes)}
    return {k: v for k, v in fm.items() if k not in inside}, inside


@gpu
@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_golden_parity(c):
    pred, gt = inputs(c)
    metrics, misc = M.compute_metrics(pred, gt, vis=c["vis"])
    div = DIVERGENT.get(c["name"], {})
    got, got_div = split(metrics, div)
    want, want_div = split(c["metrics"], div)
    assert_metrics_close(got, want, lstsq_keys(c))
    if div:
        port, _ = metrics_port.compute_metrics(pred, gt, vis=False, alignment=A)
        assert_metrics_close(got_div, split(port, div)[1], lstsq_keys(c))
        for k, w in want_div.items():
            bound = next(b for p, b in div.items() if k.startswith(p))
            if bound is not None:
                assert abs(got_div[k] - w) <= bound, (k, got_div[k], w)
    assert misc.keys() == c["misc"].keys()
    s = c["misc_stride"]
    port_misc = metrics_port.compute_metrics(pred, gt, vis=True, alignment=A)[1] if c["name"] in DIVERGENT_MAPS else None
    for k, want in c["misc"].items():
        got = misc[k][::s, ::s].cpu()
        assert got.shape == want.shape, k
        if port_misc is None:
            torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6, equal_nan=True, msg=k)
        else:
            torch.testing.assert_close(got, port_misc[k][::s, ::s].cpu(), rtol=1e-5, atol=1e-6, equal_nan=True, msg=k)
            torch.testing.assert_close(got, want, rtol=DIVERGENT_MAPS[c["name"]], atol=1e-6, equal_nan=True, msg=k)


@gpu
@pytest.mark.parametrize("H,W,th,tw", [(480, 640, 64, 64), (436, 872, 64, 64), (1365, 2048, 64, 64), (50, 70, 64, 64), (64, 64, 64, 64),
                                       (97, 33, 16, 40)])
def test_resize_matches_the_shim(H, W, th, tw):
    g = torch.Generator().manual_seed(H * W)
    mask = torch.rand(2, H, W, generator=g) > 0.6
    mask[1, : H // 2] = False
    mask = mask.cuda()
    want_mask, (_, wi, wj) = u3d.masked_nearest_resize(mask=mask, size=(th, tw), return_index=True)
    got_mask, (_, gi, gj) = M.masked_nearest_resize(mask=mask, size=(th, tw), return_index=True)
    assert torch.equal(got_mask, want_mask)
    assert torch.equal(gi.expand_as(wi), wi) and torch.equal(gj.expand_as(wj), wj)


@gpu
def test_resize_compaction_order_and_padding():
    _, gt = inputs(CASES[0])
    mask = gt["depth_mask"][None].to(torch.uint8)
    lr_mask, lr_index, lst, lst_w, count = M._resize(mask, 64, 64)
    n = int(count.item())
    want = lr_index[lr_mask].reshape(-1)
    assert n == want.numel() and torch.equal(lst[0, :n], want)
    assert torch.all(lst[0, n:] == want[0]) and torch.all(lst_w[0, :n] == 1) and torch.all(lst_w[0, n:] == 0)


@gpu
@pytest.mark.parametrize("negative", [False, True])
def test_boundary_counts_match_the_port(negative):
    pred, gt = inputs({"seed": 3, "H": 300, "W": 410, "keys": "depth_affine", "is_metric": False, "sharp": True, "segments": 0,
                       "negative": negative})
    p = pred["depth_affine_invariant"]
    counts = torch.zeros(1, 90, dtype=torch.int64, device="cuda")
    var = M.capi.MetricVariant(M.capi.MV_DEPTH, p.data_ptr(), None)
    M._boundary(gt["depth"][None].contiguous(), gt["depth_mask"][None].to(torch.uint8).contiguous(), var, counts, 90)
    for r in (1, 2, 3):
        want = metrics_port.boundary_counts(p, gt["depth"], gt["depth_mask"], r).reshape(-1)
        assert torch.equal(counts[0, (r - 1) * 30:r * 30].cpu(), want), r
        assert M.boundary_f1(p, gt["depth"], gt["depth_mask"], r) == metrics_port.boundary_f1(p, gt["depth"], gt["depth_mask"], r)


@gpu
def test_padded_and_unpadded_alignments_are_bitwise_equal():
    pred, gt = inputs(CASES[0])
    mask = gt["depth_mask"][None].to(torch.uint8)
    _, _, lst, lst_w, count = M._resize(mask, 64, 64)
    n = int(count.item())
    assert 100 < n < 4096
    d, gd = pred["depth_metric"].reshape(1, -1).gather(1, lst), gt["depth"].reshape(1, -1).gather(1, lst)
    pts = pred["points_metric"].reshape(1, -1, 3)[:, lst[0]]
    gpts = gt["points"].reshape(1, -1, 3)[:, lst[0]]
    w = torch.where(lst_w > 0, 1 / gd, 0.0)
    wp = torch.where(lst_w > 0, 1 / gpts.norm(dim=-1), 0.0)
    for fn, args_pad, args in [
        (A.align_depth_scale, (d, gd, w), (d[:, :n], gd[:, :n], w[:, :n])),
        (A.align_depth_affine, (d, gd, w), (d[:, :n], gd[:, :n], w[:, :n])),
        (A.align_points_scale, (pts, gpts, wp), (pts[:, :n], gpts[:, :n], wp[:, :n])),
        (A.align_points_xyz_shift, (pts, gpts, wp), (pts[:, :n], gpts[:, :n], wp[:, :n])),
        (A.align_points_scale_xyz_shift, (pts, gpts, wp), (pts[:, :n], gpts[:, :n], wp[:, :n])),
    ]:
        a, b = fn(*args_pad), fn(*args)
        a, b = (a if isinstance(a, tuple) else (a,)), (b if isinstance(b, tuple) else (b,))
        for x, y in zip(a, b):
            assert torch.equal(x, y), fn.__name__
    # a segment: its members at weight 1/diameter inside the full padded list, against the members alone
    seg = gt["segmentation_mask"].reshape(1, -1).gather(1, lst)
    ids, counts = torch.unique(seg[lst_w > 0], return_counts=True)
    member = (seg == ids[counts.argmax()]) & (lst_w > 0)
    m = member[0].nonzero().squeeze(-1)
    wseg = torch.where(member, torch.tensor(0.37, device="cuda"), 0.0)
    a = A.align_points_scale_xyz_shift(pts, gpts, wseg)
    b = A.align_points_scale_xyz_shift(pts[:, m], gpts[:, m], wseg[:, m])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _stack(cases):
    ps, gs = zip(*(inputs(c) for c in cases))
    pred = {k: torch.stack([p[k] for p in ps]) for k in ps[0]}
    gt = {k: (torch.stack([g[k] for g in gs]) if isinstance(gs[0][k], torch.Tensor) else gs[0][k]) for k in gs[0]
          if k != "segmentation_labels"}
    if "segmentation_labels" in gs[0]:
        gt["segmentation_labels"] = [g["segmentation_labels"] for g in gs]
    return ps, gs, pred, gt


def same(a, b):
    fa, fb = flat(a), flat(b)
    return fa.keys() == fb.keys() and all(fa[k] == fb[k] or (math.isnan(fa[k]) and math.isnan(fb[k])) for k in fa)


@gpu
@pytest.mark.parametrize("keys,segments", [("moge2", 30), ("moge1", 5), ("disparity", 0)])
def test_batch_is_bitwise_equal_to_single_calls(keys, segments):
    cases = [{"seed": 100 + i, "H": 240, "W": 320, "keys": keys, "is_metric": True, "sharp": True, "segments": segments - 4 * i if segments else 0,
              "negative": i == 1} for i in range(4)]
    ps, gs, pred, gt = _stack(cases)
    batch = M.compute_metrics_batch(pred, gt, vis=True)
    assert len(batch) == 4
    for b in range(4):
        m, misc = M.compute_metrics(ps[b], gs[b], vis=True)
        assert same(batch[b][0], m), b
        assert batch[b][1].keys() == misc.keys()
        for k in misc:
            assert torch.equal(batch[b][1][k], misc[k]), (b, k)


@gpu
def test_deterministic_across_runs():
    pred, gt = inputs(CASES[0])
    first = M.compute_metrics(pred, gt)[0]
    for _ in range(3):
        assert same(M.compute_metrics(pred, gt)[0], first)


@gpu
def test_one_host_transfer_and_no_sync_before_it():
    pred, gt = inputs(CASES[0])
    M.compute_metrics(pred, gt)            # warm-up: library load, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        call = M._launch({k: v[None] for k, v in pred.items()},
                         {k: (v[None] if isinstance(v, torch.Tensor) else v) for k, v in gt.items() if k != "segmentation_labels"},
                         [gt["segmentation_labels"]], False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert same(M._finish(call)[0][0], M.compute_metrics(pred, gt)[0])


@gpu
def test_degenerate_image_gets_nan():
    pred, gt = inputs(CASES[3])
    gt["depth_mask"] = torch.zeros_like(gt["depth_mask"])
    m, _ = M.compute_metrics(pred, gt)
    for k in ("depth_scale_invariant", "depth_affine_invariant", "points_affine_invariant"):
        assert math.isnan(m[k]["rel"]) and math.isnan(m[k]["delta1"])


@gpu
def test_vis_depth_only_gives_a_point_map():
    c = next(c for c in CASES if c["keys"] == "depth_affine")
    pred, gt = inputs(c)
    m, misc = M.compute_metrics(pred, gt, vis=True)
    assert set(misc) == {"pred_points", "pred_depth"} and misc["pred_points"].shape == (c["H"], c["W"], 3)
    torch.testing.assert_close(misc["pred_points"][..., 2], misc["pred_depth"])


@gpu
def test_end_to_end_infer_output_against_the_port():
    from moge.model.v2 import MoGeModel
    from moge_b200.configs import model_config
    from moge_b200.synthetic import make_state_dict, synthetic_images
    cfg = model_config("vits", True)
    model = MoGeModel(**cfg)
    model.load_state_dict(make_state_dict(cfg, 0, well_posed=True))
    model = model.cuda().eval()
    img = synthetic_images(1, 196, 252, 0)[0].cuda()
    out = model.infer(img, num_tokens=300, apply_mask=False)
    _, gt = synthetic_metrics_case(7, 196, 252, (), True, True, 6)
    gt = cuda(gt)
    gt["depth"] = out["depth"].float() * 1.1 + 0.05 * torch.randn_like(out["depth"].float())
    gt["depth"] = gt["depth"].abs() + 0.1
    gt["points"] = u3d.depth_map_to_point_map(gt["depth"], gt["intrinsics"])
    pred = {"points_metric": out["points"].float(), "depth_metric": out["depth"].float(), "intrinsics": out["intrinsics"].float()}
    got, _ = M.compute_metrics(pred, gt)
    want, _ = metrics_port.compute_metrics(pred, gt, alignment=A)
    assert_metrics_close(got, want, ["disparity_affine_invariant."])
