"""-m gpu: the geometry utilities (moge_b200.geometry, alias moge.utils.geometry_torch) against tests/golden/geometry.pt and the
fp64 restatements of oracle/geometry_port.py.

Bitwise against the golden: dilate_with_mask with min, max and median, theshold_depth_change, and recover_focal_shift's
degenerate images.  Within the per-element bounds that oracle/geometry_port.py derives (first-order forward error bounds of an
fp32 evaluation, times 2): dilate_with_mask with mean, gaussian_blur_2d and refine_depth_with_normal, whose bound also covers
the reference's own outputs (tests/test_geometry_torch_host.py)."""
import os

import pytest
import torch

import moge.utils.geometry_torch as G
from moge_b200.capi import MogeError
from moge_b200.synthetic import synthetic_geometry_case, synthetic_point_map
from oracle import geometry_port as gp

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "geometry.pt"), weights_only=False)


def inputs(c, mask_mode="sparse"):
    bs = c["batch_shape"] if "batch_shape" in c else (c["B"],)
    return synthetic_geometry_case(c["seed"], bs, c["H"], c["W"], c.get("mask_mode", mask_mode))


def same_bits(a, b):
    """bitwise equality of two fp32 tensors, NaN included"""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32).cpu(), b.contiguous().view(torch.int32).cpu())


def same_values(a, b):
    """equal values, NaN where the other is NaN"""
    return a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def refine(x, **kw):
    d = x["depth"].to(DEV)
    out = G.refine_depth_with_normal(d, x["normal"].to(DEV), x["intrinsics"].to(DEV), **kw)
    torch.cuda.synchronize()
    return out.cpu()


def check_refine_bound(x, out, iterations=10, kernel_size=5):
    H, W = x["depth"].shape[-2:]
    ref, bound = gp.refine_depth_with_normal(x["depth"].reshape(-1, H, W), x["normal"].reshape(-1, H, W, 3),
                                             x["intrinsics"].reshape(-1, 3, 3), iterations, kernel_size=kernel_size)
    err = (out.reshape(-1, H, W).double() - ref).abs()
    ratio = float((err / bound).max())
    print(f"refine {tuple(x['depth'].shape)} k={kernel_size} it={iterations}: max err / bound {ratio:.3f}, "
          f"max bound / depth {float((bound / ref).max()):.2e}")
    assert ratio <= 1.0


def test_refine_within_bound_on_golden_cases(gold):
    for c in gold["refine"]:
        x = inputs(c)
        out = refine(x, iterations=c["iterations"], kernel_size=c["kernel_size"])
        assert out.shape == c["depth"].shape and out.dtype == torch.float32
        check_refine_bound(x, out, c["iterations"], c["kernel_size"])


@pytest.mark.parametrize("shape", [((2,), 256, 320), ((), 517, 389)])
def test_refine_within_bound_at_larger_sizes(shape):
    bs, H, W = shape
    x = synthetic_geometry_case(60 + H, bs, H, W)
    check_refine_bound(x, refine(x))


def test_refine_clamps_depth_in_place_and_is_reproducible():
    x = synthetic_geometry_case(70, (2,), 64, 48)
    depth = x["depth"].clone()
    depth[0, 10, 10:20] = 0.0
    depth[1, 30, 5] = -1.0
    depth[1, 31, 5] = float("nan")
    d = depth.to(DEV)
    n, K = x["normal"].to(DEV), x["intrinsics"].to(DEV)
    a = G.refine_depth_with_normal(d, n, K)
    assert same_values(d.cpu(), depth.clamp_min(1e-12)), "depth.clamp_min_(eps) in place"
    assert d.cpu()[0, 10, 10].item() == torch.tensor(1e-12).item() and torch.isnan(d.cpu()[1, 31, 5])
    assert same_bits(a, G.refine_depth_with_normal(d, n, K))
    # a non-contiguous depth is clamped in place too
    dt = depth.transpose(1, 2).contiguous().to(DEV).transpose(1, 2)
    assert same_bits(G.refine_depth_with_normal(dt, n, K), a)
    assert same_values(dt.cpu(), depth.clamp_min(1e-12))
    # intrinsics broadcast over the batch
    one = G.refine_depth_with_normal(x["depth"].to(DEV), n, K[0])
    both = G.refine_depth_with_normal(x["depth"].to(DEV), n, K[0].expand(2, 3, 3))
    assert torch.equal(one, both)


def test_dilate_bitwise_and_mean_within_bound(gold):
    for c in gold["dilate"]:
        x = inputs(c)
        v, m = G.dilate_with_mask(x["depth"].to(DEV), x["mask"].to(DEV), c["filter"], c["iterations"])
        v, m = v.cpu(), m.cpu()
        assert m.dtype == torch.bool and torch.equal(m, c["mask"]), (c["filter"], c["mask_mode"])
        if c["filter"] != "mean":
            assert same_values(v, c["input"]), (c["filter"], c["iterations"], c["mask_mode"])
            continue
        H, W = c["H"], c["W"]
        ref, _, bound = gp.dilate_mean(x["depth"].reshape(-1, H, W), x["mask"].reshape(-1, H, W), c["iterations"])
        v = v.reshape(-1, H, W).double()
        assert torch.equal(torch.isnan(v), torch.isnan(ref))
        fin = ~torch.isnan(ref)
        assert ((v - ref).abs()[fin] <= bound[fin]).all()
        assert torch.equal(torch.isnan(c["input"].reshape(-1, H, W)), torch.isnan(ref))


def test_dilate_iterations_zero_and_repeatable():
    x = synthetic_geometry_case(71, (3,), 40, 56)
    d, m = x["depth"].to(DEV), x["mask"].to(DEV)
    assert G.dilate_with_mask(d, m, "mean", 0) == (d, m)
    for f in ("mean", "median"):
        a = G.dilate_with_mask(d, m, f, 4)
        b = G.dilate_with_mask(d, m, f, 4)
        assert same_bits(a[0], b[0]) and torch.equal(a[1], b[1])


def test_median_of_even_count_is_lower_middle():
    d = torch.tensor([[0.0, 4.0, 0.0], [1.0, 9.0, 3.0], [0.0, 2.0, 0.0]], device=DEV)
    m = torch.tensor([[False, True, False], [True, False, True], [False, True, False]], device=DEV)
    v, _ = G.dilate_with_mask(d, m, "median")
    assert v[1, 1].item() == 2.0                                   # sorted 1, 2, 3, 4
    m[2, 1] = False
    v, _ = G.dilate_with_mask(d, m, "median")
    assert v[1, 1].item() == 3.0                                   # sorted 1, 3, 4
    v, _ = G.dilate_with_mask(d, m, "mean")
    assert v[1, 1].item() == pytest.approx(8.0 / 3.0, rel=1e-7)


def test_threshold_bitwise(gold):
    for c in gold["threshold"]:
        x = inputs(c)
        out = G.theshold_depth_change(x["depth"].to(DEV), x["mask"].to(DEV), c["pooler"], rtol=c["rtol"], kernel_size=c["kernel_size"])
        assert out.dtype == torch.bool and torch.equal(out.cpu(), c["output"]), (c["pooler"], c["kernel_size"])


def test_blur_within_bound_and_reproducible(gold):
    for c in gold["blur"]:
        x = inputs(c)
        img = x["image"][:, :1].contiguous().to(DEV)
        out = G.gaussian_blur_2d(img, c["kernel_size"], c["sigma"])
        ref, bound = gp.gaussian_blur_2d(x["image"][:, :1], c["kernel_size"], c["sigma"])
        assert out.shape == c["output"].shape
        assert ((out.cpu().double() - ref).abs() <= bound).all()
        assert same_bits(out, G.gaussian_blur_2d(img, c["kernel_size"], c["sigma"]))
    # every channel is blurred alike
    img = synthetic_geometry_case(72, (2,), 30, 41)["image"].to(DEV)
    many = G.gaussian_blur_2d(img, 7, 1.5)
    for ch in range(3):
        assert torch.equal(many[:, ch:ch + 1], G.gaussian_blur_2d(img[:, ch:ch + 1].contiguous(), 7, 1.5))


def test_recover_focal_shift_golden(gold):
    for c in gold["focal_shift"]:
        pts, mask = synthetic_point_map(*c["args"][:7], seed=c["args"][7])
        bs = c["batch_shape"]
        pts, mask = pts.reshape(*bs, *pts.shape[1:]).to(DEV), mask.reshape(*bs, *mask.shape[1:]).to(DEV)
        focal_in = None if c["focal_in"] is None else c["focal_in"].to(DEV)
        f, s = G.recover_focal_shift(pts, mask, focal=focal_in)
        assert f.shape == bs and s.shape == bs and f.dtype == torch.float32 and s.dtype == torch.float32
        f, s = f.cpu(), s.cpu()
        if c["args"][6] in ("single", "none"):
            assert torch.equal(f, c["focal"]) and torch.equal(s, c["shift"])          # focal 1 (or the given one), shift 0
        else:
            if focal_in is not None:
                assert torch.equal(f, c["focal"])
            torch.testing.assert_close(f, c["focal"], rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(s, c["shift"], rtol=1e-5, atol=1e-6)
    # the points' dtype, without a mask
    pts, _ = synthetic_point_map(1, 64, 80, 1.2, 0.3, 0.0, "all", seed=9)
    f64, s64 = G.recover_focal_shift(pts.double().to(DEV))
    f32, s32 = G.recover_focal_shift(pts.to(DEV))
    assert f64.dtype == torch.float64 and f64.shape == (1,) and torch.equal(f64.float(), f32) and torch.equal(s64.float(), s32)


def test_closed_forms_on_gpu_match_golden(gold):
    x = {k: v.to(DEV) for k, v in gp.closed_inputs(gold["closed"]["seed"]).items()}
    out = gp.closed_calls(G, x)
    for k, ref in gold["closed"]["outputs"].items():
        got = out[k] if isinstance(ref, tuple) else (out[k],)
        for a, b in zip(got, ref if isinstance(ref, tuple) else (ref,)):
            assert a.is_cuda or k.startswith("normalized_view_plane_uv"), k       # that one takes no tensor: device=None
            # the legacy solve forms fp32 normal equations over 2 H W = 1728 rows, summed in a device-dependent order: the
            # reference's own fp32 result is up to 8e-5 (relative) from the fp64 solve of the same inputs
            rtol = 5e-4 if k == "point_map_to_depth_legacy" else 2e-6
            torch.testing.assert_close(a.cpu(), b, rtol=rtol, atol=1e-7, msg=k)


def test_cpu_inputs_and_bad_arguments_raise():
    x = synthetic_geometry_case(73, (), 20, 24)
    d, n, K, m = (x[k].to(DEV) for k in ("depth", "normal", "intrinsics", "mask"))
    with pytest.raises(MogeError, match="CUDA tensors only"):
        G.refine_depth_with_normal(d, n, K.cpu())
    with pytest.raises(MogeError, match="CUDA tensors only"):
        G.dilate_with_mask(d, m.cpu())
    with pytest.raises(MogeError, match="CUDA tensors only"):
        G.theshold_depth_change(d.cpu(), m, "max")
    with pytest.raises(MogeError, match="CUDA tensors only"):
        G.recover_focal_shift(torch.rand(20, 24, 3, device=DEV), m.cpu())
    with pytest.raises(ValueError, match="odd integer from 3 to 9"):
        G.refine_depth_with_normal(d, n, K, kernel_size=6)
    with pytest.raises(ValueError, match="odd integer from 3 to 9"):
        G.refine_depth_with_normal(d, n, K, kernel_size=11)
    with pytest.raises(ValueError, match="odd integer from 1 to 31"):
        G.gaussian_blur_2d(d[None, None], 2, 1.0)
    with pytest.raises(ValueError, match="filter must be one of"):
        G.dilate_with_mask(d, m, "mode")
    with pytest.raises(ValueError, match="64 x 64 grid only"):
        G.recover_focal_shift(torch.rand(20, 24, 3, device=DEV), downsample_size=(32, 48))
    with pytest.raises(MogeError, match="float32"):
        G.dilate_with_mask(d.double(), m)
