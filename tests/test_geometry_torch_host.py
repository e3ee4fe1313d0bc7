"""Host checks of the geometry utilities (moge_b200.geometry, alias moge.utils.geometry_torch): the oracle's fp64 restatements
against the reference's outputs in tests/golden/geometry.pt within their stated bounds, the golden's inputs, the closed forms
on the CPU, the alias's names and signatures against the reference module's, and the argument checks that run before any
device work."""
import inspect
import os

import pytest
import torch

import moge.utils.geometry_torch as alias
from moge_b200 import capi
from moge_b200.capi import MogeError
from moge_b200.synthetic import array_digest, synthetic_geometry_case, synthetic_point_map
from oracle import geometry_port as gp


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "geometry.pt"), weights_only=False)


def inputs(c, mask_mode="sparse"):
    bs = c["batch_shape"] if "batch_shape" in c else (c["B"],)
    x = synthetic_geometry_case(c["seed"], bs, c["H"], c["W"], c.get("mask_mode", mask_mode))
    assert array_digest(*[x[k].numpy() for k in ("depth", "normal", "intrinsics", "mask", "image")]) == c["inputs_sha256"]
    return x


def test_refine_restatement_within_bound_of_reference(gold):
    for c in gold["refine"]:
        x, H, W = inputs(c), c["H"], c["W"]
        out, bound = gp.refine_depth_with_normal(x["depth"].reshape(-1, H, W), x["normal"].reshape(-1, H, W, 3),
                                                 x["intrinsics"].reshape(-1, 3, 3), c["iterations"], kernel_size=c["kernel_size"],
                                                 fp32_grad=True)
        err = (c["depth"].reshape(-1, H, W).double() - out).abs()
        assert (err <= bound).all(), (c["H"], c["W"], float((err / bound).max()))


def test_dilate_restatements_match_reference(gold):
    for c in gold["dilate"]:
        x, H, W = inputs(c), c["H"], c["W"]
        d, m = x["depth"].reshape(-1, H, W), x["mask"].reshape(-1, H, W)
        if c["filter"] == "mean":
            v, mo, bound = gp.dilate_mean(d, m, c["iterations"])
            ref = c["input"].reshape(-1, H, W).double()
            assert torch.equal(torch.isnan(ref), torch.isnan(v))
            fin = ~torch.isnan(ref)
            assert ((ref - v).abs()[fin] <= bound[fin]).all()
        elif c["filter"] in ("min", "max"):
            assert c["source"] == "geometry_port.dilate_min_max"
            v, mo = gp.dilate_min_max(d, m, c["filter"], c["iterations"])
            assert torch.equal(v, c["input"].reshape(-1, H, W))
        else:
            continue
        assert torch.equal(mo, c["mask"].reshape(-1, H, W))


def test_blur_restatement_within_bound_of_reference(gold):
    for c in gold["blur"]:
        x = inputs(c)
        out, bound = gp.gaussian_blur_2d(x["image"][:, :1], c["kernel_size"], c["sigma"])
        assert ((c["output"].double() - out).abs() <= bound).all()


def test_focal_shift_golden_inputs_and_degenerate_cases(gold):
    for c in gold["focal_shift"]:
        pts, mask = synthetic_point_map(*c["args"][:7], seed=c["args"][7])
        assert array_digest(pts.reshape(*c["batch_shape"], *pts.shape[1:]).numpy(),
                            mask.reshape(*c["batch_shape"], *mask.shape[1:]).numpy()) == c["inputs_sha256"]
        assert c["focal"].shape == c["batch_shape"] and c["shift"].shape == c["batch_shape"]
        if c["args"][6] in ("single", "none"):          # fewer than two valid points: focal 1 (or the given one), shift 0
            assert torch.equal(c["shift"], torch.zeros(c["batch_shape"]))
            assert torch.equal(c["focal"], torch.ones(c["batch_shape"]) if c["focal_in"] is None else c["focal_in"])


def test_closed_forms_on_cpu_match_golden(gold):
    x = gp.closed_inputs(gold["closed"]["seed"])
    assert array_digest(*[v.numpy() for v in x.values()]) == gold["closed"]["inputs_sha256"]
    out = gp.closed_calls(alias, x)
    for k, ref in gold["closed"]["outputs"].items():
        got = out[k] if isinstance(ref, tuple) else (out[k],)
        for a, b in zip(got, ref if isinstance(ref, tuple) else (ref,)):
            assert a.shape == b.shape and a.dtype == b.dtype, k
            torch.testing.assert_close(a, b, rtol=4e-7, atol=0, msg=k)
    # the reference's geometric_mean drops the reduced dims without w whatever keepdim says
    assert gold["closed"]["outputs"]["geometric_mean_keep"].shape == (5,)


def test_alias_names_and_signatures_match_reference(gold):
    sigs = gold["signatures"]
    assert sorted(alias.__all__) == sorted(sigs)
    assert gp.public_signatures(__import__("moge_b200.geometry", fromlist=["x"])) == sigs
    for name, params in sigs.items():
        got = [(p.name, None if p.default is inspect.Parameter.empty else repr(p.default))
               for p in inspect.signature(getattr(alias, name)).parameters.values()]
        assert got == params, name
    from oracle.utils3d_geometry import load_geometry
    ref = load_geometry()                      # the compiled reference, where the build had it
    if ref is not None:
        assert gp.public_signatures(ref) == sigs


def test_abi_table_lists_geometry_entries():
    for n in ("moge_geometry_workspace_bytes", "moge_refine_depth_with_normal", "moge_dilate_with_mask",
              "moge_threshold_depth_change", "moge_gaussian_blur_2d"):
        assert n in capi.SIGNATURES


def test_argument_checks_before_device_work():
    d = torch.rand(2, 16, 16) + 0.5
    n = torch.nn.functional.normalize(torch.randn(2, 16, 16, 3), dim=-1)
    K = torch.eye(3)
    m = torch.rand(2, 16, 16) > 0.5
    for k in (4, 1, 11):
        with pytest.raises(ValueError, match="kernel_size must be an odd integer from 3 to 9"):
            alias.refine_depth_with_normal(d, n, K, kernel_size=k)
    with pytest.raises(ValueError, match="kernel_size must be an odd integer from 1 to 15"):
        alias.theshold_depth_change(d, m, "max", kernel_size=17)
    with pytest.raises(ValueError, match="Unsupported pooler"):
        alias.theshold_depth_change(d, m, "mean")
    with pytest.raises(ValueError, match="kernel_size must be an odd integer from 1 to 31"):
        alias.gaussian_blur_2d(d[:, None], 4, 1.0)
    with pytest.raises(ValueError, match="filter must be one of mean, min, max, median"):
        alias.dilate_with_mask(d, m, "mode")
    with pytest.raises(ValueError, match="64 x 64 grid only"):
        alias.recover_focal_shift(torch.rand(16, 16, 3), downsample_size=(32, 32))
    # CPU tensors: no fallback
    for call in (lambda: alias.refine_depth_with_normal(d, n, K), lambda: alias.dilate_with_mask(d, m),
                 lambda: alias.theshold_depth_change(d, m, "min"), lambda: alias.gaussian_blur_2d(d[:, None], 3, 1.0),
                 lambda: alias.recover_focal_shift(torch.rand(16, 16, 3))):
        with pytest.raises(MogeError, match="CUDA tensors only"):
            call()
