"""Colourisation kernels on the GPU (moge_b200.vis and the drop-in moge.utils.vis), bitwise against np.nanquantile and the numpy
restatement in oracle/vis_port.py."""
import warnings

import numpy as np
import pytest
import torch

from moge_b200 import vis
from oracle import vis_port

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(1, 1), (1, 57), (37, 53), (480, 640), (1365, 2048)]
CASES = ["random", "ties", "all_equal", "one_valid", "none_valid", "inf", "nonpositive", "nan"]


def case(kind, H, W, seed):
    """(depth fp32, mask bool) of one image."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.5, 20, (H, W)).astype(np.float32)
    m = rng.random((H, W)) < 0.8
    if kind == "ties":
        d = np.round(d).astype(np.float32)
    elif kind == "all_equal":
        d[:] = np.float32(3.25)
    elif kind == "one_valid":
        d[:] = np.nan
        d[H // 2, W // 2] = 2.5
        m[H // 2, W // 2] = True
    elif kind == "none_valid":
        d[:] = np.nan
    elif kind == "inf":
        d[rng.random((H, W)) < 0.3] = np.inf
    elif kind == "nonpositive":
        d[rng.random((H, W)) < 0.2] = 0.0
        d[rng.random((H, W)) < 0.2] = -rng.uniform(0.1, 5)
    elif kind == "nan":
        d[rng.random((H, W)) < 0.3] = np.nan
    return d, m


def nanq(x, q):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.float32(np.nanquantile(x, q))


def want_quantiles(d, m, qs, depth):
    with np.errstate(divide="ignore", invalid="ignore"):
        if depth:
            x = 1 / np.where((d > 0) & (m if m is not None else True), d, np.nan)
        else:
            x = d if m is None else np.where(m, d, np.nan)
    return np.array([nanq(x, q) for q in qs], dtype=np.float32)


def same(a, b):
    """Bitwise equal, except that a NaN equals any NaN (its sign and payload are the hardware's, not the algorithm's)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and a[~nan].tobytes() == b[~nan].tobytes()


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("kind", CASES)
def test_quantiles_bitwise(H, W, kind):
    d, m = case(kind, H, W, H * 31 + W + CASES.index(kind))
    qs = (0.001, 0.99, 0.5, 0.999)
    dd, dm = torch.from_numpy(d).to(DEV), torch.from_numpy(m).to(DEV)
    for depth in (True, False):
        for mask in (None, m):
            got = vis.quantiles(dd, qs, mask=None if mask is None else dm, depth=depth).cpu().numpy()
            want = want_quantiles(d, mask, qs, depth)
            assert same(got, want), (kind, depth, mask is None, got, want)


def test_batch_equals_single_images():
    B, H, W = 5, 120, 160
    ds, ms = zip(*[case(k, H, W, 70 + b) for b, k in enumerate(["random", "none_valid", "inf", "ties", "nonpositive"])])
    d, m = torch.from_numpy(np.stack(ds)).to(DEV), torch.from_numpy(np.stack(ms)).to(DEV)
    qb = vis.quantiles(d, (0.001, 0.99), mask=m, depth=True)
    for fn in (vis.colorize_depth, vis.colorize_disparity, vis.colorize_depth_affine):
        batch = fn(d, m)
        for b in range(B):
            assert torch.equal(batch[b], fn(d[b], m[b])), (fn.__name__, b)
    for b in range(B):
        assert same(qb[b].cpu().numpy(), vis.quantiles(d[b], (0.001, 0.99), mask=m[b], depth=True).cpu().numpy())
    n = torch.from_numpy(np.random.default_rng(3).standard_normal((B, H, W, 3)).astype(np.float32)).to(DEV)
    batch = vis.colorize_normal(n, m)
    for b in range(B):
        assert torch.equal(batch[b], vis.colorize_normal(n[b], m[b]))


ORACLE = {"colorize_depth": vis_port.colorize_depth, "colorize_depth_affine": vis_port.colorize_depth_affine,
          "colorize_disparity": vis_port.colorize_disparity}


def oracle(name, x, m, normalize=True):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if name == "colorize_depth_affine":
            return ORACLE[name](x, m)
        return ORACLE[name](x, m, normalize=normalize)


@pytest.mark.parametrize("H,W", [(1, 57), (37, 53), (480, 640), (1365, 2048)])
@pytest.mark.parametrize("name", sorted(ORACLE))
def test_colorizers_bitwise(H, W, name):
    import moge.utils.vis as dropin
    for k, kind in enumerate(["random", "inf", "nonpositive", "nan", "all_equal", "none_valid"]):
        d, m = case(kind, H, W, 500 + k)
        if name == "colorize_disparity":
            with np.errstate(divide="ignore"):
                d = (1 / d).astype(np.float32)
        for mask in (None, m):
            for normalize in ((True, False) if name != "colorize_depth_affine" else (True,)):
                want = oracle(name, d, mask, normalize)
                dd = torch.from_numpy(d).to(DEV)
                dm = None if mask is None else torch.from_numpy(mask).to(DEV)
                kw = {} if name == "colorize_depth_affine" else {"normalize": normalize}
                got = getattr(vis, name)(dd, dm, **kw)
                assert np.array_equal(got.cpu().numpy(), want), (name, kind, mask is None, normalize)
                bgr = getattr(vis, name)(dd, dm, bgr=True, **kw)
                assert np.array_equal(bgr.cpu().numpy(), want[..., ::-1])
                assert np.array_equal(getattr(dropin, name)(d, mask, **kw), want)
                assert dd.cpu().numpy().tobytes() == d.tobytes()            # input unmodified (NaN included)


@pytest.mark.parametrize("H,W", [(37, 53), (1365, 2048)])
def test_colorize_normal_bitwise(H, W):
    import moge.utils.vis as dropin
    rng = np.random.default_rng(H)
    n = rng.standard_normal((H, W, 3)).astype(np.float32)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n[rng.random((H, W)) < 0.05] *= 3                          # outside [-1, 1]: clipped
    n[rng.random((H, W)) < 0.02] = np.nan
    m = rng.random((H, W)) < 0.7
    dn = torch.from_numpy(n).to(DEV)
    for mask in (None, m):
        with np.errstate(invalid="ignore"):
            want = vis_port.colorize_normal(n, mask)
        got = vis.colorize_normal(dn, None if mask is None else torch.from_numpy(mask).to(DEV))
        assert np.array_equal(got.cpu().numpy(), want)
        assert np.array_equal(dropin.colorize_normal(n, mask), want)
    assert np.array_equal(dn.cpu().numpy(), n, equal_nan=True)


def test_no_host_synchronisation_and_repeatable():
    d, m = case("inf", 768, 1024, 9)
    dd, dm = torch.from_numpy(d).to(DEV), torch.from_numpy(m).to(DEV)
    n = torch.nn.functional.normalize(torch.randn(768, 1024, 3, device=DEV), dim=-1)
    first = [vis.colorize_depth(dd), vis.colorize_depth(dd, dm), vis.colorize_depth_affine(dd, dm), vis.colorize_disparity(dd),
             vis.colorize_normal(n, dm)]
    torch.cuda.synchronize()
    out = torch.empty(768, 1024, 3, dtype=torch.uint8, device=DEV)
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = [vis.colorize_depth(dd), vis.colorize_depth(dd, dm), vis.colorize_depth_affine(dd, dm), vis.colorize_disparity(dd),
                 vis.colorize_normal(n, dm)]
        vis.colorize_depth(dd, bgr=True, out=out)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(first, again):
        assert torch.equal(a, b)
    assert torch.equal(out, first[0].flip(-1))
    assert same(dd.cpu().numpy(), d) and torch.equal(dm.cpu(), torch.from_numpy(m))
