"""moge_b200.alignment (the reference's moge/utils/alignment.py on sm_90a kernels).

CPU: the golden inputs are reproducible, arguments are validated, and the size bound is rejected before any launch.
GPU: parity with the reference's outputs (tests/golden/alignment.pt, oracle/make_alignment_golden.py), a brute-force check that
does not rely on the reference, determinism, batch independence, gradients and the least-squares solve."""
import ctypes as C
import hashlib
import os

import pytest
import torch

from moge_b200 import capi
from moge_b200 import alignment as A
from moge_b200.synthetic import alignment_arguments, synthetic_alignment_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "alignment.pt")
CASES = torch.load(GOLDEN, weights_only=False)
gpu = pytest.mark.gpu


def _case_id(c):
    return f"{c['fn']}-{'x'.join(map(str, c['batch_shape'])) or 'scalar'}-n{c['n']}-{c['trunc']}{'-single' if c['single_positive'] else ''}"


def _args(c):
    return alignment_arguments(c["fn"], c["batch_shape"], c["n"], c["seed"], c["trunc"], c["single_positive"])


def _digest(args):
    h = hashlib.sha256()
    for a in args:
        if isinstance(a, torch.Tensor):
            h.update(a.contiguous().numpy().tobytes())
    return h.hexdigest()


def _cuda(args):
    return tuple(a.cuda() if isinstance(a, torch.Tensor) else a for a in args)


# ------------------------------------------------------------------------------------------------------------ fp64 objectives
def _trunc_terms(r, t):
    if t is None:
        return r
    return torch.minimum(r, t.double()) if isinstance(t, torch.Tensor) else r.clamp_max(t)


def objective(fn, args, out):
    """sum_i min(t, w_i |residual_i|) in fp64 at the solution `out` of `fn`, per problem (the batch shape; (..., 3) for
    align_points_xyz_shift)."""
    src, tgt, w, t = (a.double().cpu() if isinstance(a, torch.Tensor) else a for a in args)
    out = tuple(o.double().cpu() for o in (out if isinstance(out, tuple) else (out,)))
    if fn in ("align", "align_depth_scale"):
        r = w * (out[0][..., None] * src - tgt).abs()
    elif fn == "align_points_scale":
        r = w[..., None] * (out[0][..., None, None] * src - tgt).abs()
        r = r.flatten(-2)
        if isinstance(t, torch.Tensor):
            t = t[..., None].expand(*t.shape, 3).flatten(-2)
    elif fn == "align_points_z_shift":
        r = w * (out[0][..., None, 2] + src[..., 2] - tgt[..., 2]).abs()
    elif fn == "align_points_xyz_shift":
        r = w[..., None, :] * (out[0][..., :, None] + (src - tgt).swapaxes(-2, -1)).abs()
    elif fn == "align_depth_affine":
        r = w * (out[0][..., None] * src + out[1][..., None] - tgt).abs()
    else:        # align_points_scale_z_shift / _xyz_shift
        r = w[..., None] * (out[0][..., None, None] * src + out[1][..., None, :] - tgt).abs()
        r = r.flatten(-2)
    return _trunc_terms(r, t).sum(-1)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_golden_inputs_are_reproduced():
    assert len(CASES) >= 50
    for c in CASES:
        assert _digest(_args(c)) == c["inputs_sha256"], _case_id(c)


def test_every_function_is_exported_under_the_reference_path():
    import moge.utils.alignment as drop_in
    for name in A.__all__:
        assert getattr(drop_in, name) is getattr(A, name)
    assert {c["fn"] for c in CASES} == set(A.__all__)


def test_argument_validation():
    src, tgt, w = synthetic_alignment_case((2,), 16, 0)
    with pytest.raises(capi.MogeError, match="CUDA"):
        A.align_points_scale_xyz_shift(src, tgt, w)
    with pytest.raises(capi.MogeError, match="CUDA"):
        A.align(src[..., 2], tgt[..., 2], w, trunc=0.5)
    with pytest.raises(capi.MogeError, match="CUDA"):
        A.align_affine_lstsq(src[..., 2], tgt[..., 2])
    with pytest.raises(capi.MogeError, match="trunc"):
        A.align_depth_affine(src[..., 2], tgt[..., 2], w, trunc=-1.0)
    with pytest.raises(capi.MogeError, match="scalar trunc"):
        A.align_points_scale_z_shift(src, tgt, w, trunc=torch.ones(2, 16))
    with pytest.raises(capi.MogeError, match="eps"):
        A.align(src[..., 2], tgt[..., 2], w, eps=1e-6)


def test_size_bound_is_rejected_before_any_launch():
    """The bound is checked before the library touches a device: the calls fail with the bound in the message even on a host without
    a GPU, and with null data pointers."""
    L = capi.lib()
    size = C.c_size_t()
    assert L.moge_align(1, 1, 1, None, 0, 1, 12289, 1, 1, 1, None, 0, None) != 0
    assert b"12288" in L.moge_last_error()
    assert L.moge_align_anchored(1, 1, 1, capi.ANCHOR_POINTS_XYZ, -1.0, 1, 4097, 1, 1, 1, None, 0, None) != 0
    assert b"4096" in L.moge_last_error()
    assert L.moge_align_workspace_bytes(capi.ANCHOR_DEPTH, 1, 1, 5000, C.byref(size)) != 0
    assert b"4096" in L.moge_last_error()
    assert L.moge_align_anchored(1, 1, 1, 7, -1.0, 1, 16, 1, 1, 1, None, 0, None) != 0
    assert b"mode" in L.moge_last_error()
    x = torch.zeros(2, 4097, 3)
    with pytest.raises(capi.MogeError, match="4096"):
        A.align_points_scale_xyz_shift(x, x, x[..., 0])
    with pytest.raises(capi.MogeError, match="12288"):
        A.align(x[0, :, 0].repeat(4), x[0, :, 0].repeat(4), x[0, :, 0].repeat(4))


# ------------------------------------------------------------------------------------------------------------ GPU: golden parity
@gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_golden_parity(case):
    fn = case["fn"]
    args = _args(case)
    got = getattr(A, fn)(*_cuda(args))
    got = tuple(g.cpu() for g in (got if isinstance(got, tuple) else (got,)))
    ref = case["outputs"]
    if fn == "align":
        got, ref = got[:1], ref[:1]          # loss and index are checked through the objective
    if fn == "align_affine_lstsq":
        for g, r in zip(got, ref):
            assert torch.allclose(g, r, rtol=1e-4, atol=1e-5), (g, r)
        return
    oe, orf = objective(fn, args, got), objective(fn, args, ref)
    assert torch.isfinite(oe).all()
    assert (oe <= orf * (1 + 1e-6) + 1e-12).all(), (oe, orf)
    assert ((oe - orf).abs() <= 1e-5 * orf.abs() + 1e-12).all(), (oe, orf)
    tie = (oe - orf).abs() <= 1e-6 * orf.abs() + 1e-12
    for g, r in zip(got, ref):
        close = torch.isclose(g, r, rtol=1e-5, atol=1e-6)
        if close.dim() > tie.dim():
            close = close.all(-1)
        if not close.all():
            print(f"{_case_id(case)}: values differ where the objectives tie within 1e-6:", g[~close].tolist(), r[~close].tolist())
        assert (close | tie).all(), (g, r, oe, orf)


# ------------------------------------------------------------------------------------------------------------ GPU: brute force
def _plain_objectives(x, y, w, t):
    """fp64 objective at every candidate a_i = y_i / max(x_i, 1e-7) (signs flipped, fp32 as the reference); rows (b, n) -> (b, n)"""
    s = torch.sign(x)
    xs, ys = x * s, y * s
    a = (ys / xs.clamp_min(1e-7)).double()
    r = w.double()[:, None, :] * (a[:, :, None] * x.double()[:, None, :] - y.double()[:, None, :]).abs()
    return _trunc_terms(r, t).sum(-1)


def _anchored_problem(src, tgt, w, b, p, mode):
    if mode == capi.ANCHOR_DEPTH:
        return src[b] - src[b, p], tgt[b] - tgt[b, p], w[b]
    off_s, off_t = src[b, p].clone(), tgt[b, p].clone()
    if mode == capi.ANCHOR_POINTS_Z:
        off_s[:2] = 0
        off_t[:2] = 0
    return (src[b] - off_s).flatten(), (tgt[b] - off_t).flatten(), w[b][:, None].expand(-1, 3).flatten()


def _anchored_check(src, tgt, w, t, mode):
    """the fp64 objective at the engine's (anchor, element) equals the least over every positive-weight anchor and candidate"""
    _, anchor, index = A._anchored(mode, src.cuda(), tgt.cuda(), w.cuda(), t, src.shape[0], src.shape[1])
    for b in range(src.shape[0]):
        best = min(float(_plain_objectives(*(v[None] for v in _anchored_problem(src, tgt, w, b, p, mode)), t).min())
                   for p in torch.nonzero(w[b] > 0).flatten().tolist())
        got = float(_plain_objectives(*(v[None] for v in _anchored_problem(src, tgt, w, b, int(anchor[b]), mode)), t)[0, int(index[b])])
        assert abs(got - best) <= 1e-6 * abs(best) + 1e-12, (mode, b, got, best)


@gpu
@pytest.mark.parametrize("trunc", [None, 0.1])
@pytest.mark.parametrize("n", [37, 96])
def test_brute_force_minimum(n, trunc):
    src, tgt, w = synthetic_alignment_case((3,), n, 90 + n)
    z, zt = src[..., 2], tgt[..., 2]
    for x, y, ww in ((z, zt, w), (src.flatten(-2), tgt.flatten(-2), w[..., None].expand(-1, -1, 3).flatten(-2))):
        _, _, index = A.align(x.cuda(), y.cuda(), ww.cuda(), trunc)
        objs = _plain_objectives(x, y, ww, trunc)
        got = objs.gather(1, index.cpu()[:, None])[:, 0]
        assert torch.allclose(got, objs.min(-1).values, rtol=1e-6, atol=1e-12), (got, objs.min(-1).values)
    _anchored_check(z, zt, w, trunc, capi.ANCHOR_DEPTH)
    _anchored_check(src, tgt, w, trunc, capi.ANCHOR_POINTS_Z)
    _anchored_check(src, tgt, w, trunc, capi.ANCHOR_POINTS_XYZ)


# ------------------------------------------------------------------------------------------------------------ GPU: properties
@gpu
@pytest.mark.parametrize("trunc", [None, 0.1])
def test_batch_results_are_bit_identical_to_single_problems_and_repeatable(trunc):
    src, tgt, w = (t.cuda() for t in synthetic_alignment_case((5,), 300, 7))
    for fn in (A.align_points_scale_xyz_shift, A.align_points_scale_z_shift):
        s1, h1 = fn(src, tgt, w, trunc)
        s2, h2 = fn(src, tgt, w, trunc)
        assert torch.equal(s1, s2) and torch.equal(h1, h2)
        for b in range(5):
            sb, hb = fn(src[b:b + 1], tgt[b:b + 1], w[b:b + 1], trunc)
            assert torch.equal(sb[0], s1[b]) and torch.equal(hb[0], h1[b])
    s1, h1 = A.align_depth_affine(src[..., 2], tgt[..., 2], w, trunc)
    for b in range(5):
        sb, hb = A.align_depth_affine(src[b, :, 2], tgt[b, :, 2], w[b], trunc)
        assert torch.equal(sb, s1[b]) and torch.equal(hb, h1[b])
    a1, l1, i1 = A.align(src[..., 2], tgt[..., 2], w, trunc)
    a2, l2, i2 = A.align(src[..., 2], tgt[..., 2], w, trunc)
    assert torch.equal(a1, a2) and torch.equal(l1, l2) and torch.equal(i1, i2)
    for b in range(5):
        ab, lb, ib = A.align(src[b, :, 2], tgt[b, :, 2], w[b], trunc)
        assert torch.equal(ab, a1[b]) and torch.equal(ib, i1[b])


@gpu
@pytest.mark.parametrize("trunc", [None, 0.1])
def test_large_batches_match_single_problems(trunc):
    """More problems than resident CTAs: a plain-align CTA solves several problems in turn (reusing its shared memory and truncated
    scratch), and the anchored grid has one anchor range per image."""
    src, tgt, w = (t.cuda() for t in synthetic_alignment_case((400,), 64, 12))
    x, y = src[..., 2], tgt[..., 2]
    a, loss, index = A.align(x, y, w, trunc)
    scale, shift = A.align_points_scale_xyz_shift(src, tgt, w, trunc)
    for b in range(400):
        ab, lb, ib = A.align(x[b], y[b], w[b], trunc)
        assert torch.equal(ab, a[b]) and torch.equal(ib, index[b]), b
        if trunc is not None:            # the untruncated loss is a torch sum, whose reduction order may follow the batch shape
            assert torch.equal(lb, loss[b]), b
    for b in range(0, 400, 37):
        sb, hb = A.align_points_scale_xyz_shift(src[b], tgt[b], w[b], trunc)
        assert torch.equal(sb, scale[b]) and torch.equal(hb, shift[b]), b


@gpu
def test_images_without_positive_weight_get_nan():
    src, tgt, w = (t.cuda() for t in synthetic_alignment_case((3,), 50, 8))
    w[1] = 0
    s, h = A.align_points_scale_xyz_shift(src, tgt, w)
    assert torch.isnan(s[1]) and torch.isnan(h[1]).all() and torch.isfinite(s[[0, 2]]).all()
    s, h = A.align_depth_affine(src[..., 2], tgt[..., 2], w, 0.1)
    assert torch.isnan(s[1]) and torch.isnan(h[1]) and torch.isfinite(s[[0, 2]]).all()


@gpu
def test_gradient_flows_through_the_closed_form():
    src, tgt, w = (t.cuda() for t in synthetic_alignment_case((2,), 200, 9))
    src.requires_grad_(True)
    tgt.requires_grad_(True)
    scale, shift = A.align_points_scale_xyz_shift(src, tgt, w, 0.1)
    gs, gt = torch.autograd.grad(scale.sum() + shift.sum(), (src, tgt))
    _, anchor, index = A._anchored(capi.ANCHOR_POINTS_XYZ, src.detach(), tgt.detach(), w, 0.1, 2, 200)
    s2, t2 = src.detach().double().requires_grad_(True), tgt.detach().double().requires_grad_(True)
    i1 = anchor * 3 + index % 3
    fs, ft = s2.flatten(-2), t2.flatten(-2)
    src_1, tgt_1 = fs.gather(1, i1[:, None])[:, 0], ft.gather(1, i1[:, None])[:, 0]
    src_2, tgt_2 = fs.gather(1, index[:, None])[:, 0], ft.gather(1, index[:, None])[:, 0]
    sc = (tgt_2 - tgt_1) / torch.where(src_2 != src_1, src_2 - src_1, 1.0)
    ia = anchor[:, None, None].expand(-1, -1, 3)
    sh = t2.gather(1, ia)[:, 0] - sc[:, None] * s2.gather(1, ia)[:, 0]
    es, et = torch.autograd.grad(sc.sum() + sh.sum(), (s2, t2))
    assert torch.allclose(gs.double(), es, rtol=1e-4, atol=1e-5) and torch.allclose(gt.double(), et, rtol=1e-4, atol=1e-5)
    assert gs.abs().sum() > 0


@gpu
@pytest.mark.parametrize("weighted", [False, True])
def test_affine_lstsq_matches_linalg_lstsq(weighted):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 3, 50_000, generator=g) + 2.0
    y = 1.7 * x - 0.4 + 0.1 * torch.randn(2, 3, 50_000, generator=g)
    w = torch.rand(2, 3, 50_000, generator=g) if weighted else None
    a, b = A.align_affine_lstsq(x.cuda(), y.cuda(), None if w is None else w.cuda())
    ws = torch.ones_like(x).double() if w is None else w.sqrt().double()
    M = torch.stack([ws * x.double(), torch.ones_like(x).double()], dim=-1)
    ea, eb = torch.linalg.lstsq(M, (ws * y.double())[..., None]).solution.squeeze(-1).unbind(-1)
    assert torch.allclose(a.cpu().double(), ea, rtol=1e-5, atol=1e-6) and torch.allclose(b.cpu().double(), eb, rtol=1e-5, atol=1e-6)
