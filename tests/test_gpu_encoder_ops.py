"""-m gpu: operator tests of the encoder's row plumbing, each against a plain fp64 reference of the same operation:

- K1 preprocess: antialiased bilinear resize to (14h, 14w), ImageNet normalisation, im2col into 592-column rows;
- K3 pos table: bicubic resampling of the 37 x 37 pos-embed grid at ((h+0.1)/37, (w+0.1)/37), + the patch bias; the cls row;
- patch embed: the EPI_PATCH GEMM (row b*(T+1)+1+t = patches[b*T+t] W^T + table[t]) and the cls rows;
- the LayerNorm-fold producer of patch embed and of EPI_RESID (proj, fc2): the fp32 row, its 16-bit copy x16 and the per-group
  (sum, sum of squares) of the rounded row in stats[row, part];
- ln_rstd, the chain producer -> ln_rstd -> folded-LayerNorm consumer, and the tap LayerNorm.

The faults these catch are local (a token-to-row mapping off at an image boundary, a statistics slot at the wrong part, a ragged
last row tile without its x16 or statistics, a pos-table row off by one on a one-row grid): each spoils a few rows, which the
24 blocks of attention after them would mix away in an end-to-end comparison.  So every output is prefilled with NaN and the rows
past its end with a finite sentinel, and every test asserts that every row was written and that nothing past the end was touched.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from moge_b200.configs import IMAGE_MEAN, IMAGE_STD, INTERP_OFFSET, LN_EPS, PATCH, POS_GRID
from oracle.moge_port import pos_embed_for_grid
from gpu_util import rel_l2, stream, dt, check_tiles, TILE_LINEAR

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}      # test_gpu_ops' tolerances for 16-bit outputs
RESID_TOL = 2e-5 + 1e-4                                  # test_linear_residual_layerscale's bound on x - res
SENTINEL = 1232.0      # exact in fp16, bf16 and fp32 (77 * 16)
PAD = 64               # rows past the end that must stay untouched
STATS_LD = 16          # MOGE_STATS_LD
KP = 592               # patch row width: 3 * 14 * 14 = 588 columns, zero-padded to a multiple of 16
U = 2.0 ** -24         # fp32 unit roundoff
NAN = float("nan")


def lib():
    return capi.lib()


def prefilled(rows, *shape, dtype=torch.float32):
    """rows + PAD rows of `shape`: NaN in the first `rows`, SENTINEL after them"""
    t = torch.full((rows + PAD, *shape), NAN, dtype=dtype, device=DEV)
    t[rows:] = SENTINEL
    return t


def untouched(t, rows):
    return bool((t[rows:].float() == SENTINEL).all())


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ the producer contract
def check_producer(x, x16, stats, parts, M, dtype, what):
    """The LayerNorm-fold producer's contract on rows [0, M) of x (fp32), x16 and stats [rows, STATS_LD, 2], independent of the
    column-group width: x16 is the rounded x, slots [0, parts) hold the partial sums of the ROUNDED row and [parts, STATS_LD) are
    not written, and rows past M are untouched.  The slots' total must match the fp64 (sum x16, sum x16^2) of the row within
    (N+1) 2^-24 sum|term|: the first-order worst case of fp32 summation of N terms in any order (N-1 roundings), with one more
    rounding for each square."""
    N = x.shape[1]
    assert 1 <= parts <= STATS_LD and N % parts == 0, f"{what}: parts = {parts} for N = {N}"
    assert untouched(x, M) and untouched(x16, M) and untouched(stats, M), f"{what}: a row past M = {M} was written"
    xs, hs, ss = x[:M], x16[:M], stats[:M]
    assert bool(torch.isfinite(xs).all()), f"{what}: an fp32 row below M was not written"
    assert torch.equal(hs, xs.to(dtype)), f"{what}: x16 is not the rounded fp32 row"
    assert bool(torch.isfinite(ss[:, :parts]).all()), f"{what}: a statistics slot below parts = {parts} was not written"
    assert bool(torch.isnan(ss[:, parts:]).all()), f"{what}: a statistics slot at or past parts = {parts} was written"
    h = hs.double()
    tot = ss[:, :parts].double().sum(1)
    sq = h.square().sum(1)
    e1 = ((tot[:, 0] - h.sum(1)).abs() / ((N + 1) * U * h.abs().sum(1))).max().item()
    e2 = ((tot[:, 1] - sq).abs() / ((N + 1) * U * sq)).max().item()
    print(f"producer {what}: parts {parts}, row sums at {e1:.3f} and {e2:.3f} of their bounds")
    assert e1 <= 1 and e2 <= 1, f"{what}: statistics off the rounded rows' sums ({e1:.2f}, {e2:.2f} of the bound)"


def run_ln_rstd(stats, parts, M, D):
    rstd = prefilled(M)
    capi.check(lib().moge_op_ln_rstd(stats.data_ptr(), parts, M, D, rstd.data_ptr(), stream()))
    torch.cuda.synchronize()
    assert untouched(rstd, M), "ln_rstd wrote past its rows"
    return rstd[:M]


def check_rstd(rstd, x16, what):
    """rstd of the rounded rows against fp64, within (3/2)(D+2) 2^-24 (1 + mu^2/sigma^2) relative (see test_ln_rstd)"""
    h = x16.double()
    D = h.shape[1]
    mu, var = h.mean(1), h.var(1, unbiased=False)
    ref = 1 / torch.sqrt(var + LN_EPS)
    bound = 1.5 * (D + 2) * U * (1 + mu.square() / var)
    r = ((rstd.double() - ref).abs() / ref / bound)
    print(f"ln_rstd {what}: worst row at {r.max().item():.3f} of its bound (mu/sigma up to {(mu.abs() / var.sqrt()).max().item():.1f})")
    assert bool(torch.isfinite(rstd).all()), f"{what}: an rstd row was not written"
    assert r.max().item() <= 1, f"{what}: rstd of row {int(r.argmax())} is {r.max().item():.2f} times its bound"


# ------------------------------------------------------------------------------------------------ K1 preprocess
def im2col(x, h, w):
    """(B, 3, 14h, 14w) -> (B*h*w, 588), column (c, py, px)"""
    B = x.shape[0]
    return x.reshape(B, 3, h, PATCH, w, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(B * h * w, 3 * PATCH * PATCH)


def normalise_patches(img, h, w, ftype):
    """the K1 chain in `ftype` on img's device: resize (unless the grid is the image's own), normalise, im2col"""
    x = img.to(ftype)
    if x.shape[-2:] != (PATCH * h, PATCH * w):
        x = F.interpolate(x, (PATCH * h, PATCH * w), mode="bilinear", align_corners=False, antialias=True)
    mean = torch.tensor(IMAGE_MEAN, dtype=ftype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(IMAGE_STD, dtype=ftype, device=x.device).view(1, 3, 1, 1)
    return im2col((x - mean) / std, h, w)


def run_preprocess(img, h, w, dtype):
    B, _, H, W = img.shape
    M = B * h * w
    out = prefilled(M, KP, dtype=dtype)
    capi.check(lib().moge_op_preprocess(img.data_ptr(), dt(img.dtype), B, H, W, h, w, out.data_ptr(), dt(dtype), stream()))
    torch.cuda.synchronize()
    assert untouched(out, M), "preprocess wrote past its rows"
    return out[:M]


def ulp16(v, dtype):
    """the spacing of `dtype` at |v| (subnormal spacing below the normal range)"""
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** emin)))
    return torch.exp2(e - mant)


PRE_CASES = [      # (B, H, W, h, w)
    (1, 518, 518, 37, 37),       # the identity grid
    (1, 1036, 777, 37, 28),      # down-sampling in both directions at a non-integer ratio
    (1, 98, 126, 10, 12),        # up-sampling
    (1, 700, 200, 20, 20),       # down rows, up columns
    (1, 30, 700, 1, 50),         # a one-row grid
    (1, 700, 30, 50, 1),         # a one-column grid
    (3, 200, 150, 12, 9),        # three distinct images
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("image_dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W,h,w", PRE_CASES)
def test_preprocess(B, H, W, h, w, image_dtype, dtype):
    """Each element within one 16-bit ulp of the fp64 chain plus 2 delta, delta = max |fp32 chain - fp64 chain| of the case (the
    fp32 chain is what the reference project computes; the kernel is another fp32 evaluation of it, in another order).  The four
    pad columns are exactly zero, and on the identity grid the rows are bitwise the normalised image."""
    g = torch.Generator().manual_seed(B * 1000003 + H * 1009 + W + h)
    img = torch.rand(B, 3, H, W, generator=g).to(image_dtype).to(DEV)
    out = run_preprocess(img, h, w, dtype)
    assert bool((out[:, 588:] == 0).all()), "a pad column is not zero"
    got = out[:, :588]
    assert bool(torch.isfinite(got.float()).all()), "a patch row was not written"
    if (H, W) == (PATCH * h, PATCH * w):
        assert torch.equal(got, normalise_patches(img.float(), h, w, torch.float32).to(dtype)), "the identity grid is not bitwise"
    cpu = img.cpu()
    ref = normalise_patches(cpu, h, w, torch.float64)
    delta = (normalise_patches(cpu, h, w, torch.float32).double() - ref).abs().max().item()
    ref = ref.to(DEV)
    err = (got.double() - ref).abs()
    r = (err / (ulp16(ref, dtype) + 2 * delta)).max().item()
    print(f"preprocess {B}x{H}x{W} @ {h}x{w} {image_dtype} -> {dtype}: delta {delta:.2e}, max err {err.max().item():.2e}, "
          f"worst element at {r:.3f} of its bound")
    assert r <= 1, f"an element is {r:.2f} times its bound (delta {delta:.2e})"


# ------------------------------------------------------------------------------------------------ K3 pos table
def pos_inputs(D, seed):
    g = gen(seed)
    pos = torch.randn(1, 1 + POS_GRID * POS_GRID, D, generator=g, device=DEV)       # unit scale, distinct rows
    cls = torch.randn(1, 1, D, generator=g, device=DEV)
    bias = 0.3 * torch.randn(D, generator=g, device=DEV)
    return pos, cls, bias


def run_pos_table(pos, cls, bias, h, w):
    D, T = pos.shape[-1], h * w
    table = prefilled(T, D)
    cls_row = prefilled(1, D)
    capi.check(lib().moge_op_pos_table(pos.data_ptr(), cls.data_ptr(), bias.data_ptr(), D, h, w, table.data_ptr(), cls_row.data_ptr(),
                                       stream()))
    torch.cuda.synchronize()
    assert untouched(table, T) and untouched(cls_row, 1), "pos table wrote past its rows"
    return table[:T], cls_row[0]


def pos_table_reference(pos, bias, h, w):
    """fp64 bicubic (A = -0.75, align_corners=False) of the 37 x 37 grid at scale ((h+0.1)/37, (w+0.1)/37), + bias: (h*w, D)"""
    D = pos.shape[-1]
    grid = pos[0, 1:].double().reshape(1, POS_GRID, POS_GRID, D).permute(0, 3, 1, 2)
    s = ((h + INTERP_OFFSET) / POS_GRID, (w + INTERP_OFFSET) / POS_GRID)
    out = F.interpolate(grid, scale_factor=s, mode="bicubic", align_corners=False, antialias=False)
    assert out.shape[-2:] == (h, w)
    return out.permute(0, 2, 3, 1).reshape(h * w, D) + bias.double()


@pytest.mark.parametrize("D", [384, 1024])
@pytest.mark.parametrize("h,w", [(37, 37), (35, 35), (60, 60), (37, 74), (74, 37), (1, 50), (50, 1), (5, 3), (100, 100)])
def test_pos_table(h, w, D):
    """max |got - ref64| <= 4 max |ref32 - ref64|, ref32 being the fp32 port (oracle.moge_port.pos_embed_for_grid) + bias; the
    fp64 reference is pinned to the port (fp32 against fp64 measured 2.5e-6 to 3.6e-6 of max |ref| over these grids).  At 37 x 37
    the table is bitwise pos + bias, as the reference returns the grid unchanged there.  The cls row is bitwise cls + pos[0]."""
    pos, cls, bias = pos_inputs(D, seed=100 * h + w + D)
    table, cls_row = run_pos_table(pos, cls, bias, h, w)
    assert torch.equal(cls_row, cls[0, 0] + pos[0, 0]), "cls row is not cls + pos[0]"
    assert bool(torch.isfinite(table).all()), "a table row was not written"
    if (h, w) == (POS_GRID, POS_GRID):
        assert torch.equal(table, pos[0, 1:] + bias), "the 37 x 37 table is not bitwise pos + bias"
        return
    ref = pos_table_reference(pos, bias, h, w)
    ref32 = pos_embed_for_grid(pos, h, w)[0, 1:] + bias
    scale = ref.abs().max().item()
    delta = (ref32.double() - ref).abs().max().item()
    err = (table.double() - ref).abs().max().item()
    print(f"pos table {h}x{w} D={D}: |ref32 - ref64| {delta / scale:.2e}, |got - ref64| {err / scale:.2e} of max |ref|")
    assert delta <= 1e-5 * scale, f"the fp64 reference is off the fp32 port by {delta / scale:.2e} of max |ref|"
    assert err <= 4 * delta, f"max |got - ref64| = {err:.3e} > 4 x {delta:.3e}"


# ------------------------------------------------------------------------------------------------ patch embed
# rel-L2 / worst-tile bound of the patch rows against the fp64 product of the op's own patches and table and the 16-bit weight:
# fp32 accumulation over K = 592 and one fp32 rounding of the table add.  Measured on an H100 80GB HBM3 (700 W) over the cases
# below: whole 4.7e-7 to 5.1e-7 (fp16), 3.3e-7 to 3.6e-7 (bf16); worst tile 5.3e-7 and 3.8e-7, at 1.02 to 1.11 times the whole.
PATCH_TOL = 1.5e-6


def patch_inputs(D, seed):
    g = gen(seed)
    w = torch.randn(D, 3, PATCH, PATCH, generator=g, device=DEV) / math.sqrt(3 * PATCH * PATCH)
    b = 0.1 * torch.randn(D, generator=g, device=DEV)
    pos, cls, _ = pos_inputs(D, seed + 1)
    return w, b, pos, cls


def run_patch_embed(img, h, w, wp, bp, pos, cls, dtype):
    B, _, H, W = img.shape
    D = wp.shape[0]
    M = B * (h * w + 1)
    x, x16, stats = prefilled(M, D), prefilled(M, D, dtype=dtype), prefilled(M, STATS_LD, 2)
    parts = C.c_int(0)
    capi.check(lib().moge_op_patch_embed(img.data_ptr(), dt(img.dtype), B, H, W, h, w, wp.data_ptr(), bp.data_ptr(), pos.data_ptr(),
                                         cls.data_ptr(), D, x.data_ptr(), x16.data_ptr(), stats.data_ptr(), C.byref(parts), dt(dtype),
                                         stream()))
    torch.cuda.synchronize()
    return x, x16, stats, parts.value


def patch_image(B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, PATCH * h + 8, PATCH * w + 6, generator=g).to(DEV)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [384, 768, 1024])
@pytest.mark.parametrize("B,h,w", [(1, 37, 37), (3, 10, 12), (5, 16, 8), (2, 1, 50), (2, 50, 1)])
def test_patch_embed(B, h, w, D, dtype):
    """Row b*(T+1)+1+t = patches[b*T+t] W^T + table[t] against fp64 on the op's own patches and table (tested above), so that the
    GEMM epilogue is what is checked; cls rows bitwise cls + pos[0]; the producer contract on every row, cls rows included.
    Cases: one image with a 89-row last tile, row tiles straddling images (T = 120), T = 128, one-row and one-column grids."""
    T, N = h * w, h * w + 1
    wp, bp, pos, cls = patch_inputs(D, seed=D + 31 * T + B)
    img = patch_image(B, h, w, seed=T + B)
    x, x16, stats, parts = run_patch_embed(img, h, w, wp, bp, pos, cls, dtype)
    check_producer(x, x16, stats, parts, B * N, dtype, f"patch embed {B}x({h},{w}) D={D} {dtype}")
    patches = run_preprocess(img, h, w, dtype)
    table, cls_row = run_pos_table(pos, cls, bp, h, w)
    w16 = wp.reshape(D, -1).to(dtype).double()
    ref = (patches[:, :588].double() @ w16.t()).view(B, T, D) + table.double()
    xs = x[:B * N].view(B, N, D)
    assert torch.equal(xs[:, 0], (cls[0, 0] + pos[0, 0]).expand(B, D)), "a cls row is not cls + pos[0]"
    got, ref = xs[:, 1:].reshape(B * T, D), ref.reshape(B * T, D)
    e = rel_l2(got, ref)
    assert e < PATCH_TOL, f"patch rows: rel-L2 {e:.2e}"
    check_tiles(got, ref, TILE_LINEAR, PATCH_TOL, f"patch embed {B}x({h},{w}) D={D} {dtype}")


# ------------------------------------------------------------------------------------------------ EPI_RESID producer
def resid_case(M, D, K, dtype, seed, ratios=(0, 1, 3, 10)):
    """a, W (16-bit), bias, LayerScale gamma of mixed magnitude (1e-3 to 1, both signs), and residual rows with a per-row offset
    mu = r sigma, r cycling through `ratios`"""
    g = gen(seed)
    a = torch.randn(M, K, generator=g, device=DEV).to(dtype)
    w = (torch.randn(D, K, generator=g, device=DEV) / math.sqrt(K)).to(dtype)
    b = torch.randn(D, generator=g, device=DEV)
    sign = torch.randint(0, 2, (D,), generator=g, device=DEV) * 2 - 1
    gamma = sign * torch.pow(10.0, -3 * torch.rand(D, generator=g, device=DEV))
    sigma = 0.5 + 1.5 * torch.rand(M, 1, generator=g, device=DEV)
    r = torch.tensor(ratios, dtype=torch.float32, device=DEV)[torch.arange(M, device=DEV) % len(ratios)].view(M, 1)
    rsign = torch.randint(0, 2, (M, 1), generator=g, device=DEV) * 2 - 1
    res = r * rsign * sigma + sigma * torch.randn(M, D, generator=g, device=DEV)
    return dict(a=a, w=w, b=b, gamma=gamma, res=res)


def run_resid(case, dtype):
    M, K = case["a"].shape
    D = case["w"].shape[0]
    x, x16, stats = prefilled(M, D), prefilled(M, D, dtype=dtype), prefilled(M, STATS_LD, 2)
    x[:M] = case["res"]
    parts = C.c_int(0)
    capi.check(lib().moge_op_linear_resid_ln(case["a"].data_ptr(), case["w"].data_ptr(), case["b"].data_ptr(), case["gamma"].data_ptr(),
                                             x.data_ptr(), x16.data_ptr(), stats.data_ptr(), C.byref(parts), M, D, K, dt(dtype),
                                             stream()))
    torch.cuda.synchronize()
    return x, x16, stats, parts.value


@pytest.mark.parametrize("M", [1, 100, 128, 129, 1370, 2741, 8229, 43840])
@pytest.mark.parametrize("K_mult", [1, 4], ids=["proj", "fc2"])
@pytest.mark.parametrize("D", [384, 768, 1024])
@pytest.mark.parametrize("dtype", DTYPES)
def test_linear_resid_producer(dtype, D, K_mult, M):
    """x += gamma (a W^T + b) with the producer side on: the GEMM's contribution x - res against fp64, tile by tile, as
    test_linear_residual_layerscale checks it, then the producer contract.  M: one row, one partial tile, one full tile, a
    one-row last tile, the batch-1 and batch-2 rows, and 6 x 1371 + 3 and 32 x 1370 rows."""
    K = K_mult * D
    case = resid_case(M, D, K, dtype, seed=M + 7 * D + K)
    x, x16, stats, parts = run_resid(case, dtype)
    what = f"resid M={M} D={D} K={K} {dtype}"
    check_producer(x, x16, stats, parts, M, dtype, what)
    ref = case["gamma"].double() * (case["a"].double() @ case["w"].double().t() + case["b"].double())
    got = x[:M].double() - case["res"].double()
    e = rel_l2(got, ref)
    assert e < RESID_TOL, f"{what}: rel-L2 {e:.2e}"
    check_tiles(got, ref, TILE_LINEAR, RESID_TOL, what)


def test_linear_resid_rejects_more_statistics_groups_than_slots():
    """N = 1152 needs 18 groups of 64 columns, more than the 16 slots per row: the call fails before it launches, x unchanged"""
    M, D, K, dtype = 256, 1152, 384, torch.float16
    case = resid_case(M, D, K, dtype, seed=5)
    x, x16, stats = prefilled(M, D), prefilled(M, D, dtype=dtype), prefilled(M, STATS_LD, 2)
    x[:M] = case["res"]
    x0, x160, stats0 = x.clone(), x16.clone(), stats.clone()
    parts = C.c_int(-1)
    rc = lib().moge_op_linear_resid_ln(case["a"].data_ptr(), case["w"].data_ptr(), case["b"].data_ptr(), case["gamma"].data_ptr(),
                                       x.data_ptr(), x16.data_ptr(), stats.data_ptr(), C.byref(parts), M, D, K, dt(dtype), stream())
    torch.cuda.synchronize()
    assert rc != 0
    assert "statistics groups" in lib().moge_last_error().decode()
    assert torch.equal(x, x0), "x changed"
    assert torch.equal(x16[M:], x160[M:]) and bool(torch.isnan(x16[:M]).all()) and torch.equal(stats[M:], stats0[M:])
    assert bool(torch.isnan(stats[:M]).all())


# ------------------------------------------------------------------------------------------------ ln_rstd
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [384, 768, 1024])
@pytest.mark.parametrize("producer", ["patch_embed", "resid"])
def test_ln_rstd(producer, D, dtype):
    """rstd = 1 / sqrt(E[x^2] - E[x]^2 + eps) from a producer's partial sums, against the fp64 rstd of its x16 rows.

    Bound, first order in u = 2^-24, with S1 = sum x, S2 = sum x^2 over the row's D rounded values, mu = S1/D, sigma^2 = S2/D - mu^2:
    - fp32 summation in any order (the producer's groups, then the slots here) gives |dS2| <= (D+1) u S2 (D-1 additions, one
      rounding per square) and |dS1| <= (D-1) u sum|x| <= (D-1) u sqrt(D S2);
    - so d(S2/D) <= (D+1) u (sigma^2 + mu^2) and d(mu^2) = 2 |mu| |dS1| / D <= 2 (D-1) u |mu| sqrt(sigma^2 + mu^2)
      <= (D-1) u (sigma^2 + 2 mu^2);
    - the products by 1/D, the square of mu and the subtraction add a few u (sigma^2 + mu^2), well inside the (D+2) - (D+1) slack;
    - so var is within 3 (D+2) u (sigma^2 + mu^2) absolute, i.e. 3 (D+2) u (1 + mu^2/sigma^2) relative, and rstd = var^-1/2
      (eps only shrinks the relative error; rsqrtf adds 2^-22) within (3/2) (D+2) u (1 + mu^2/sigma^2).
    This pins the domain elementwise.cu documents for the single-pass form: |mu| up to about 10 sigma, where the bound is ~1e-2 at
    D = 1024, and the rows here reach mu = 10 sigma."""
    if producer == "patch_embed":
        B, h, w = 3, 10, 12
        wp, bp, pos, cls = patch_inputs(D, seed=D + 17)
        x, x16, stats, parts = run_patch_embed(patch_image(B, h, w, seed=3), h, w, wp, bp, pos, cls, dtype)
        M = B * (h * w + 1)
    else:
        M = 2741
        x, x16, stats, parts = run_resid(resid_case(M, D, D, dtype, seed=D + 3), dtype)
    rstd = run_ln_rstd(stats, parts, M, D)
    check_rstd(rstd, x16[:M], f"{producer} D={D} {dtype}")


# ------------------------------------------------------------------------------------------------ producer -> ln_rstd -> consumer
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,D", [(1370, 384), (1370, 768), (1370, 1024), (43840, 1024)])
@pytest.mark.parametrize("N_mult,epi", [(3, 0), (4, 1)], ids=["qkv", "fc1"])
def test_producer_rstd_consumer_chain(N_mult, epi, M, D, dtype):
    """The engine's proj -> ln_rstd -> qkv (N = 3D, store) and fc2 -> ln_rstd -> fc1 (N = 4D, GELU) on the producer's own rows,
    against fp64 F.linear(F.layer_norm(x)) of the new fp32 rows.  M = 1370 runs 128 x 128 consumer tiles, M = 43840 at D = 1024
    the 128 x 256 ones.  The rows' offsets go up to 3 sigma: at 10 sigma the 16-bit rounding of the row itself (the fold's operand)
    would by estimate cost about 2% in bf16, more than TOL."""
    N = N_mult * D
    case = resid_case(M, D, D, dtype, seed=M + D + epi, ratios=(0, 1, 3))
    x, x16, stats, parts = run_resid(case, dtype)
    rstd = run_ln_rstd(stats, parts, M, D)
    g = gen(M + N)
    lg = 1 + 0.3 * torch.randn(D, generator=g, device=DEV)
    lb = 0.2 * torch.randn(D, generator=g, device=DEV)
    w = torch.randn(N, D, generator=g, device=DEV) / math.sqrt(D)
    b = torch.randn(N, generator=g, device=DEV)
    out = prefilled(M, N, dtype=dtype)
    capi.check(lib().moge_op_linear_ln_rows(x16.data_ptr(), rstd.data_ptr(), lg.data_ptr(), lb.data_ptr(), w.data_ptr(), b.data_ptr(),
                                            out.data_ptr(), M, N, D, epi, dt(dtype), stream()))
    torch.cuda.synchronize()
    assert untouched(out, M), "the consumer wrote past M"
    got = out[:M]
    assert bool(torch.isfinite(got.float()).all()), "a consumer row below M was not written"
    ref = F.linear(F.layer_norm(x[:M].double(), (D,), lg.double(), lb.double(), LN_EPS), w.double(), b.double())
    if epi == 1:
        ref = F.gelu(ref)
    e = rel_l2(got, ref)
    assert e < TOL[dtype], f"rel-L2 {e:.2e}"
    check_tiles(got, ref, TILE_LINEAR, TOL[dtype], f"chain M={M} D={D} N={N} {dtype}")


# ------------------------------------------------------------------------------------------------ tap LayerNorm
# rel-L2 bound of the tap LayerNorm's fp32 cls rows against fp64 (two-pass statistics and the affine map in fp32).  Measured on an
# H100 80GB HBM3 (700 W): 4.0e-8 to 2.4e-7.
CLS_TOL = 1e-6


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_cls", [True, False], ids=["cls_out", "no_cls"])
@pytest.mark.parametrize("tap", [0, 3])
@pytest.mark.parametrize("T", [120, 1369])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("D", [384, 1024])
def test_layernorm_taps(D, B, T, tap, with_cls, dtype):
    """Tap `tap` of 4: patch row (b, t) lands at row b*T + t, columns [tap*D, (tap+1)*D) of the (B*T, 4D) tap buffer, every other
    column keeps the sentinel; cls rows go to cls_out only, in fp32.  Against fp64 F.layer_norm with TOL and the tile check."""
    N, ld, off = T + 1, 4 * D, tap * D
    g = gen(D + B + T + tap)
    sigma = 0.5 + 2 * torch.rand(B * N, 1, generator=g, device=DEV)
    x = sigma * torch.randn(B * N, D, generator=g, device=DEV) + 3 * torch.randn(B * N, 1, generator=g, device=DEV)
    gm = 1 + 0.3 * torch.randn(D, generator=g, device=DEV)
    bt = 0.2 * torch.randn(D, generator=g, device=DEV)
    out = torch.full((B * T + PAD, ld), SENTINEL, dtype=dtype, device=DEV)
    out[:B * T, off:off + D] = NAN
    cls_out = prefilled(B, D) if with_cls else None
    capi.check(lib().moge_op_layernorm_taps(x.data_ptr(), gm.data_ptr(), bt.data_ptr(), out.data_ptr(), capi.ptr(cls_out), B, N, D, ld,
                                            off, dt(dtype), stream()))
    torch.cuda.synchronize()
    ref = F.layer_norm(x.double(), (D,), gm.double(), bt.double(), LN_EPS).view(B, N, D)
    got = out[:B * T, off:off + D]
    assert bool(torch.isfinite(got.float()).all()), "a patch row of the tap slice was not written"
    rest = out.clone()
    rest[:B * T, off:off + D] = SENTINEL
    assert bool((rest.float() == SENTINEL).all()), "a column outside the tap slice, or a row past B*T, was written"
    ref_p = ref[:, 1:].reshape(B * T, D)
    e = rel_l2(got, ref_p)
    assert e < TOL[dtype], f"rel-L2 {e:.2e}"
    check_tiles(got, ref_p, TILE_LINEAR, TOL[dtype], f"tap LayerNorm B={B} T={T} D={D} tap {tap} {dtype}")
    if with_cls:
        assert untouched(cls_out, B), "cls_out written past B rows"
        ec = rel_l2(cls_out[:B], ref[:, 0])
        print(f"tap LayerNorm cls rows: rel-L2 {ec:.2e}")
        assert ec < CLS_TOL, f"cls rows: rel-L2 {ec:.2e}"

