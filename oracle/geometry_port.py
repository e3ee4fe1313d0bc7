"""fp64 restatements of the reference's `refine_depth_with_normal`, `dilate_with_mask(filter='mean')` and `gaussian_blur_2d`
(moge/utils/geometry_torch.py), each with a per-element bound on the error of an fp32 computation of the same function.
TEST INFRASTRUCTURE ONLY: tests/test_gpu_geometry_torch.py bounds the kernels of moge_b200/csrc/geometry.cu with them, and
tests/test_geometry_torch_host.py pins them to the reference's own fp32 outputs in tests/golden/geometry.pt.  Also the masked
window min / max of `dilate_with_mask` that the reference's code means (it calls Tensor.min / max with a tuple of dims, which
torch rejects), in fp32, from which the golden takes those cases.

The bounds are first-order forward error bounds in units of u = 2^-24 (fp32 rounding), accumulated alongside the fp64 values:
each rounded operation adds u times the magnitude of its result, a sum of n terms adds n u times the sum of their magnitudes in
any order, logf / expf add 1 and 2 ulp (2u and 4u relative), and errors already present propagate through the operation's
partial derivatives, evaluated with the fp64 values.  The terms dropped are of second order in the errors; a factor of 2 on
the result covers them (SAFETY).  The fp32 constants of the reference (0.1, 0.9, damp, eps and the clamp bound 0.1 enter its
fp32 arithmetic as fp32 operands) are the fp32 values here too, so they carry no error of their own.
"""
import inspect
import math

import numpy as np
import torch

U = 2.0 ** -24
SAFETY = 2.0


def f32(x: float) -> float:
    """x rounded to fp32, as the reference's fp32 tensor arithmetic takes a Python float operand."""
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------------------ refine
def _taps(k: int, H: int, W: int, eps: float):
    """per tap (a, b) in row-major order: (offset a - r, b - r, duv x, duv y, 1 / (10 max(|duv|, eps)))"""
    r = k // 2
    out = []
    for a in range(k):
        for b in range(k):
            dx, dy = (b - r) / W, (a - r) / H
            out.append((a, b, dx, dy, 1.0 / (10.0 * max(math.hypot(dx, dy), eps))))
    return out


def _grad(normal: torch.Tensor, intrinsics: torch.Tensor, H: int, W: int):
    """(g (B, H, W, 2), magnitude bound of its numerator / denominator terms) of g = -(n_xy K2) / (n_z + n_xy . (K2 uv + k))"""
    Ki = torch.inverse(intrinsics)                                   # (B, 3, 3)
    K2, kt = Ki[:, None, None, :2, :2], Ki[:, None, None, :2, 2]
    u = (torch.arange(W, dtype=torch.float64) + 0.5) / W
    v = (torch.arange(H, dtype=torch.float64) + 0.5) / H
    uv = torch.stack(torch.meshgrid(u, v, indexing="xy"), dim=-1)    # (H, W, 2)
    nxy, nz = normal[..., :2], normal[..., 2]
    ray = (K2 @ uv[None, ..., None]).squeeze(-1) + kt                # (B, H, W, 2)
    den = nz + (nxy * ray).sum(-1)
    num = (nxy[..., None, :] @ K2).squeeze(-2)                       # n_xy K2: (B, H, W, 2)
    g = -num / den[..., None]
    # magnitudes of the terms an fp32 evaluation rounds (K2 from an fp32 inverse, uv from fp32 arithmetic)
    num_mag = (nxy.abs()[..., None, :] @ K2.abs()).squeeze(-2)
    den_mag = nz.abs() + (nxy.abs() * ((K2.abs() @ uv[None, ..., None]).squeeze(-1) + kt.abs())).sum(-1)
    dg = (num_mag / den.abs()[..., None] + g.abs() * (den_mag / den.abs())[..., None]) * 8 * U + U * g.abs()
    return g, dg


def refine_depth_with_normal(depth, normal, intrinsics, iterations: int = 10, damp: float = 1e-3, eps: float = 1e-12,
                             kernel_size: int = 5, fp32_grad: bool = False):
    """(refined depth (B, H, W) fp64, bound (B, H, W)) of depth (B, H, W), normal (B, H, W, 3), intrinsics (B, 3, 3) (fp32 inputs).
    The bound is on |fp32 result - fp64 result| of an implementation that takes log and exp in fp32, the weights, their sum and
    the sweeps in fp32 with one rounding per operation and sums in any order, and the Laplacian term rounded once to fp32 from
    fp64 (the GPU kernels), or with `fp32_grad` the gradient and the Laplacian term in fp32 too (the reference)."""
    depth, normal, intrinsics = depth.double(), normal.double(), intrinsics.double()
    B, H, W = depth.shape
    r = kernel_size // 2
    eps32, damp32, c01, c09, clampv = f32(eps), f32(damp), f32(0.1), f32(0.9), f32(0.1)
    ld = depth.clamp_min(eps32).log()
    e_ld = 2 * U * ld.abs()
    if iterations <= 0 or H <= 2 * r or W <= 2 * r:
        out = ld.exp()
        return out, SAFETY * out * (e_ld + 4 * U)
    I = (slice(None), slice(r, H - r), slice(r, W - r))
    h, w = H - 2 * r, W - 2 * r

    def win(x, a, b):                                                # x at offset (a - r, b - r) of every interior pixel
        return x[:, a:a + h, b:b + w]

    ldc, e_ldc = ld[I], e_ld[I]
    g, dg = _grad(normal, intrinsics, H, W)
    if not fp32_grad:
        dg = torch.zeros_like(dg)
    gc, dgc = g[I], dg[I]
    tc_rel = 8 * U if fp32_grad else 4 * U                           # rounding of t = (ld_n - ld_c) / |duv| / 10
    taps = _taps(kernel_size, H, W, eps32)
    ws, ews = [], []
    tot = torch.zeros(B, h, w, dtype=torch.float64)
    lap = torch.zeros_like(tot)
    e_lap = torch.zeros_like(tot)
    lap_mag = torch.zeros_like(tot)
    for a, b, dx, dy, c in taps:
        t = (win(ld, a, b) - ldc) * c
        dt = c * (win(e_ld, a, b) + e_ldc) + tc_rel * t.abs()
        wk = torch.exp(-t * t)
        ew = wk * (2 * t.abs() * dt + 2 * U * t * t + 4 * U)
        gs = win(g, a, b) + gc
        ak = gs[..., 0] * (dx / 2) + gs[..., 1] * (dy / 2)
        tot += wk
        lap += wk * ak
        lap_mag += wk * (gs[..., 0].abs() * abs(dx / 2) + gs[..., 1].abs() * abs(dy / 2))
        e_lap += ew * ak.abs() + wk * ((win(dg, a, b) + dgc)[..., 0] * abs(dx / 2) + (win(dg, a, b) + dgc)[..., 1] * abs(dy / 2))
        ws.append(wk)
        ews.append(ew)
    n = len(taps)
    e_tot = sum(ews) + n * U * tot
    e_lap += ((n + 6) * U * lap_mag) if fp32_grad else U * lap.abs()
    e_lap = torch.where(lap.abs() - e_lap > clampv, torch.zeros_like(e_lap), e_lap)    # saturated: the clamp absorbs the error
    lap = lap.clamp(-clampv, clampv)
    cterm = damp32 * ldc - lap
    e_c = damp32 * e_ldc + e_lap + U * (damp32 * ldc.abs() + cterm.abs())
    den = tot + damp32
    e_den = e_tot + U * den
    x, e = ld.clone(), e_ld.clone()
    for _ in range(iterations):
        s = torch.zeros_like(tot)
        e_s = torch.zeros_like(tot)
        s_mag = torch.zeros_like(tot)
        for (a, b, _, _, _), wk, ew in zip(taps, ws, ews):
            xk = win(x, a, b)
            s += wk * xk
            e_s += ew * xk.abs() + wk * win(e, a, b)
            s_mag += wk * xk.abs()
        e_s += n * U * s_mag
        num = cterm + s
        e_num = e_c + e_s + U * num.abs()
        q = num / den
        e_q = e_num / den + q.abs() * e_den / den + U * q.abs()
        xc, ec = x[I], e[I]
        y = c01 * xc + c09 * q
        e_y = c01 * ec + c09 * e_q + U * (c01 * xc.abs() + c09 * q.abs() + y.abs())
        x, e = x.clone(), e.clone()
        x[I], e[I] = y, e_y
    out = x.exp()
    return out, SAFETY * out * (e + 4 * U)


# ------------------------------------------------------------------------------------------------------------ dilate
_CROSS = ((-1, 0), (0, -1), (0, 1), (1, 0))                          # up, left, right, down: the window's row-major order


def _neighbours(x, fill):
    """(4, B, H, W): each pixel's cross neighbours, `fill` outside the map"""
    p = torch.nn.functional.pad(x[:, None], (1, 1, 1, 1), value=fill)[:, 0]
    H, W = x.shape[-2:]
    return torch.stack([p[:, 1 + di:1 + di + H, 1 + dj:1 + dj + W] for di, dj in _CROSS])


def dilate_mean(input, mask, iterations: int = 1):
    """(values fp64, mask, bound) of dilate_with_mask(input, mask, 'mean', iterations) for fp32 input (B, H, W) without NaN:
    per step, a filled pixel's mean of n <= 4 values has error (sum of their errors + (n - 1) u sum |v|) / n + u |mean|."""
    x, m = input.double(), mask.clone()
    e = torch.zeros_like(x)
    for _ in range(iterations):
        nb_m = _neighbours(m, False)
        nb_x, nb_e = _neighbours(x, 0.0), _neighbours(e, 0.0)
        cnt = nb_m.sum(0)
        vals = torch.where(nb_m, nb_x, 0.0)
        mean = vals.sum(0) / cnt
        e_mean = (torch.where(nb_m, nb_e, 0.0).sum(0) + (cnt - 1).clamp_min(0) * U * vals.abs().sum(0)) / cnt + U * mean.abs()
        x = torch.where(m, x, mean)
        e = torch.where(m, e, e_mean)
        m = nb_m.any(0) | m
    return x, m, SAFETY * e


def dilate_min_max(input, mask, filter: str, iterations: int = 1):
    """dilate_with_mask(input, mask, 'min' | 'max', iterations) on (B, H, W) fp32 as the reference's code means it: the masked
    window's amin / amax (NaN propagating), +inf / -inf where no neighbour is valid."""
    fill = float("inf") if filter == "min" else -float("inf")
    x, m = input.clone(), mask.clone()
    for _ in range(iterations):
        nb_m = _neighbours(m, False)
        v = torch.where(nb_m, _neighbours(x, 0.0), fill)
        r = v.amin(0) if filter == "min" else v.amax(0)
        x = torch.where(m, x, r)
        m = nb_m.any(0) | m
    return x, m


# ------------------------------------------------------------------------------------------------------------ blur
def gaussian_blur_2d(input, kernel_size: int, sigma: float):
    """(blurred fp64, bound) of gaussian_blur_2d(input (B, C, H, W), kernel_size, sigma) with fp64 weights.  An fp32
    implementation builds its weights as the reference does (exp of an fp32 argument with 2 roundings, a normalising sum of k
    terms and a division, an outer product): relative weight error rho = 2 (4u + 2u max|arg| + (k + 1) u) + u; its k^2-term sum
    adds k^2 u times the sum of |w x|."""
    k = kernel_size
    t = torch.arange(-k // 2 + 1, k // 2 + 1, dtype=torch.float64)
    arg = t * t / (2 * sigma ** 2)
    k1 = torch.exp(-arg)
    k1 = k1 / k1.sum()
    w = k1[:, None] * k1[None, :]
    x = torch.nn.functional.pad(input.double(), (k // 2,) * 4, mode="replicate")
    B, C, H, W = input.shape
    out = torch.zeros(B, C, H, W, dtype=torch.float64)
    mag = torch.zeros_like(out)
    for a in range(k):
        for b in range(k):
            xs = x[:, :, a:a + H, b:b + W]
            out += w[a, b] * xs
            mag += w[a, b] * xs.abs()
    rho = 2 * (4 * U + 2 * U * float(arg.max()) + (k + 1) * U) + U
    return out, SAFETY * ((rho + k * k * U) * mag + U * out.abs())


# ------------------------------------------------------------------------------------------------------------ closed forms
def closed_inputs(seed: int = 50):
    """seeded inputs of the closed forms"""
    g = torch.Generator().manual_seed(seed)
    x = 0.1 + torch.rand(3, 5, 7, generator=g)
    w = torch.rand(3, 5, 7, generator=g) > 0.3
    v1, v2 = torch.randn(4, 6, 3, generator=g), torch.randn(4, 6, 3, generator=g)
    focal = 0.5 + torch.rand(5, generator=g)
    K = torch.zeros(2, 3, 3)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 0.7 + torch.rand(2, generator=g), 0.9 + torch.rand(2, generator=g), 0.5, 0.5, 1
    from moge_b200.synthetic import synthetic_point_map
    pts, _ = synthetic_point_map(2, 24, 36, 1.2, 0.3, 0.01, "all", seed=51)
    uv = 0.5 * torch.randn(24, 36, 2, generator=g)
    return {"x": x, "w": w, "v1": v1, "v2": v2, "focal": focal, "K": K, "points": pts, "uv": uv}


def closed_calls(mod, c):
    """name -> output of every closed form of module `mod` on the inputs c"""
    out = {}
    for fn in ("weighted_mean", "harmonic_mean", "geometric_mean"):
        f = getattr(mod, fn)
        out[fn + "_all"] = f(c["x"])
        out[fn + "_dim"] = f(c["x"], dim=-1)
        out[fn + "_w_dims_keep"] = f(c["x"], c["w"], dim=(-2, -1), keepdim=True)
        out[fn + "_keep"] = f(c["x"], dim=(0, 2), keepdim=True)
    for W, H, a in ((36, 24, None), (17, 31, None), (64, 64, None), (40, 30, 2.0)):
        out[f"normalized_view_plane_uv_{W}x{H}_{a}"] = mod.normalized_view_plane_uv(W, H, aspect_ratio=a)
    out["focal_to_fov"] = mod.focal_to_fov(c["focal"])
    out["fov_to_focal"] = mod.fov_to_focal(mod.focal_to_fov(c["focal"]))
    out["angle_diff_vec3"] = mod.angle_diff_vec3(c["v1"], c["v2"])
    out["intrinsics_to_fov"] = torch.stack(mod.intrinsics_to_fov(c["K"]))
    out["point_map_to_depth_legacy"] = mod.point_map_to_depth_legacy(c["points"])
    out["view_plane_uv_to_focal"] = mod.view_plane_uv_to_focal(c["uv"])
    return out


def public_signatures(module):
    """name -> [(parameter, repr of its default or None)] of the public functions defined in `module` (not those it imports)"""
    out = {}
    for name, f in vars(module).items():
        if not name.startswith("_") and inspect.isfunction(f) and f.__module__ == module.__name__:
            out[name] = [(p.name, None if p.default is inspect.Parameter.empty else repr(p.default))
                         for p in inspect.signature(f).parameters.values()]
    return out
