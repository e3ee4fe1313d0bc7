"""Generate tests/golden/geometry.pt from the UNMODIFIED reference `moge/utils/geometry_torch.py` (CPU, fp32).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_geometry_golden.py

utils3d resolves to the stand-in under oracle/utils3d_shim, with `sliding_window`, `sliding_window_2d` and `uv_map` from
oracle/utils3d_geometry.py.  Inputs come from the seeded generators in moge_b200.synthetic, so the file stores each case's recipe
and the SHA-256 of its inputs rather than the inputs, and the reference's outputs:
- refine: refine_depth_with_normal at square, 2:1, 1:2 and odd sizes, with batch dimensions, kernel sizes 3 to 9, no sweep, a
  map with one interior row and one a stencil radius wider than its border on each side;
- dilate: dilate_with_mask with each filter at 1 and 3 iterations, over all-valid, sparse, scene and empty masks.  The
  reference's 'min' and 'max' branches raise TypeError (Tensor.min / max with a tuple of dims); the maker checks that they do
  and takes those cases from oracle/geometry_port.dilate_min_max, the masked window min / max that the code means;
- threshold: theshold_depth_change with both poolers, kernel sizes 1 to 7 and two tolerances;
- blur: gaussian_blur_2d of one-channel maps (the reference's (1, 1, k, k) weight with groups = C only runs for C = 1);
- focal_shift: recover_focal_shift (SciPy on the host) with all, random, single-pixel and empty masks, a known focal, and
  batch dimensions;
- closed: the closed-form functions on seeded inputs;
- signatures: the parameter names and defaults of every public function of the module.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")

import importlib.util  # noqa: E402

import torch  # noqa: E402

from moge_b200.synthetic import array_digest, synthetic_geometry_case, synthetic_point_map  # noqa: E402
from oracle import geometry_port, utils3d_geometry  # noqa: E402
from oracle.geometry_port import closed_calls, closed_inputs  # noqa: E402

utils3d_geometry.install()
_REF = os.path.join(os.environ["MOGE_REFERENCE"], "moge")


def _load_reference():
    """the real reference module, loaded from its file as `reference_moge_golden.utils.geometry_torch` so that its relative
    imports (.tools, .geometry_numpy) resolve to the reference's own files"""
    import types
    pkg = types.ModuleType("reference_moge_golden")
    pkg.__path__ = [_REF]
    sys.modules["reference_moge_golden"] = pkg
    sub = types.ModuleType("reference_moge_golden.utils")
    sub.__path__ = [os.path.join(_REF, "utils")]
    sys.modules["reference_moge_golden.utils"] = sub
    spec = importlib.util.spec_from_file_location("reference_moge_golden.utils.geometry_torch", os.path.join(_REF, "utils", "geometry_torch.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


ref = _load_reference()
OUT = os.path.join(ROOT, "tests", "golden", "geometry.pt")

# (seed, batch_shape, H, W, kernel_size, iterations)
REFINE = [
    (0, (), 48, 48, 5, 10),
    (1, (2,), 40, 80, 5, 10),
    (2, (), 80, 40, 5, 10),
    (3, (2, 2), 37, 53, 3, 4),
    (4, (), 45, 61, 7, 10),
    (5, (), 41, 39, 9, 6),
    (6, (), 5, 30, 5, 10),          # a single interior row (the border is 2 pixels wide)
    (7, (), 7, 30, 5, 10),          # one stencil radius wider than the border on each side: 3 interior rows
    (8, (2,), 33, 35, 5, 0),        # no sweep
]
# (seed, batch_shape, H, W, mask_mode)
DILATE_MAPS = [(10, (2,), 33, 47, "sparse"), (11, (), 64, 32, "scene"), (12, (), 17, 19, "all"), (13, (), 16, 16, "none")]
FILTERS, DILATE_ITERS = ("mean", "min", "max", "median"), (1, 3)
# (seed, batch_shape, H, W, mask_mode, pooler, rtol, kernel_size)
THRESHOLD = [
    (20, (2,), 33, 47, "scene", "max", 0.2, 3),
    (20, (2,), 33, 47, "scene", "min", 0.2, 3),
    (21, (), 64, 32, "sparse", "max", 0.05, 5),
    (21, (), 64, 32, "sparse", "min", 0.05, 5),
    (22, (), 31, 29, "all", "min", 0.2, 7),
    (23, (), 16, 16, "none", "max", 0.2, 1),
]
# (seed, batch, H, W, kernel_size, sigma)
BLUR = [(30, 2, 33, 47, 5, 1.0), (31, 1, 40, 24, 3, 0.5), (32, 3, 21, 19, 9, 2.0)]
# (args of synthetic_point_map, batch_shape, with focal)
FOCAL = [
    ((1, 96, 128, 1.25, 0.4, 0.0, "all", 40), (), False),
    ((2, 75, 133, 0.9, -0.2, 0.01, "random", 41), (2,), False),
    ((2, 64, 64, 1.1, 0.3, 0.0, "half", 42), (2,), True),
    ((1, 80, 60, 1.0, 0.0, 0.0, "single", 43), (), False),
    ((1, 80, 60, 1.0, 0.0, 0.0, "none", 44), (), True),
    ((4, 50, 70, 1.3, 0.1, 0.0, "random", 45), (2, 2), False),
]


def geometry_inputs(seed, batch_shape, H, W, mask_mode="sparse"):
    c = synthetic_geometry_case(seed, batch_shape, H, W, mask_mode)
    return c, array_digest(*[c[k].numpy() for k in ("depth", "normal", "intrinsics", "mask", "image")])


def refine_cases():
    out = []
    for seed, bs, H, W, k, it in REFINE:
        c, digest = geometry_inputs(seed, bs, H, W)
        depth = c["depth"].clone()
        res = ref.refine_depth_with_normal(depth, c["normal"], c["intrinsics"], iterations=it, kernel_size=k)
        out.append({"seed": seed, "batch_shape": bs, "H": H, "W": W, "kernel_size": k, "iterations": it, "inputs_sha256": digest,
                    "depth": res})
        print(f"refine {bs} {H}x{W} k={k} it={it}: max |log change| {float((res.log() - c['depth'].log()).abs().max()):.3e}")
    return out


def dilate_cases():
    out = []
    for seed, bs, H, W, mode in DILATE_MAPS:
        c, digest = geometry_inputs(seed, bs, H, W, mode)
        for filt in FILTERS:
            for it in DILATE_ITERS:
                if filt in ("min", "max"):
                    try:
                        ref.dilate_with_mask(c["depth"], c["mask"], filt, it)
                        raise AssertionError("the reference's dilate_with_mask(filter=%r) ran" % filt)
                    except TypeError:
                        pass
                    x, m = geometry_port.dilate_min_max(c["depth"].reshape(-1, H, W), c["mask"].reshape(-1, H, W), filt, it)
                    x, m = x.reshape(c["depth"].shape), m.reshape(c["mask"].shape)
                    source = "geometry_port.dilate_min_max"
                else:
                    x, m = ref.dilate_with_mask(c["depth"], c["mask"], filt, it)
                    source = "reference"
                out.append({"seed": seed, "batch_shape": bs, "H": H, "W": W, "mask_mode": mode, "filter": filt, "iterations": it,
                            "inputs_sha256": digest, "input": x, "mask": m, "source": source})
        print(f"dilate {bs} {H}x{W} {mode}")
    return out


def threshold_cases():
    out = []
    for seed, bs, H, W, mode, pooler, rtol, k in THRESHOLD:
        c, digest = geometry_inputs(seed, bs, H, W, mode)
        res = ref.theshold_depth_change(c["depth"], c["mask"], pooler, rtol=rtol, kernel_size=k)
        out.append({"seed": seed, "batch_shape": bs, "H": H, "W": W, "mask_mode": mode, "pooler": pooler, "rtol": rtol,
                    "kernel_size": k, "inputs_sha256": digest, "output": res})
        print(f"threshold {bs} {H}x{W} {mode} {pooler} k={k}: {int(res.sum())} set")
    return out


def blur_cases():
    out = []
    for seed, B, H, W, k, sigma in BLUR:
        c, digest = geometry_inputs(seed, (B,), H, W)
        res = ref.gaussian_blur_2d(c["image"][:, :1].contiguous(), k, sigma)
        out.append({"seed": seed, "B": B, "H": H, "W": W, "kernel_size": k, "sigma": sigma, "inputs_sha256": digest, "output": res})
    return out


def focal_cases():
    out = []
    for args, bs, with_focal in FOCAL:
        pts, mask = synthetic_point_map(*args[:7], seed=args[7])
        H, W = pts.shape[1:3]
        pts, mask = pts.reshape(*bs, H, W, 3), mask.reshape(*bs, H, W)
        focal = torch.linspace(0.8, 1.4, pts[..., 0, 0, 0].numel()).reshape(bs) if with_focal else None
        f, s = ref.recover_focal_shift(pts, mask, focal=focal)
        out.append({"args": args, "batch_shape": bs, "focal_in": focal, "inputs_sha256": array_digest(pts.numpy(), mask.numpy()),
                    "focal": f, "shift": s})
        print(f"focal_shift {args[6]} {bs}: focal {f.flatten().tolist()} shift {s.flatten().tolist()}")
    return out


def reference_signatures():
    """name -> [(parameter, repr of its default or None)] of every public function the reference module defines"""
    return geometry_port.public_signatures(ref)


def main():
    c = closed_inputs()
    gold = {"refine": refine_cases(), "dilate": dilate_cases(), "threshold": threshold_cases(), "blur": blur_cases(),
            "focal_shift": focal_cases(),
            "signatures": reference_signatures(),
            "closed": {"seed": 50, "inputs_sha256": array_digest(*[v.numpy() for v in c.values()]), "outputs": closed_calls(ref, c)}}
    torch.save(gold, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
