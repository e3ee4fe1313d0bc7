"""Panorama mesh export on the GPU against the numpy restatement in oracle/utils3d_normals.py: point_map_to_normal_map bitwise over
shapes, masks, batches and inf / NaN points; normal_map_edge bracketed between the restatement at tol (1 + 1e-6) and tol (1 - 1e-6)
(the kernel's acosf and numpy's arccos may each be 2 ulp off); mesh_from_panorama on an analytic room and on infer_panorama()
output; the single-image cleaning step composed from the public functions; one host wait, inputs unmodified, repeatable."""
import numpy as np
import pytest
import torch

from moge_b200 import capi
from moge_b200 import mesh as M
from moge_b200.synthetic import synthetic_panorama_scene
from oracle import utils3d_mesh as OM
from oracle import utils3d_normals as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
REL = 1e-6
ULP = 4                      # kernel vs numpy angle, where both are finite: 2 ulp each from the correctly rounded arccos


def _bytes_equal(got: torch.Tensor, want: np.ndarray) -> bool:
    """Bitwise, except that a NaN's sign and payload are not compared (x86 makes -NaN from inf - inf, the GPU its canonical NaN)."""
    if got.dtype != torch.float32 or tuple(got.shape) != want.shape:
        return False
    g = got.cpu().numpy()
    nan = np.isnan(want)
    return np.array_equal(np.isnan(g), nan) and g[~nan].tobytes() == want[~nan].tobytes()


def _points(H, W, seed, special=True):
    """Random points with ~1 % inf and ~1 % NaN coordinates, and a ~80 % mask."""
    g = np.random.default_rng(seed)
    p = g.normal(size=(H, W, 3)).astype(np.float32)
    if special:
        p[g.random((H, W, 3)) < 0.01] = np.inf
        p[g.random((H, W, 3)) < 0.01] = np.nan
    return p, g.random((H, W)) < 0.8


@pytest.mark.parametrize("H,W", [(1, 1), (1, 57), (43, 1), (37, 53), (1024, 2048)])
@pytest.mark.parametrize("masked", [False, True])
def test_point_map_to_normal_map_bitwise(H, W, masked):
    cases = [_points(H, W, H * W)]
    if H * W > 1_000_000:
        p, _, m, _ = synthetic_panorama_scene(H, W, 0)
        cases.append((p, m))
    for p, m in cases:
        dp = torch.from_numpy(p).to(DEV)
        if masked:
            dm = torch.from_numpy(m).to(DEV)
            n, nm = M.point_map_to_normal_map(dp, dm)
            wn, wm = O.point_map_to_normal_map(p, m)
            assert nm.dtype == torch.bool and np.array_equal(nm.cpu().numpy(), wm)
        else:
            n, wn = M.point_map_to_normal_map(dp), O.point_map_to_normal_map(p)
        assert _bytes_equal(n, wn), int((n.cpu().numpy() != wn).sum())
        assert torch.equal(dp.cpu().nan_to_num(), torch.from_numpy(p).nan_to_num())          # the input is not modified


def test_point_map_to_normal_map_batch():
    p = np.stack([_points(37, 53, 90 + b)[0] for b in range(3)])
    m = np.stack([_points(37, 53, 90 + b)[1] for b in range(3)])
    n, nm = M.point_map_to_normal_map(torch.from_numpy(p).to(DEV)[None], torch.from_numpy(m).to(DEV)[None])
    assert n.shape == (1, 3, 37, 53, 3) and nm.shape == (1, 3, 37, 53)
    for b in range(3):
        wn, wm = O.point_map_to_normal_map(p[b], m[b])
        assert _bytes_equal(n[0, b], wn) and np.array_equal(nm[0, b].cpu().numpy(), wm)
    assert _bytes_equal(M.point_map_to_normal_map(torch.from_numpy(p).to(DEV)), O.point_map_to_normal_map(p))


def _angle(normals: torch.Tensor, mask, k):
    """The kernel's pooled angle map (the ABI's diagnostic output)."""
    H, W = normals.shape[:2]
    n = normals.contiguous()[None]
    m = None if mask is None else mask.contiguous().view(torch.uint8)[None]
    angle = torch.empty(1, H, W, dtype=torch.float32, device=DEV)
    M._normal_edge(n, m, None, None, 5.0, k, angle)
    return angle[0]


def _ulps(a: np.ndarray, b: np.ndarray) -> int:
    fin = np.isfinite(a) & np.isfinite(b)
    if not fin.any():
        return 0
    ia, ib = a[fin].view(np.int32).astype(np.int64), b[fin].view(np.int32).astype(np.int64)
    return int(np.abs(ia - ib).max())


def check_bracket(got: np.ndarray, lo: np.ndarray, hi: np.ndarray, what: str) -> int:
    """lo ⊆ got ⊆ hi: the kernel's map lies between the restatement at the two bracketing tolerances."""
    assert not (lo & ~got).any() and not (got & ~hi).any(), what
    n = int((lo != hi).sum())
    print(f"{what}: {n} bracket pixels, {int(got.sum())} set")
    return n


def _scene_normals(H, W, seed=0):
    p, _, m, _ = synthetic_panorama_scene(H, W, seed)
    return O.point_map_to_normal_map(p, m)


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("masked", [False, True])
def test_normal_map_edge_bracketed(k, masked):
    n, nm = _scene_normals(512, 1024)
    r, _ = _points(61, 77, k)
    rm = np.random.default_rng(k).random((61, 77)) < 0.8
    for normals, mask, name in ((n, nm, "room 512x1024"), (r, rm, "random 61x77")):
        dn, dm = torch.from_numpy(normals).to(DEV), torch.from_numpy(mask).to(DEV)
        m_np, m_dev = (mask, dm) if masked else (None, None)
        got = M.normal_map_edge(dn, tol=5, kernel_size=k, mask=m_dev).cpu().numpy()
        lo = O.normal_map_edge(normals, 5 * (1 + REL), k, m_np)
        hi = O.normal_map_edge(normals, 5 * (1 - REL), k, m_np)
        check_bracket(got, lo, hi, f"{name} k={k} masked={masked}")
        a, wa = _angle(dn, m_dev, k).cpu().numpy(), O.normal_angle_map(normals, k, m_np)
        assert np.array_equal(np.isnan(a), np.isnan(wa)) and np.array_equal(np.isinf(a), np.isinf(wa))
        ulps = _ulps(a, wa)
        print(f"{name} k={k} masked={masked}: NaN angles {int(np.isnan(a).sum())}, max |angle - numpy| {ulps} ulp")
        assert ulps <= ULP
        if name.startswith("room"):
            assert np.isnan(wa).any() and lo.any()                 # the contract's NaN and edge paths are exercised
        assert torch.equal(dn.cpu().nan_to_num(), torch.from_numpy(normals).nan_to_num())


def _cleaned_bracket(points, depth, mask, threshold=0.03):
    """The restatement's cleaned mask at 5 (1 + 1e-6) and 5 (1 - 1e-6) degrees: (smallest, largest)."""
    normals, nm = O.point_map_to_normal_map(points, mask)
    de = OM.depth_map_edge(depth, rtol=threshold)
    angle = O.normal_angle_map(normals, 3, nm)
    with np.errstate(invalid="ignore"):
        lo = mask & ~(de & (angle > np.deg2rad(5 * (1 - REL))))
        hi = mask & ~(de & (angle > np.deg2rad(5 * (1 + REL))))
    return lo, hi


def check_panorama_mesh(res, points, depth, mask, image, what, threshold=0.03):
    cleaned = res["mask_cleaned"].cpu().numpy()
    lo, hi = _cleaned_bracket(points, depth, mask, threshold)
    n = check_bracket(cleaned, lo, hi, what)
    print(f"{what}: {int((mask & ~cleaned).sum())} pixels cleaned, {res['faces'].shape[0]} faces")
    want = OM.build_mesh_from_map(points, image.astype(np.float32) / 255, OM.uv_map(*depth.shape), mask=cleaned, tri=True)
    assert res["faces"].dtype == torch.int32 and np.array_equal(res["faces"].cpu().numpy(), want[0])
    for k, w in zip(("vertices", "vertex_colors", "vertex_uvs"), want[1:]):
        assert _bytes_equal(res[k], w), k
    if n == 0:                        # no pixel near the threshold: the whole result is the restatement's
        full = O.mesh_from_panorama(points, depth, mask, image, threshold)
        assert np.array_equal(cleaned, full["mask_cleaned"]) and np.array_equal(res["faces"].cpu().numpy(), full["faces"])


def test_mesh_from_panorama_analytic_room():
    points, depth, mask, image = synthetic_panorama_scene(1024, 2048, 3)
    out = {"points": torch.from_numpy(points).to(DEV), "depth": torch.from_numpy(depth).to(DEV), "mask": torch.from_numpy(mask).to(DEV)}
    res = M.mesh_from_panorama(out, torch.from_numpy(image).to(DEV))
    assert set(res) == {"faces", "vertices", "vertex_colors", "vertex_uvs", "mask_cleaned"}
    assert (mask & ~res["mask_cleaned"].cpu().numpy()).any() and res["faces"].shape[0] > 3_000_000
    check_panorama_mesh(res, points, depth, mask, image, "room 2048x1024")
    free = M.mesh_from_panorama(out, torch.from_numpy(image).to(DEV), threshold=float("inf"))
    assert np.array_equal(free["mask_cleaned"].cpu().numpy(), mask)
    check_panorama_mesh(free, points, depth, mask, image, "room 2048x1024 threshold inf", threshold=np.inf)


def _v1_model():
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vits")
    m = MoGeModel(**cfg)
    m.load_state_dict(make_v1_state_dict(cfg, 7, well_posed=True))
    return m.to(DEV).eval()


def test_mesh_from_panorama_infer_panorama_v1():
    from moge_b200.panorama import infer_panorama
    from moge_b200.synthetic import synthetic_panorama
    image = synthetic_panorama(256, 512, 3)
    dimg = torch.from_numpy(image).to(DEV)
    out = infer_panorama(_v1_model(), dimg)
    res = M.mesh_from_panorama(out, dimg)
    host = {k: v.cpu().numpy() for k, v in out.items()}
    assert res["faces"].shape[0] > 0
    check_panorama_mesh(res, host["points"], host["depth"], host["mask"], image, "infer_panorama MoGe-1 ViT-S 512x256")


def test_single_image_cleaning_composed_from_public_functions():
    """infer_baseline.py:120-127 on a MoGe-2 infer() output: mask & ~(depth_map_edge(depth, rtol, mask=mask) & normal_map_edge(
    normals, tol=5, mask=normals_mask)) with (normals, normals_mask) = point_map_to_normal_map(points, mask)."""
    from moge.model.v2 import MoGeModel
    from moge_b200.configs import model_config
    from moge_b200.synthetic import make_state_dict, synthetic_images
    cfg = model_config("vits", True)
    model = MoGeModel(**cfg)
    model.load_state_dict(make_state_dict(cfg, 0, well_posed=True))
    model = model.to(DEV).eval()
    img = synthetic_images(1, 196, 252, 0)[0]
    out = model.infer(img.to(DEV), num_tokens=300)
    points, depth, mask = out["points"], out["depth"], out["mask"]
    normals, nmask = M.point_map_to_normal_map(points, mask=mask)
    for threshold in (0.03, 0.3):
        keep = mask & ~(M.depth_map_edge(depth, rtol=threshold, mask=mask) & M.normal_map_edge(normals, tol=5, mask=nmask))
        p, d, m = points.cpu().numpy(), depth.cpu().numpy(), mask.cpu().numpy()
        wn, wm = O.point_map_to_normal_map(p, m)
        assert _bytes_equal(normals, wn) and np.array_equal(nmask.cpu().numpy(), wm)
        de = OM.depth_map_edge(d, rtol=threshold, mask=m)
        angle = O.normal_angle_map(wn, 3, wm)
        with np.errstate(invalid="ignore"):
            lo = m & ~(de & (angle > np.deg2rad(5 * (1 - REL))))
            hi = m & ~(de & (angle > np.deg2rad(5 * (1 + REL))))
        got = keep.cpu().numpy()
        check_bracket(got, lo, hi, f"MoGe-2 cleaning rtol={threshold}")
        print(f"MoGe-2 cleaning rtol={threshold}: {int((m & ~got).sum())} of {int(m.sum())} pixels cleaned")


def test_one_host_wait_inputs_unmodified_and_repeatable(monkeypatch):
    points, depth, mask, image = synthetic_panorama_scene(300, 600, 9)
    out = {"points": torch.from_numpy(points).to(DEV), "depth": torch.from_numpy(depth).to(DEV), "mask": torch.from_numpy(mask).to(DEV)}
    dimg = torch.from_numpy(image).to(DEV)
    first = M.mesh_from_panorama(out, dimg)                    # warm-up: library load, allocator
    torch.cuda.synchronize()
    waits = []
    original = torch.cuda.Event.synchronize

    def counted(self):
        waits.append(1)
        torch.cuda.set_sync_debug_mode(0)
        try:
            original(self)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(torch.cuda.Event, "synchronize", counted)
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = M.mesh_from_panorama(out, dimg)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(waits) == 1
    for k in first:
        assert again[k].cpu().numpy().tobytes() == first[k].cpu().numpy().tobytes(), k
    for k, v in (("points", points), ("depth", depth), ("mask", mask)):
        assert np.array_equal(out[k].cpu().numpy(), v), k
    assert np.array_equal(dimg.cpu().numpy(), image)
