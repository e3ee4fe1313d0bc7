"""Mixed-size panorama inference on the GPU: infer_panoramas_many against each member's own infer_panorama (bitwise: depth,
mask, points, the views and the per-level LSMR iterations and istop), in permuted order, with view batches that straddle
panoramas, against infer_panoramas on a one-size list; the golden room's merges solved in one mixed call beside systems of other
sizes against tests/golden/panorama.pt; a mixed merge without host waits; and inputs left unmodified."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "panorama.pt")
# the thresholds of test_gpu_panorama.py and test_gpu_panorama_batch.py
ITN_BAND = 0.01
SENS_MULT = 10.0

# (H, W, seed): above the 1920 x 960 merge cap, an odd width and height, a non-2:1 aspect, two of one size, and a panorama
# whose merge is a single level (under 256 px)
SIZES = [(1024, 2048, 1), (128, 256, 2), (97, 257, 3), (96, 320, 4), (128, 256, 5), (64, 128, 6)]


@pytest.fixture(scope="module")
def model():
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vits")
    m = MoGeModel(**cfg)
    m.load_state_dict(make_v1_state_dict(cfg, 7, well_posed=True))
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def images():
    from moge_b200.synthetic import synthetic_panorama
    return [torch.from_numpy(synthetic_panorama(H, W, s)).to(DEV) for H, W, s in SIZES]


@pytest.fixture(scope="module")
def singles(model, images):
    from moge_b200.panorama import infer_panorama, last_merge_stats
    out = []
    for image in images:
        res = infer_panorama(model, image, return_views=True)
        out.append((res, last_merge_stats()))
    return out


def _assert_member(got, want, tag):
    assert set(got) == set(want), (tag, set(got), set(want))
    for key, w in want.items():
        assert got[key].shape == w.shape and torch.equal(got[key], w), (tag, key)


def test_many_equals_single(model, images, singles):
    from moge_b200.panorama import infer_panoramas_many, last_merge_stats
    before = [im.clone() for im in images]
    out = infer_panoramas_many(model, images, return_views=True)
    stats = last_merge_stats()
    assert len(out) == len(images) and len(stats) == len(images)
    for k, ((res, st), got) in enumerate(zip(singles, out)):
        _assert_member(got, res, k)
        assert stats[k] == st, (k, stats[k], st)
        print(f"{SIZES[k][:2]}: levels {[(s['width'], s['height']) for s in st]}, iterations {[s['iterations'] for s in st]}")
    assert len(stats[0]) == 4 and len(stats[-1]) == 1                      # pyramids of different depths in one call
    plain = infer_panoramas_many(model, images)
    for k, ((res, _), got) in enumerate(zip(singles, plain)):
        assert set(got) == {"depth", "mask", "points"}
        assert all(torch.equal(got[key], res[key]) for key in got), k
    assert all(torch.equal(a, b) for a, b in zip(images, before))


def test_many_permuted(model, images, singles):
    from moge_b200.panorama import infer_panoramas_many, last_merge_stats
    order = [3, 0, 5, 2, 4, 1]
    out = infer_panoramas_many(model, [images[k] for k in order], return_views=True)
    stats = last_merge_stats()
    for pos, k in enumerate(order):
        _assert_member(out[pos], singles[k][0], (pos, k))
        assert stats[pos] == singles[k][1]


@pytest.mark.parametrize("batch_size", [7, 30])
def test_many_straddling_view_batches(model, images, singles, batch_size):
    from moge_b200.panorama import infer_panoramas_many
    out = infer_panoramas_many(model, images, batch_size=batch_size, return_views=True)
    for k, ((res, _), got) in enumerate(zip(singles, out)):
        _assert_member(got, res, (batch_size, k))


def test_many_one_size_equals_batch(model, images):
    from moge_b200.panorama import infer_panoramas, infer_panoramas_many, last_merge_stats
    same = [images[1], images[4], images[1]]
    out = infer_panoramas_many(model, same, return_views=True)
    many_stats = last_merge_stats()
    batch = infer_panoramas(model, torch.stack(same), return_views=True)
    assert last_merge_stats() == many_stats
    for k, got in enumerate(out):
        _assert_member(got, {key: v[k] for key, v in batch.items()}, k)


def test_many_wrong_device_before_device_work(images):
    from moge_b200.capi import MogeError
    from moge_b200.panorama import infer_panoramas_many

    class Elsewhere:
        device = torch.device("cuda", 1)

        def infer(self, *args, **kwargs):
            raise AssertionError("argument errors must be raised before the view pass")
    with pytest.raises(MogeError, match=r"panorama 0 is on cuda:0, not on cuda:1"):
        infer_panoramas_many(Elsewhere(), images[:2])
    Elsewhere.device = None                                  # no device to match: the first panorama's is the one
    with pytest.raises(MogeError, match=r"panorama 1: a 1 x 128 map"):
        infer_panoramas_many(Elsewhere(), [images[0], images[0][:1, :128]])


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN, weights_only=False)


def _cams(g):
    return g["extrinsics"].numpy(), list(g["intrinsics"].numpy())


def _unpack(bits, h, w):
    return torch.from_numpy(np.unpackbits(bits.numpy())[:h * w].reshape(h, w).astype(bool))


@pytest.fixture(scope="module")
def room(gold):
    from moge_b200.synthetic import array_digest, synthetic_room_views
    dist, masks = synthetic_room_views(gold["room"]["resolution"], gold["room"]["seed"])
    assert array_digest(dist, masks) == gold["room"]["inputs_sha256"]
    noisy = (dist * np.exp(0.03 * np.random.RandomState(5).standard_normal(dist.shape))).astype(np.float32)
    return [(torch.from_numpy(d).to(DEV), torch.from_numpy(masks).to(DEV)) for d in (dist, noisy)]


def test_mixed_merge_against_reference(gold, room):
    """Every golden merge case of the room in one mixed merge, beside a noisy room at 1000 x 500 and at 256 x 128."""
    from moge_b200.panorama import _merge, last_merge_stats
    extr, intr = _cams(gold)
    cases = gold["merge"]
    sizes = [(c["width"], c["height"]) for c in cases] + [(1000, 500), (256, 128)]
    members = [room[0]] * len(cases) + [room[1], room[1]]
    src = torch.stack([d for d, _ in members])
    msk = torch.stack([m for _, m in members])
    depth, mask, launches = _merge("test", sizes, src, msk, extr, intr, True)
    stats = last_merge_stats()
    assert len(launches) == 3 and len(launches[-1]["members"]) == len(sizes)
    offsets = np.cumsum([0] + [w * h for w, h in sizes])
    for i, case in enumerate(cases):
        per_level = []                                       # this member's (b, row_mask) per level, coarsest first
        for lv in launches:
            pos = [m for m, _ in lv["members"]].index(i) if i in [m for m, _ in lv["members"]] else None
            if pos is None:
                continue
            rows = [2 * h * w + (h - 1) * (w + 1) for w, h in lv["sizes"]]
            r0 = sum(rows[:pos])
            per_level.append((lv["b"][r0:r0 + rows[pos]], lv["row_mask"][r0:r0 + rows[pos]]))
        assert len(per_level) == len(case["levels"]) == len(stats[i])
        for (b, rm), g, st in zip(per_level, case["levels"], stats[i]):
            rm = rm.cpu().numpy().astype(bool)
            np.testing.assert_array_equal(rm, np.unpackbits(g["row_mask"].numpy())[:g["rows"]].astype(bool))
            if "b" in g:
                assert np.abs(b.cpu().numpy()[rm] - g["b"].numpy().astype(np.float64)).max() <= 2e-6
            assert st["istop"] == g["istop"]
            assert abs(st["iterations"] - g["itn"]) <= max(2, ITN_BAND * g["itn"])
        w, h = sizes[i]
        d = depth[offsets[i]:offsets[i + 1]].view(h, w)
        s = case["depth_stride"]
        rel = (d.cpu()[::s, ::s].double() / case["depth"].double() - 1).abs().max().item()
        print(f"mixed {w}x{h}: depth rel err {rel:.2e}, reference sensitivity {case['sensitivity']:.2e}")
        assert rel <= SENS_MULT * max(case["sensitivity"], 1e-6)
        assert torch.equal(mask[offsets[i]:offsets[i + 1]].view(h, w).cpu(), _unpack(case["mask"], h, w))


def test_mixed_merge_no_host_wait_inputs_kept(gold, room):
    from moge_b200.panorama import _merge
    extr, intr = _cams(gold)
    sizes = [(600, 300), (200, 100), (1000, 500)]
    src = torch.stack([room[0][0], room[1][0], room[0][0]])
    msk = torch.stack([room[0][1], room[1][1], room[1][1]])
    s0, m0 = src.clone(), msk.clone()
    a = _merge("test", sizes, src, msk, extr, intr, False)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = _merge("test", sizes, src, msk, extr, intr, False)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(src, s0) and torch.equal(msk, m0)
