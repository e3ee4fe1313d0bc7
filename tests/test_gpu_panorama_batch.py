"""Batched panorama inference on the GPU: split_panoramas, merge_panoramas and infer_panoramas against the single-panorama calls
on each member (bitwise: depth, mask, per-level LSMR iterations and istop, and the per-level tensors), the batched merge of the
golden room against tests/golden/panorama.pt, and a batched merge without host waits."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "panorama.pt")
# the thresholds of test_gpu_panorama.py
ITN_BAND = 0.01
SENS_MULT = 10.0


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN, weights_only=False)


def _cams(g):
    return g["extrinsics"].numpy(), list(g["intrinsics"].numpy())


def _unpack(bits, h, w):
    return torch.from_numpy(np.unpackbits(bits.numpy())[:h * w].reshape(h, w).astype(bool))


@pytest.fixture(scope="module")
def members(gold):
    """Five merge inputs: the golden room, an all-empty-mask copy and three copies with seeded multiplicative noise on the
    distances of different strengths, so that the members' solves stop at different iteration counts."""
    from moge_b200.synthetic import array_digest, synthetic_room_views
    dist, masks = synthetic_room_views(gold["room"]["resolution"], gold["room"]["seed"])
    assert array_digest(dist, masks) == gold["room"]["inputs_sha256"]
    rng = np.random.RandomState(11)
    out = [(dist, masks)]
    for k, amp in enumerate((0.03, 0.0, 0.1, 0.01)):
        if k == 1:
            out.append((dist, np.zeros_like(masks)))
            continue
        noisy = (dist * np.exp(amp * rng.standard_normal(dist.shape))).astype(np.float32)
        out.append((noisy, masks))
    return [(torch.from_numpy(d).to(DEV), torch.from_numpy(m).to(DEV)) for d, m in out]


def test_split_panoramas_bitwise(gold):
    from moge_b200.panorama import split_panorama, split_panoramas
    from moge_b200.synthetic import synthetic_panorama
    extr, intr = _cams(gold)
    case = gold["split"][0]
    H, W, res = case["H"], case["W"], case["resolution"]
    imgs = torch.from_numpy(np.stack([synthetic_panorama(H, W, s) for s in (case["seed"], 17, 29)])).to(DEV)
    before = imgs.clone()
    f32, u8 = split_panoramas(imgs, extr, intr, res, return_uint8=True)
    assert f32.shape == (3, 12, 3, res, res) and u8.shape == (3, 12, res, res, 3)
    for k in range(3):
        sf, su = split_panorama(imgs[k], extr, intr, res, return_uint8=True)
        assert torch.equal(f32[k], sf) and torch.equal(u8[k], su)
    if "views" in case:
        assert torch.equal(u8[0].cpu(), case["views"])
    assert torch.equal(imgs, before)
    assert torch.equal(split_panoramas(imgs, extr, intr, res), f32)


def _single(gold, case, src, mask):
    from moge_b200.panorama import last_merge_stats, merge_panorama
    extr, intr = _cams(gold)
    depth, pm, levels = merge_panorama(case["width"], case["height"], src, mask, extr, intr, return_levels=True)
    return depth, pm, levels, last_merge_stats()


@pytest.mark.parametrize("P", [1, 2, 5])
@pytest.mark.parametrize("ci", [0, 1, 2])
def test_merge_panoramas_equals_single(gold, members, P, ci):
    from moge_b200.panorama import last_merge_stats, merge_panoramas
    case = gold["merge"][ci]
    extr, intr = _cams(gold)
    chosen = members[:P]
    src = torch.stack([d for d, _ in chosen])
    msk = torch.stack([m for _, m in chosen])
    depth, pm, levels = merge_panoramas(case["width"], case["height"], src, msk, extr, intr, return_levels=True)
    stats = last_merge_stats()
    assert depth.shape == (P, case["height"], case["width"]) and pm.shape == depth.shape and len(stats) == P
    iterations = []
    for k, (d, m) in enumerate(chosen):
        sd, sm, slv, sst = _single(gold, case, d, m)
        assert torch.equal(depth[k], sd), (k, (depth[k] != sd).sum().item())
        assert torch.equal(pm[k], sm)
        assert stats[k] == sst, (k, stats[k], sst)
        for lv, s in zip(levels, slv):
            assert (lv["width"], lv["height"]) == (s["width"], s["height"])
            for key in ("b", "row_mask", "depth"):
                assert torch.equal(lv[key][k], s[key]), (k, key, lv["width"])
        iterations.append(tuple(st["iterations"] for st in sst))
        print(f"{case['width']}x{case['height']} P={P} member {k}: iterations {iterations[-1]}, "
              f"istop {[st['istop'] for st in sst]}")
    if P >= 2:
        assert len(set(iterations)) >= min(P, 4), iterations          # the members stop at different iteration counts
    if P >= 3:
        assert all(st["iterations"] == 0 for st in stats[2]) and not pm[2].any()     # the empty member stops at once


def test_merge_panoramas_against_reference(gold, members):
    from moge_b200.panorama import last_merge_stats, merge_panoramas
    extr, intr = _cams(gold)
    src = torch.stack([members[0][0], members[3][0]])
    msk = torch.stack([members[0][1], members[3][1]])
    for case in gold["merge"]:
        depth, mask, levels = merge_panoramas(case["width"], case["height"], src, msk, extr, intr, return_levels=True)
        stats = last_merge_stats()[0]
        for lv, g, st in zip(levels, case["levels"], stats):
            rm = lv["row_mask"][0].cpu().numpy().astype(bool)
            np.testing.assert_array_equal(rm, np.unpackbits(g["row_mask"].numpy())[:g["rows"]].astype(bool))
            if "b" in g:
                assert np.abs(lv["b"][0].cpu().numpy()[rm] - g["b"].numpy().astype(np.float64)).max() <= 2e-6
            assert st["istop"] == g["istop"]
            assert abs(st["iterations"] - g["itn"]) <= max(2, ITN_BAND * g["itn"])
        s = case["depth_stride"]
        rel = (depth[0].cpu()[::s, ::s].double() / case["depth"].double() - 1).abs().max().item()
        print(f"batched {case['width']}x{case['height']}: depth rel err {rel:.2e}, reference sensitivity {case['sensitivity']:.2e}")
        assert rel <= SENS_MULT * max(case["sensitivity"], 1e-6)
        assert torch.equal(mask[0].cpu(), _unpack(case["mask"], case["height"], case["width"]))


def test_merge_panoramas_no_host_wait_inputs_kept(gold, members):
    from moge_b200.panorama import merge_panoramas
    case = gold["merge"][1]
    extr, intr = _cams(gold)
    src = torch.stack([d for d, _ in members[:3]])
    msk = torch.stack([m for _, m in members[:3]])
    s0, m0 = src.clone(), msk.clone()
    a = merge_panoramas(case["width"], case["height"], src, msk, extr, intr)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = merge_panoramas(case["width"], case["height"], src, msk, extr, intr)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(src, s0) and torch.equal(msk, m0)


def _v1_model():
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vits")
    m = MoGeModel(**cfg)
    m.load_state_dict(make_v1_state_dict(cfg, 7, well_posed=True))
    return m.to(DEV).eval()


def _v2_model():
    from moge.model.v2 import MoGeModel
    from moge_b200.configs import model_config
    from moge_b200.synthetic import make_state_dict
    cfg = model_config("vits", True)
    m = MoGeModel(**cfg)
    m.load_state_dict(make_state_dict(cfg, 0, well_posed=True))
    return m.to(DEV).eval()


@pytest.mark.parametrize("make_model", [_v1_model, _v2_model], ids=["moge1", "moge2"])
def test_infer_panoramas_equals_single(make_model):
    from moge_b200.panorama import infer_panorama, infer_panoramas
    from moge_b200.synthetic import synthetic_panorama
    model = make_model()
    imgs = torch.from_numpy(np.stack([synthetic_panorama(128, 256, s) for s in (3, 5, 8)])).to(DEV)
    before = imgs.clone()
    singles = [infer_panorama(model, imgs[k], return_views=True) for k in range(3)]
    for batch_size in (None, 5):
        out = infer_panoramas(model, imgs, batch_size=batch_size, return_views=True)
        assert out["depth"].shape == (3, 128, 256) and out["points"].shape == (3, 128, 256, 3)
        for k, single in enumerate(singles):
            for key, want in single.items():
                assert torch.equal(out[key][k], want), (batch_size, k, key)
    plain = infer_panoramas(model, imgs)
    assert set(plain) == {"depth", "mask", "points"} and all(torch.equal(plain[k], out[k]) for k in plain)
    assert torch.equal(imgs, before)
