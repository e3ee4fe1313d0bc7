"""MoGe-1 mixed-shape batches (MoGeModel.infer_many, moge_v1_forward_groups): every image must come out of one packed engine call
as it comes out of infer() alone, the encoder must run once per block for all shapes, and the golden cases must keep their
parity with the reference when they share a call with an image of another shape."""
import ctypes as C
import os

import pytest
import torch

from gpu_util import rel_l2
from moge_b200 import capi
from moge_b200.configs import default_num_tokens, model_config, v1_model_config, v1_resized_size
from moge_b200.synthetic import make_v1_state_dict, synthetic_images

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.startswith("v1_") and f.endswith(".pt"))
# five shapes, some repeated: (H, W)
SHAPES = [(98, 196), (126, 168), (140, 140), (168, 126), (196, 98), (126, 168), (98, 196), (140, 140), (140, 140)]
TOKENS = 130


def _model(cfg, sd, dtype=torch.float16):
    from moge.model.v1 import MoGeModel
    m = MoGeModel(**cfg)
    m.load_state_dict(sd)
    m = m.to(DEV)
    return m.bfloat16() if dtype == torch.bfloat16 else m.half()


@pytest.fixture(scope="module")
def small():
    cfg = v1_model_config("vits")
    return cfg, make_v1_state_dict(cfg, 7, well_posed=True)


def _images(shapes, seed):
    return [synthetic_images(1, H, W, seed + i)[0].to(DEV) for i, (H, W) in enumerate(shapes)]


def _assert_matches_infer(model, imgs, many, num_tokens, **kw):
    assert len(many) == len(imgs)
    for i, im in enumerate(imgs):
        one = model.infer(im, num_tokens=num_tokens, **kw)
        assert set(one.keys()) == set(many[i].keys())
        assert torch.equal(one["mask"], many[i]["mask"]), i
        m = one["mask"]
        for k in ("points", "depth"):
            e = rel_l2(many[i][k][m], one[k][m])
            assert e < 1e-5, (i, k, e)
        assert rel_l2(many[i]["intrinsics"], one["intrinsics"]) < 1e-5, i


def test_infer_many_mixed_shapes_matches_per_image_infer(small):
    model = _model(*small)
    imgs = _images(SHAPES, 60)
    many = model.infer_many(imgs, num_tokens=TOKENS)
    torch.cuda.synchronize()
    names = [n for n, _, _ in model.engine_ops()]
    assert sum(n.startswith("attention") for n in names) == 12            # ONE attention launch per block for all five shapes
    assert sum(n.startswith("resize_bicubic_aa") for n in names) == 5     # one resize per shape group
    assert sum(n.startswith("head_output") for n in names) == 5
    assert "head_output.g4" in names and "convT.g4.l0" in names           # per-group names, level last
    _assert_matches_infer(model, imgs, many, TOKENS)
    # the same with fov_x, apply_mask and force_projection passed through
    many = model.infer_many(imgs[:4], fov_x=55.0, num_tokens=TOKENS, apply_mask=False, force_projection=False)
    _assert_matches_infer(model, imgs[:4], many, TOKENS, fov_x=55.0, apply_mask=False, force_projection=False)


def test_infer_many_chunks_into_several_calls(small):
    model = _model(*small)
    imgs = _images(SHAPES, 70)

    def geometry(H, W):
        rh, rw = v1_resized_size(H, W, TOKENS)
        return (rh, rw), (rh // 14) * (rw // 14) + 1

    model.max_chunk_tokens = 3 * max(geometry(H, W)[1] for H, W in SHAPES)       # several engine calls, with mixed groups
    calls = model._pack_calls(imgs, geometry)
    assert len(calls) > 1 and any(len(c) > 1 for c in calls)
    many = model.infer_many(imgs, num_tokens=TOKENS)
    torch.cuda.synchronize()
    _assert_matches_infer(model, imgs, many, TOKENS)


def test_infer_many_bf16_matches_per_image_infer(small):
    model = _model(*small, dtype=torch.bfloat16)
    imgs = _images(SHAPES[:6], 80)
    many = model.infer_many(imgs, num_tokens=TOKENS)
    torch.cuda.synchronize()
    _assert_matches_infer(model, imgs, many, TOKENS)


def test_infer_many_deterministic(small):
    model = _model(*small)
    imgs = _images(SHAPES, 90)
    a = model.infer_many(imgs, num_tokens=TOKENS)
    b = model.infer_many(imgs, num_tokens=TOKENS)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        for k in x:
            assert torch.equal(x[k], y[k]), k


def _groups(groups):
    arr = (capi.V1Group * len(groups))()
    for g, (B, H, W, rh, rw) in zip(arr, groups):
        g.B, g.H, g.W, g.rh, g.rw = B, H, W, rh, rw
    return arr


def test_group_workspace_bytes_and_checks(small):
    model = _model(*small)
    model._ensure_engine()
    L, e = capi.lib(), model._engine
    shapes = [(2, 98, 196, *v1_resized_size(98, 196, 500)), (1, 518, 518, *v1_resized_size(518, 518, 1200)),
              (3, 140, 140, *v1_resized_size(140, 140, 130))]
    single = []
    for s in shapes:
        a = C.c_size_t()
        capi.check(L.moge_v1_workspace_bytes_groups(e, _groups([s]), 1, C.byref(a)))
        single.append(a.value)
    both = C.c_size_t()
    capi.check(L.moge_v1_workspace_bytes_groups(e, _groups(shapes), 3, C.byref(both)))
    assert max(single) < both.value <= sum(single), (both.value, single)
    # every group is checked before anything runs
    assert L.moge_v1_workspace_bytes_groups(e, _groups([shapes[0], (1, 98, 98, 13, 98)]), 2, C.byref(both)) != 0
    assert "smaller than one 14-pixel patch" in L.moge_last_error().decode()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    img = torch.zeros(2, 3, 98, 196, device=DEV)
    arr = _groups([shapes[0]])
    arr[0].image, arr[0].image_dtype = img.data_ptr(), capi.F32
    assert L.moge_v1_forward_groups(e, arr, 1, ws.data_ptr(), ws.numel(), capi.current_stream()) != 0      # null outputs
    assert "null argument" in L.moge_last_error().decode()
    out = torch.empty(2, 98, 196, 3, device=DEV)
    arr[0].points, arr[0].mask, arr[0].image_dtype = out.data_ptr(), out.data_ptr(), 7
    assert L.moge_v1_forward_groups(e, arr, 1, ws.data_ptr(), ws.numel(), capi.current_stream()) != 0
    assert "image dtype" in L.moge_last_error().decode()
    assert L.moge_engine_forward_groups(e, (capi.Group * 1)(), 1, ws.data_ptr(), ws.numel(), capi.current_stream()) != 0
    # a MoGe-2 engine is refused
    h = C.c_void_p()
    capi.check(L.moge_engine_create(C.byref(capi.make_config(model_config("vits", True), capi.F16)), 0, C.byref(h)))
    try:
        assert L.moge_v1_workspace_bytes_groups(h, _groups([shapes[0]]), 1, C.byref(both)) != 0
        assert "not a MoGe-1 engine" in L.moge_last_error().decode()
    finally:
        L.moge_engine_destroy(h)


def _case(name):
    gold = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    meta = gold["meta"]
    cfg = v1_model_config(meta["size"])
    cfg["remap_output"] = meta["remap_output"]
    sd = make_v1_state_dict(cfg, meta["seed"], well_posed=meta["well_posed"])
    img = synthetic_images(*meta["shape"], meta["seed"])
    return gold, cfg, sd, img


@pytest.mark.parametrize("name", CASES)
def test_v1_golden_through_infer_many(name):
    """Each golden case shares its engine call with images of another shape, which take the first rows of the packed encoder
    matrices and the first decoder group, so the case runs at a non-zero row offset as group 1."""
    gold, cfg, sd, img = _case(name)
    meta = gold["meta"]
    s = meta["stride"]
    model = _model(cfg, sd)
    num_tokens = meta["num_tokens"]
    tokens = num_tokens if num_tokens is not None else default_num_tokens(cfg["num_tokens_range"], 9)
    B, H, W = meta["shape"]
    Ho, Wo = (H + 28, W - 14) if W > H else (H - 14, W + 28)
    other = synthetic_images(B + 1, Ho, Wo, meta["seed"] + 100).to(DEV)
    # forward: the batched path's raw outputs (other group first)
    rh, rw = v1_resized_size(H, W, tokens)
    outs = model._forward_groups([(other, *v1_resized_size(Ho, Wo, tokens)), (img.to(DEV), rh, rw)])
    torch.cuda.synchronize()
    for k, got in zip(("points", "mask"), outs[1]):
        err = rel_l2(got[:, ::s, ::s], gold["forward"][k])
        print(f"{name} batched forward {k}: rel-L2 {err:.2e}")
        assert err < 1e-3, (name, k, err)
    if not meta["well_posed"]:
        return
    imgs = [im for im in img.to(DEV)] + [im for im in other]
    for key, ref in gold["infer"].items():
        many = model.infer_many(imgs, num_tokens=num_tokens, **ref["kwargs"])
        torch.cuda.synchronize()
        got = {k: torch.stack([many[b][k] for b in range(B)]) for k in many[0]}
        agree = float((got["mask"][:, ::s, ::s].cpu() == ref["mask"]).float().mean())
        print(f"{name} infer_many[{key}] mask agreement {agree:.5f}")
        assert agree > 0.997, (name, key, agree)
        m = got["mask"][:, ::s, ::s].cpu() & ref["mask"]
        for k in ("points", "depth"):
            err = rel_l2(got[k][:, ::s, ::s].cpu()[m], ref[k][m])
            print(f"{name} infer_many[{key}] {k}: rel-L2 {err:.2e}")
            assert err < 5e-3, (name, key, k, err)
        assert rel_l2(got["intrinsics"], ref["intrinsics"]) < 2e-3, (name, key)
