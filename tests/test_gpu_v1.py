"""MoGe-1 on the engine (moge.model.v1.MoGeModel): golden parity against the unmodified reference (tests/golden/v1_*.pt, written
by oracle/make_v1_golden.py), operator checks of the new kernels, and the engine properties the MoGe-2 tests pin (batching,
chunking, graph replay, determinism, checkpoint loading)."""
import os

import pytest
import torch
import torch.nn.functional as F

from gpu_util import border_ok, check_tiles, dt, empty_padded, from_padded_nhwc, rel_l2, stream, tile_conv, to_padded_nhwc
from moge_b200 import capi
from moge_b200.configs import uv_spans, v1_model_config
from moge_b200.synthetic import make_v1_state_dict, synthetic_images
from oracle import moge_v1_port
from oracle.moge_port import view_plane_uv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.startswith("v1_") and f.endswith(".pt"))


def _model(cfg, sd, dtype=torch.float16):
    from moge.model.v1 import MoGeModel
    m = MoGeModel(**cfg)
    m.load_state_dict(sd)
    m = m.to(DEV)
    return m.bfloat16() if dtype == torch.bfloat16 else m.half()


def _case(name):
    gold = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    meta = gold["meta"]
    cfg = v1_model_config(meta["size"])
    cfg["remap_output"] = meta["remap_output"]
    sd = make_v1_state_dict(cfg, meta["seed"], well_posed=meta["well_posed"])
    img = synthetic_images(*meta["shape"], meta["seed"])
    return gold, cfg, sd, img


def _tokens(cfg, meta):
    if meta["num_tokens"] is not None:
        return meta["num_tokens"]
    lo, hi = cfg["num_tokens_range"]
    return int(lo + (9 / 9) * (hi - lo))


@pytest.mark.parametrize("name", CASES)
def test_v1_golden(name):
    gold, cfg, sd, img = _case(name)
    meta = gold["meta"]
    s = meta["stride"]
    model = _model(cfg, sd)
    out = model.forward(img.to(DEV), _tokens(cfg, meta))
    for k in ("points", "mask"):
        err = rel_l2(out[k][:, ::s, ::s], gold["forward"][k])
        print(f"{name} forward {k}: rel-L2 {err:.2e} (reference autocast: {meta['reference_autocast_deviation']})")
        assert err < 1e-3, (name, k, err)
    if not meta["well_posed"]:
        return
    for key, ref in gold["infer"].items():
        got = model.infer(img.to(DEV), num_tokens=meta["num_tokens"], **ref["kwargs"])
        agree = float((got["mask"][:, ::s, ::s].cpu() == ref["mask"]).float().mean())
        print(f"{name} infer[{key}] mask agreement {agree:.5f}")
        assert agree > 0.997, (name, key, agree)
        m = got["mask"][:, ::s, ::s].cpu() & ref["mask"]
        for k in ("points", "depth"):
            err = rel_l2(got[k][:, ::s, ::s].cpu()[m], ref[k][m])
            print(f"{name} infer[{key}] {k}: rel-L2 {err:.2e}")
            assert err < 5e-3, (name, key, k, err)
        err = rel_l2(got["intrinsics"], ref["intrinsics"])
        assert err < 2e-3, (name, key, err)
        if not ref["kwargs"].get("apply_mask", True):
            assert torch.isfinite(got["points"]).all()


def _small():
    cfg = v1_model_config("vits")
    sd = make_v1_state_dict(cfg, 7, well_posed=True)
    return cfg, sd


def test_v1_bf16():
    cfg, sd = _small()
    img = synthetic_images(2, 126, 168, 7)
    out = _model(cfg, sd, torch.bfloat16).forward(img.to(DEV), 192)
    ref = moge_v1_port.forward(cfg, sd, img, 192)
    for k in ("points", "mask"):
        err = rel_l2(out[k], ref[k])
        print(f"bf16 {k}: {err:.2e}")
        assert err < 1e-2, (k, err)


def test_v1_vitl_batch8_against_gpu_port():
    cfg = v1_model_config("vitl")
    sd = make_v1_state_dict(cfg, 30, well_posed=True)
    img = synthetic_images(8, 518, 518, 30)
    out = _model(cfg, sd).forward(img.to(DEV), 2500)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    ref = moge_v1_port.forward(cfg, sd_dev, img.to(DEV), 2500)
    for k in ("points", "mask"):
        err = rel_l2(out[k], ref[k])
        print(f"ViT-L B=8 {k}: rel-L2 vs GPU-run port {err:.2e}")
        assert err < 1e-3, (k, err)


def test_v1_batch_invariance_chunks_and_determinism():
    cfg, sd = _small()
    model = _model(cfg, sd)
    img = synthetic_images(3, 98, 140, 8).to(DEV)
    full = model.forward(img, 150)
    again = model.forward(img, 150)
    for k in full:
        assert torch.equal(full[k], again[k]), k                 # graph replay into fresh outputs, bit for bit
    for b in range(3):
        one = model.forward(img[b:b + 1], 150)
        for k in full:
            assert rel_l2(one[k][0], full[k][b]) < 1e-5, (b, k)
    model.max_chunk_tokens = 2 * (150 + 1)                        # chunks of at most 2 images: a 2 + 1 split
    chunked = model.forward(img, 150)
    for k in full:
        assert rel_l2(chunked[k], full[k]) < 1e-5, k


def test_v1_infer_squeeze_fov_tensor_and_options():
    cfg, sd = _small()
    model = _model(cfg, sd)
    img = synthetic_images(2, 112, 140, 9)
    one = model.infer(img[0].to(DEV), num_tokens=160)
    assert one["points"].shape == (112, 140, 3) and one["depth"].shape == (112, 140) and one["intrinsics"].shape == (3, 3)
    assert one["mask"].dtype == torch.bool
    fov = torch.tensor([50.0, 70.0])
    got = model.infer(img.to(DEV), fov_x=fov.to(DEV), num_tokens=160)
    raw = model.forward(img.to(DEV), 160)
    ref = moge_v1_port.postprocess(raw["points"].cpu(), raw["mask"].cpu(), 140 / 112, fov_x=fov)
    assert rel_l2(got["intrinsics"], ref["intrinsics"]) < 1e-5
    m = got["mask"].cpu() & ref["mask"]
    for k in ("points", "depth"):
        assert rel_l2(got[k].cpu()[m], ref[k][m]) < 5e-3, k
    nomask = model.infer(img.to(DEV), num_tokens=160, apply_mask=False, force_projection=False)
    ref = moge_v1_port.postprocess(raw["points"].cpu(), raw["mask"].cpu(), 140 / 112, apply_mask=False, force_projection=False)
    assert torch.isfinite(nomask["points"]).all()
    for k in ("points", "depth"):
        assert rel_l2(nomask[k].cpu(), ref[k]) < 5e-3, k


@pytest.mark.parametrize("kw", [{}, {"fov_x": 55.0}, {"apply_mask": False}, {"force_projection": False}])
def test_v1_postprocess_chain_exact(kw):
    # the post-processing after the focal/shift solve (threshold, intrinsics, depth, re-projection or z shift, masking) against
    # the oracle's, with the engine's own focal and shift injected: only fp32 rounding separates the two
    cfg, sd = _small()
    model = _model(cfg, sd)
    img = synthetic_images(2, 112, 140, 11)
    raw = model.forward(img.to(DEV), 160)
    B, H, W = raw["mask"].shape
    aspect = W / H
    pts = raw["points"].clone()
    focal_in = None
    if "fov_x" in kw:
        focal_in = torch.full((B,), aspect / (1 + aspect ** 2) ** 0.5 / torch.tan(torch.deg2rad(torch.tensor(kw["fov_x"] / 2))).item(),
                              device=DEV)
    focal, shift = torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    depth, intr = torch.empty(B, H, W, device=DEV), torch.empty(B, 3, 3, device=DEV)
    mask_out = torch.empty(B, H, W, dtype=torch.uint8, device=DEV)
    capi.check(capi.lib().moge_v1_postprocess(pts.data_ptr(), raw["mask"].data_ptr(), 0.5, capi.ptr(focal_in), B, H, W,
                                              int(kw.get("force_projection", True)), int(kw.get("apply_mask", True)), depth.data_ptr(),
                                              mask_out.data_ptr(), intr.data_ptr(), focal.data_ptr(), shift.data_ptr(), stream()))
    torch.cuda.synchronize()
    if focal_in is not None:
        assert torch.equal(focal, focal_in)
    ref = moge_v1_port.postprocess(raw["points"].cpu(), raw["mask"].cpu(), aspect, 0.5, None, kw.get("force_projection", True),
                                   kw.get("apply_mask", True), focal_shift=(focal.cpu(), shift.cpu()))
    assert torch.equal(mask_out.cpu().bool(), ref["mask"])
    assert rel_l2(intr, ref["intrinsics"]) < 1e-6
    fin = torch.isfinite(ref["depth"])
    assert torch.equal(torch.isfinite(depth.cpu()), fin)
    assert rel_l2(depth.cpu()[fin], ref["depth"][fin]) < 1e-5
    assert rel_l2(pts.cpu()[fin], ref["points"][fin]) < 1e-5


def test_v1_from_pretrained_round_trip(tmp_path):
    from moge.model.v1 import MoGeModel
    cfg, sd = _small()
    path = tmp_path / "model.pt"
    torch.save({"model_config": cfg, "model": sd}, path)
    a = MoGeModel.from_pretrained(str(path)).to(DEV).half()
    b = _model(cfg, sd)
    img = synthetic_images(1, 98, 126, 3).to(DEV)
    oa, ob = a.forward(img, 120), b.forward(img, 120)
    for k in oa:
        assert torch.equal(oa[k], ob[k]), k
    ops = a.engine_ops()
    assert any(n.startswith("groupnorm_stats") for n, _, _ in ops) and len(a.engine_profile()) == len(ops)


@pytest.mark.parametrize("shape", [((518, 518), (700, 700)), ((1036, 518), (700, 350)), ((98, 126), (140, 181)),
                                   ((600, 800), (350, 466)), ((1024, 768), (808, 606))])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_op_resize_bicubic_aa(shape, dtype):
    (H, W), (Ho, Wo) = shape
    g = torch.Generator().manual_seed(H + W)
    x = torch.rand(2, 3, H, W, generator=g).to(DEV, dtype)
    out = torch.empty(2, 3, Ho, Wo, device=DEV)
    capi.check(capi.lib().moge_op_resize_bicubic_aa(x.data_ptr(), dt(dtype), 2, 3, H, W, Ho, Wo, out.data_ptr(), stream()))
    torch.cuda.synchronize()
    ref = F.interpolate(x.float(), (Ho, Wo), mode="bicubic", align_corners=False, antialias=True)
    assert float((out - ref).abs().max()) < 1e-4


@pytest.mark.parametrize("B,H,W,C,G", [(2, 13, 21, 64, 1), (1, 40, 50, 128, 4), (2, 7, 9, 256, 1), (1, 33, 65, 512, 16)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_op_groupnorm_relu(B, H, W, C, G, dtype):
    g = torch.Generator().manual_seed(C + H)
    x = (torch.randn(B, C, H, W, generator=g) * 2 + 0.5).to(DEV)
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(C, generator=g)).to(DEV)
    xp = to_padded_nhwc(x, dtype)
    out = empty_padded(B, H, W, C, dtype, DEV)
    capi.check(capi.lib().moge_op_groupnorm_relu(xp.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), B, H, W, C, G, dt(dtype),
                                                 stream()))
    torch.cuda.synchronize()
    xin = from_padded_nhwc(xp, H, W)
    ref = F.relu(F.group_norm(xin, G, gamma, beta, 1e-5))
    got = from_padded_nhwc(out, H, W)
    tol = 1e-2 if dtype == torch.bfloat16 else 2e-3
    assert float((got - ref).abs().max() / ref.abs().max()) < tol
    assert border_ok(out, H, W)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 3, 4, 128, 64), (1, 4, 3, 64, 128)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_op_convT_input_grid_uv(B, H, W, Cin, Cout, dtype):
    """ConvTranspose2d(Cin + 2 -> Cout, k2 s2) over cat(x, uv) with uv on the INPUT grid (v1.py:123-129), as the engine runs it
    (convT GEMM + uv_convT_kernel, the UV rows packed by the same load-time kernel), against torch.  The UV rows are large so
    that taking u, v on the output grid instead (MoGe-2's convention) fails the tolerance by a wide margin; the test checks that."""
    g = torch.Generator().manual_seed(Cin + Cout + H)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cin + 2, Cout, 2, 2, generator=g) / Cin ** 0.5
    w[Cin:] = 4.0 * torch.randn(2, Cout, 2, 2, generator=g)
    bias = 0.1 * torch.randn(Cout, generator=g)
    aspect = 1.3
    su, sv = uv_spans(aspect)
    xp = to_padded_nhwc(x.to(DEV), dtype)
    out = empty_padded(B, 2 * H, 2 * W, Cout, dtype, DEV)
    wd, bd = w.to(DEV), bias.to(DEV)
    capi.check(capi.lib().moge_op_conv_transpose_uv(xp.data_ptr(), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), B, H, W, Cin, Cout, su, sv,
                                           dt(dtype), stream()))
    torch.cuda.synchronize()
    assert border_ok(out, 2 * H, 2 * W)
    got = from_padded_nhwc(out, 2 * H, 2 * W).cpu()
    xq = x.to(dtype).float()                       # the engine's operands: 16-bit map and feature rows, fp32 UV rows
    wq = w.clone()
    wq[:Cin] = w[:Cin].to(dtype).float()
    uv_in = view_plane_uv(W, H, aspect).permute(2, 0, 1)[None].expand(B, -1, -1, -1)
    ref = F.conv_transpose2d(torch.cat([xq, uv_in], dim=1), wq, bias, stride=2)
    uv_out = view_plane_uv(2 * W, 2 * H, aspect).permute(2, 0, 1)
    wrong = F.conv_transpose2d(xq, wq[:Cin], bias, stride=2) + wq[Cin].repeat(1, H, W) * uv_out[0] + wq[Cin + 1].repeat(1, H, W) * uv_out[1]
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max()) / scale
    err_wrong = float((wrong - ref).abs().max()) / scale
    tol = 1e-2 if dtype == torch.bfloat16 else 2e-3
    print(f"convT uv {dtype}: err {err:.2e}, output-grid convention would be {err_wrong:.2e}")
    assert err < tol, err
    assert err_wrong > 5 * tol, err_wrong
    # tile by tile on the 2H x 2W output grid, so that a wrong UV phase at a ragged edge is named by its tile
    check_tiles(got, ref, tile_conv(Cout), tol, f"convT uv {dtype}")
