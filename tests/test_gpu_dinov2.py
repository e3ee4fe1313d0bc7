"""-m gpu: the DINOv2 backbone (moge_b200.dinov2) against the reference's fp32 outputs (tests/golden/dinov2.pt, written by
oracle/make_dinov2_golden.py: 16 kept patch tokens per output, class tokens whole) and, on every token, against the fp32
restatement oracle/dinov2_port.py that the maker pins to the reference; and its own invariances: per image against a batch of one, chunked against unchunked, each output
left out in turn, channel-major against token-major, and the MoGe-2 encoder's taps through the backbone's own weight keys.

Error bound, per element (the 16-bit operand model of the encoder's op tests, test_gpu_ops / test_gpu_encoder_ops: each GEMM
operand rounded once to 16 bits, unit roundoff u = 2^-11 for fp16 and 2^-8 for bf16, fp32 accumulation).  Every transformer block
rounds R = 6 operands on the way to its two residual updates (norm1 rows, q / k / v, the softmax weights, the attention output,
norm2 rows, the GELU hidden rows); each rounding perturbs the block's output by about u relative to the stream's scale, with
independent signs, so after block l the stream's error is about u sqrt(R (l + 1)) times the row's RMS, and the final LayerNorm
keeps that relative size.  An element is accepted within K = 6 such standard deviations:
    |out - ref| <= K u sqrt(R (l + 1)) rms(ref row)
with rms over the D features of the element's row (its token).  The bound is the model's, not fitted to a measurement; the test
prints the worst ratio of error to bound.
"""
import pytest
import torch

from moge_b200 import capi, dinov2
from moge_b200.configs import IMAGE_MEAN, IMAGE_STD, model_config
from moge_b200.synthetic import make_dinov2_state_dict, make_state_dict, synthetic_dino_input, synthetic_images
from oracle.dinov2_port import intermediate_layers

pytestmark = pytest.mark.gpu
DEV = "cuda"
K_SIGMA, R_ROUNDINGS = 6.0, 6
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
CTORS = {"vits": dinov2.dinov2_vits14, "vitb": dinov2.dinov2_vitb14}
_models = {}


def get_model(size, seed, dtype=torch.float16):
    key = (size, seed, dtype)
    if key not in _models:
        m = CTORS[size](pretrained=False)
        m.load_state_dict(make_dinov2_state_dict(size, seed))
        m = m.to(DEV)
        m = m.half() if dtype == torch.float16 else m.bfloat16()
        _models.clear()
        _models[key] = m
    return _models[key]


def golden(golden_dir):
    return torch.load(f"{golden_dir}/dinov2.pt", weights_only=False)


def check_bound(got, ref, layer, dtype, feat_dim, what):
    got = got.detach().float().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), what
    rms = ref.double().pow(2).mean(dim=feat_dim, keepdim=True).sqrt()
    bound = K_SIGMA * U16[dtype] * (R_ROUNDINGS * (layer + 1)) ** 0.5 * rms
    ratio = float(((got.double() - ref.double()).abs() / bound).max())
    print(f"{what}: worst |err| / bound = {ratio:.3f}")
    assert ratio <= 1.0, (what, ratio)


def run_call(model, call, kw, x):
    if call == "gil":
        return model.get_intermediate_layers(x, **kw)
    if call == "forward_features":
        return model.forward_features(x)
    return model(x)


def pick(t, idx, channel_major):
    """The golden's kept tokens of a (B, T, D) or (B, D, h, w) output (oracle/make_dinov2_golden.py): (B, k, D) or (B, D, k)."""
    t = t.detach().float().cpu()
    return t.flatten(2)[:, :, idx] if channel_major else t[:, idx]


def compare(m, out, ref, call, kw, idx, dtype, what):
    """The engine's outputs against the reference's (the kept tokens, class tokens whole)."""
    depth = m.n_blocks
    if call == "gil":
        layers = m._layers(kw["n"])
        chw = bool(kw.get("reshape"))
        fd = 1 if chw else -1
        assert isinstance(out, tuple) and len(out) == len(ref) == len(layers)
        for j, (o, r) in enumerate(zip(out, ref)):
            if kw.get("return_class_token"):
                assert isinstance(o, tuple) and len(o) == 2
                check_bound(pick(o[0], idx, chw), r[0], layers[j], dtype, fd, f"{what} layer {layers[j]} tokens")
                check_bound(o[1], r[1], layers[j], dtype, -1, f"{what} layer {layers[j]} cls")
            else:
                check_bound(pick(o, idx, chw), r, layers[j], dtype, fd, f"{what} layer {layers[j]}")
    elif call == "forward_features":
        assert set(out) == set(ref) | {"masks"}
        assert out["x_norm_regtokens"].shape == ref["x_norm_regtokens"].shape
        check_bound(out["x_norm_clstoken"], ref["x_norm_clstoken"], depth - 1, dtype, -1, f"{what} x_norm_clstoken")
        check_bound(pick(out["x_norm_patchtokens"], idx, False), ref["x_norm_patchtokens"], depth - 1, dtype, -1,
                    f"{what} x_norm_patchtokens")
        check_bound(pick(out["x_prenorm"], torch.cat([torch.tensor([0]), idx + 1]), False), ref["x_prenorm"], depth - 1, dtype, -1,
                    f"{what} x_prenorm")
        assert out["masks"] is None
    else:
        check_bound(out, ref, depth - 1, dtype, -1, f"{what} forward")


def compare_port(m, out, kw, x, sd, dtype, what):
    """Every patch token of a get_intermediate_layers call against oracle/dinov2_port.py in fp32 on the CPU (the golden's maker
    checks the port against the reference on these calls)."""
    layers = m._layers(kw["n"])
    port = intermediate_layers(sd, x, layers, m.num_heads, norm=kw.get("norm", True))
    for layer, o, p in zip(layers, out, port):
        t = o[0] if kw.get("return_class_token") else o
        if kw.get("reshape"):
            t = t.flatten(2).transpose(1, 2)
        check_bound(t, p, layer, dtype, -1, f"{what} layer {layer} all tokens vs port")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_golden_cases(golden_dir, dtype):
    for c in golden(golden_dir)["cases"]:
        B, H, W = c["shape"]
        m = get_model(c["size"], c["seed"], dtype)
        x = synthetic_dino_input(B, H, W, c["seed"])
        out = run_call(m, c["call"], c["kwargs"], x.to(DEV))
        torch.cuda.synchronize()
        what = f"{c['size']} {B}x{H}x{W} {c['call']} {c['kwargs']}"
        compare(m, out, c["out"], c["call"], c["kwargs"], c["tokens"], dtype, what)
        if c["call"] == "gil":
            compare_port(m, out, c["kwargs"], x, make_dinov2_state_dict(c["size"], c["seed"]), dtype, what)


@pytest.mark.parametrize("xdtype", [torch.float16, torch.bfloat16])
def test_16_bit_inputs(xdtype):
    """x in fp16 / bf16 is read as such: the outputs equal those of the same values passed in fp32."""
    m = get_model("vits", 1)
    x = synthetic_dino_input(2, 98, 126, 5).to(xdtype)
    a = m.get_intermediate_layers(x.to(DEV), n=2, return_class_token=True)
    b = m.get_intermediate_layers(x.float().to(DEV), n=2, return_class_token=True)
    for (ta, ca), (tb, cb) in zip(a, b):
        assert torch.equal(ta, tb) and torch.equal(ca, cb)


def all_outputs(m, x, layers, flags):
    return m._run(x, layers, flags, True, True, True)


def test_each_image_equals_a_batch_of_one():
    m = get_model("vits", 1)
    x = synthetic_dino_input(3, 112, 140, 9).to(DEV)
    for flags in (capi.DINO_NORM, capi.DINO_CHANNEL_MAJOR):
        full = all_outputs(m, x, [2, 7, 11], flags)
        for i in range(3):
            one = all_outputs(m, x[i:i + 1], [2, 7, 11], flags)
            assert torch.equal(full[0][:, i:i + 1], one[0]) and torch.equal(full[1][:, i:i + 1], one[1]), (flags, i)
            assert torch.equal(full[2][i:i + 1], one[2]), (flags, i)


def test_chunked_equals_unchunked():
    m = get_model("vits", 1)
    x = synthetic_dino_input(5, 70, 98, 31).to(DEV)
    full = all_outputs(m, x, [4, 11], capi.DINO_NORM | capi.DINO_CHANNEL_MAJOR)
    gil = m.get_intermediate_layers(x, n=[4, 11], reshape=True, return_class_token=True)
    old = m.max_chunk_tokens
    try:
        m.max_chunk_tokens = 2 * 36 + 5                   # 2 images per engine call: chunks of 2, 2, 1
        chunked = all_outputs(m, x, [4, 11], capi.DINO_NORM | capi.DINO_CHANNEL_MAJOR)
        gil_c = m.get_intermediate_layers(x, n=[4, 11], reshape=True, return_class_token=True)
    finally:
        m.max_chunk_tokens = old
    for a, b in zip(full, chunked):
        assert torch.equal(a, b)
    for (ta, ca), (tb, cb) in zip(gil, gil_c):
        assert torch.equal(ta, tb) and torch.equal(ca, cb)


def test_each_output_may_be_left_out():
    """Each of out_tokens, out_cls and out_prenorm NULL in turn: the others are unchanged."""
    m = get_model("vits", 1)
    x = synthetic_dino_input(2, 98, 126, 4).to(DEV)
    for flags in (0, capi.DINO_NORM, capi.DINO_NORM | capi.DINO_CHANNEL_MAJOR):
        ref = all_outputs(m, x, [3, 11], flags)
        for drop in range(3):
            want = [i != drop for i in range(3)]
            got = m._run(x, [3, 11], flags, *want)
            for i in range(3):
                assert (got[i] is None) == (not want[i])
                if want[i]:
                    assert torch.equal(got[i], ref[i]), (flags, drop, i)
    assert torch.equal(m(x), all_outputs(m, x, [11], capi.DINO_NORM)[1][0])


def test_channel_major_is_the_permuted_token_major():
    m = get_model("vitb", 4)
    x = synthetic_dino_input(2, 126, 98, 6).to(DEV)
    for norm in (True, False):
        tm = m.get_intermediate_layers(x, n=3, norm=norm, return_class_token=True)
        cm = m.get_intermediate_layers(x, n=3, norm=norm, reshape=True, return_class_token=True)
        for (t, ct), (c, cc) in zip(tm, cm):
            assert c.is_contiguous() and c.shape == (2, 768, 9, 7)
            assert torch.equal(t.reshape(2, 9, 7, 768).permute(0, 3, 1, 2), c) and torch.equal(ct, cc)


def test_moge2_backbone_weights_match_the_port():
    """A synthetic MoGe-2 checkpoint's encoder.backbone.* tensors, loaded under the backbone's own keys, give at the model's
    token grid the oracle port's fp32 taps (normalised, the patch tokens; oracle/dinov2_port.py over oracle/moge_port.py)
    within the bound."""
    cfg = model_config("vits")
    sd = make_state_dict(cfg, 2)
    bb = "encoder.backbone."
    m = dinov2.dinov2_vits14(pretrained=False)
    m.load_state_dict({k[len(bb):]: v for k, v in sd.items() if k.startswith(bb)})
    m = m.to(DEV).half()
    taps = list(cfg["encoder"]["intermediate_layers"])
    h, w = 10, 13
    img = synthetic_images(2, 14 * h, 14 * w, 8)
    x = (img - torch.tensor(IMAGE_MEAN).view(1, 3, 1, 1)) / torch.tensor(IMAGE_STD).view(1, 3, 1, 1)
    got = m.get_intermediate_layers(x.to(DEV), n=taps, norm=True)
    ref = intermediate_layers(sd, x, taps, 6, prefix=bb)
    for layer, g, r in zip(taps, got, ref):
        check_bound(g, r, layer, torch.float16, -1, f"MoGe-2 tap {layer}")
