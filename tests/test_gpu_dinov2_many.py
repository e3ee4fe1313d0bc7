"""-m gpu: the DINOv2 backbone's mixed-shape lists (get_intermediate_layers_many, forward_features_many, forward_many and the C
entry point moge_dino_forward_groups).  Every output of every image is bitwise what the same image gets from a call of its own,
whatever else shares its engine call: the shape mix has a 1 x 37 token grid, a shape whose packed rows fit in one 128-row GEMM
tile (42 x 42: 10 rows per image) and repeated shapes.  The same holds with the list permuted, split into several calls by
`max_chunk_tokens`, and with more shapes than one call may carry.  Each output may be left out at the C level, a mixed call's
tokens are within the 16-bit operand bound of test_gpu_dinov2 against the fp32 port, and a call over G shapes is one front-end
launch and one export launch per exported block."""
import pytest
import torch

from moge_b200 import capi, dinov2
from moge_b200.synthetic import make_dinov2_state_dict, synthetic_dino_input
from oracle.dinov2_port import intermediate_layers
from test_gpu_dinov2 import check_bound

pytestmark = pytest.mark.gpu
DEV = "cuda"
CTORS = {"vits": dinov2.dinov2_vits14, "vitb": dinov2.dinov2_vitb14}
SHAPES = [(98, 126), (14, 518), (42, 42), (98, 126), (126, 98), (42, 42), (70, 70), (98, 126), (518, 14)]
KWARGS = [dict(n=1), dict(n=4, return_class_token=True), dict(n=[2, 7], reshape=True), dict(n=2, norm=False),
          dict(n=[0, 5, 11], reshape=True, return_class_token=True, norm=False)]
_models = {}


def get_model(size, dtype):
    key = (size, dtype)
    if key not in _models:
        m = CTORS[size](pretrained=False)
        m.load_state_dict(make_dinov2_state_dict(size, 3))
        m = m.to(DEV)
        m = m.half() if dtype == torch.float16 else m.bfloat16()
        _models.clear()
        _models[key] = m
    return _models[key]


def make_images(shapes, seed=0):
    """One normalised image per shape; every third one in fp16, to mix input dtypes in one list."""
    out = []
    for i, (H, W) in enumerate(shapes):
        x = synthetic_dino_input(1, H, W, seed + i)[0].to(DEV)
        out.append(x.half() if i % 3 == 2 else x)
    return out


def flat(o):
    """The tensors of one image's result, in a fixed order."""
    if isinstance(o, torch.Tensor):
        return [o]
    if isinstance(o, dict):
        return [o[k] for k in ("x_norm_clstoken", "x_norm_regtokens", "x_norm_patchtokens", "x_prenorm")]
    return [t for item in o for t in flat(item)]


def single(m, x, call, kw):
    """The image's own call, batch dimension dropped."""
    if call == "gil":
        out = m.get_intermediate_layers(x[None], **kw)
        return [t[0] for t in flat(out)]
    if call == "features":
        out = m.forward_features(x[None])
        return [t[0] for t in flat(out)]
    return [m(x[None])[0]]


def many(m, images, call, kw):
    if call == "gil":
        return m.get_intermediate_layers_many(images, **kw)
    if call == "features":
        return m.forward_features_many(images)
    return m.forward_many(images)


def assert_equal_to_single(m, images, outs, call, kw):
    assert len(outs) == len(images)
    for i, (x, o) in enumerate(zip(images, outs)):
        if isinstance(o, dict):
            assert o["masks"] is None
        got, want = flat(o), single(m, x, call, kw)
        assert len(got) == len(want), (i, call, kw)
        for a, b in zip(got, want):
            assert a.shape == b.shape and torch.equal(a, b), (i, tuple(x.shape), call, kw)


@pytest.mark.parametrize("size", ["vits", "vitb"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_each_image_equals_its_own_call(size, dtype):
    m = get_model(size, dtype)
    images = make_images(SHAPES)
    for kw in KWARGS:
        assert_equal_to_single(m, images, many(m, images, "gil", kw), "gil", kw)
    for call in ("features", "forward"):
        assert_equal_to_single(m, images, many(m, images, call, {}), call, {})


def test_permuted_chunked_and_more_shapes_than_one_call():
    m = get_model("vits", torch.float16)
    kw = dict(n=[3, 11], reshape=True, return_class_token=True)
    images = make_images(SHAPES, seed=20)
    base = m.get_intermediate_layers_many(images, **kw)
    perm = [4, 0, 8, 2, 6, 1, 7, 3, 5]
    permuted = m.get_intermediate_layers_many([images[i] for i in perm], **kw)
    for j, i in enumerate(perm):
        assert all(torch.equal(a, b) for a, b in zip(flat(permuted[j]), flat(base[i])))
    old = m.max_chunk_tokens
    try:
        m.max_chunk_tokens = 2 * 64                      # at most two 98 x 126 images per call: several calls
        chunked = m.get_intermediate_layers_many(images, **kw)
    finally:
        m.max_chunk_tokens = old
    for a, b in zip(chunked, base):
        assert all(torch.equal(s, t) for s, t in zip(flat(a), flat(b)))
    # 70 distinct shapes: more than MOGE_DINO_MAX_GROUPS, so two engine calls
    shapes = [(14 * (1 + i % 10), 14 * (1 + i // 10)) for i in range(70)]
    images = make_images(shapes, seed=40)
    outs = m.get_intermediate_layers_many(images, **kw)
    assert_equal_to_single(m, images, outs, "gil", kw)


def test_each_output_may_be_left_out_at_the_c_level():
    """moge_dino_forward_groups over three shapes with out_tokens, out_cls and out_prenorm NULL in turn: the others are unchanged."""
    m = get_model("vits", torch.float16)
    xs = [synthetic_dino_input(B, H, W, 7 + B).to(DEV) for B, H, W in ((2, 98, 126), (3, 42, 42), (1, 14, 518))]
    layers = [3, 11]
    for flags in (0, capi.DINO_NORM, capi.DINO_NORM | capi.DINO_CHANNEL_MAJOR):
        def run(want):
            groups = [(x, m._alloc(x.shape[0], x.shape[2] // 14, x.shape[3] // 14, len(layers), flags, *want)) for x in xs]
            m._dino_call(groups, layers, flags)
            return [outs for _, outs in groups]
        ref = run((True, True, True))
        for drop in range(3):
            want = [k != drop for k in range(3)]
            got = run(want)
            for g in range(len(xs)):
                for k in range(3):
                    assert (got[g][k] is None) == (not want[k])
                    if want[k]:
                        assert torch.equal(got[g][k], ref[g][k]), (flags, drop, g, k)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_mixed_call_within_the_bound_of_the_port(dtype):
    """One mixed call: every token of every image against oracle/dinov2_port.py in fp32 on the CPU, per image."""
    m = get_model("vits", dtype)
    sd = make_dinov2_state_dict("vits", 3)
    images = make_images(SHAPES[:7], seed=60)
    layers = [1, 6, 11]
    for norm in (True, False):
        outs = m.get_intermediate_layers_many(images, n=layers, norm=norm)
        for i, (x, o) in enumerate(zip(images, outs)):
            port = intermediate_layers(sd, x.float().cpu()[None], layers, m.num_heads, norm=norm)
            for layer, t, p in zip(layers, o, port):
                check_bound(t[None], p, layer, dtype, -1, f"image {i} {tuple(x.shape)} norm={norm} layer {layer}")


def test_one_front_end_and_one_export_launch_per_block():
    m = get_model("vits", torch.float16)
    images = make_images(SHAPES)
    for reshape, name in ((False, "dino_export"), (True, "dino_export_chw")):
        m.get_intermediate_layers_many(images, n=4, reshape=reshape)
        names = [op[0] for op in m.engine_ops()]
        assert names.count("dino_patchify") == 1, names
        assert names.count(name) == 4, names
        assert sum(n.startswith("dino_patchify") for n in names) == 1 and sum(n.startswith("dino_export") for n in names) == 4
        assert names.count("dino_prenorm") == 1 and names.count("gemm.patch_embed.g0") == 1     # 6 groups in one call
