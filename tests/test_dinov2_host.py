"""CPU: host side of the DINOv2 backbone (moge_b200.dinov2, aliases under moge.model.dinov2): constructors and the variants they
refuse, state-dict keys, the layer selection of get_intermediate_layers, and the argument checks, which all run before any device
work (a model still on the CPU gets past them only to the engine's 'no CPU path' error)."""
import ctypes as C
import os

import pytest
import torch

from moge_b200 import capi, dinov2
from moge_b200.synthetic import make_dinov2_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dinov2.pt")


def test_aliases_resolve_to_the_engine_classes():
    from moge.model.dinov2 import DinoVisionTransformer
    from moge.model.dinov2.hub.backbones import dinov2_vitl14, dinov2_vitg14, dinov2_vits14_reg
    from moge.model.dinov2.models.vision_transformer import vit_large
    assert DinoVisionTransformer is dinov2.DinoVisionTransformer
    assert dinov2_vitl14 is dinov2.dinov2_vitl14 and vit_large is dinov2.vit_large
    assert dinov2_vitg14 is dinov2.dinov2_vitg14 and dinov2_vits14_reg is dinov2.dinov2_vits14_reg


@pytest.mark.parametrize("ctor, dims", [(dinov2.dinov2_vits14, (384, 12, 6)), (dinov2.dinov2_vitb14, (768, 12, 12)),
                                        (dinov2.dinov2_vitl14, (1024, 24, 16))])
def test_hub_constructors(ctor, dims):
    m = ctor(pretrained=False)
    assert (m.embed_dim, m.n_blocks, m.num_heads) == dims
    assert m.num_features == m.embed_dim and m.patch_size == 14 and m.num_register_tokens == 0 and m.num_tokens == 1
    with pytest.raises(NotImplementedError, match="pretrained=True"):
        ctor()                                  # the reference's default downloads; here it says to load a state dict


@pytest.mark.parametrize("ctor", [dinov2.dinov2_vitg14, dinov2.dinov2_vits14_reg, dinov2.dinov2_vitb14_reg,
                                  dinov2.dinov2_vitl14_reg, dinov2.dinov2_vitg14_reg])
def test_rejected_hub_variants_say_why(ctor):
    with pytest.raises(NotImplementedError, match="ViT-g|register"):
        ctor(pretrained=False)


@pytest.mark.parametrize("kw, match", [
    (dict(ffn_layer="swiglufused"), "SwiGLU"), (dict(ffn_layer="identity"), "GELU MLP"), (dict(num_register_tokens=4), "register"),
    (dict(patch_size=16), "patch_size"), (dict(img_size=224), "37 x 37"), (dict(init_values=None), "LayerScale"),
    (dict(block_chunks=1), "block_chunks"), (dict(interpolate_antialias=True), "antialias"),
    (dict(interpolate_offset=0.0), "offset")])
def test_rejected_configs_say_why(kw, match):
    args = dict(patch_size=14, img_size=518, init_values=1.0, block_chunks=0)
    args.update(kw)
    with pytest.raises(NotImplementedError, match=match):
        dinov2.vit_small(**args)


def test_unknown_ffn_layer_raises_like_the_reference():
    with pytest.raises(NotImplementedError):
        dinov2.vit_small(patch_size=14, img_size=518, init_values=1.0, block_chunks=0, ffn_layer="conv")


def test_state_dict_keys_match_the_reference():
    g = torch.load(GOLDEN, weights_only=False)
    for size, ctor in (("vits", dinov2.dinov2_vits14), ("vitb", dinov2.dinov2_vitb14)):
        m = ctor(pretrained=False)
        assert sorted(m._expected_keys()) == sorted(g["keys"][size])
        sd = make_dinov2_state_dict(size, 0)
        assert sorted(sd) == sorted(g["keys"][size])
        rep = m.load_state_dict(sd)
        assert rep.missing_keys == [] and rep.unexpected_keys == []
        assert set(m.state_dict()) == set(sd)


def test_load_state_dict_report():
    m = dinov2.dinov2_vits14(pretrained=False)
    sd = make_dinov2_state_dict("vits", 0)
    sd.pop("norm.bias")
    sd["head.weight"] = torch.zeros(1)
    with pytest.raises(RuntimeError, match="DinoVisionTransformer"):
        m.load_state_dict(sd)
    rep = m.load_state_dict(sd, strict=False)
    assert rep.missing_keys == ["norm.bias"] and rep.unexpected_keys == ["head.weight"]


def test_layer_selection_follows_the_reference():
    m = dinov2.dinov2_vits14(pretrained=False)
    assert m._layers(1) == [11] and m._layers(4) == [8, 9, 10, 11] and m._layers(0) == []
    assert m._layers([3, 1]) == [1, 3]                  # the reference collects in block order
    assert m._layers((0, 11)) == [0, 11] and m._layers(range(2)) == [0, 1]
    for bad, msg in ((13, "only 12 / 13"), ([12], "only 0 / 1"), ([-1], "only 0 / 1"), ([2, 2], "only 1 / 2")):
        with pytest.raises(AssertionError, match=msg):
            m._layers(bad)


def test_bad_inputs_raise_before_device_work():
    m = dinov2.dinov2_vits14(pretrained=False)
    m.load_state_dict(make_dinov2_state_dict("vits", 0))
    with pytest.raises(AssertionError, match="height 100 is not a multiple of patch height 14"):
        m.get_intermediate_layers(torch.zeros(1, 3, 100, 98))
    with pytest.raises(AssertionError, match="width 100 is not a multiple"):
        m.forward_features(torch.zeros(1, 3, 98, 100))
    with pytest.raises(ValueError, match=r"\(B, 3, H, W\)"):
        m(torch.zeros(3, 98, 98))
    with pytest.raises(ValueError, match=r"\(B, 3, H, W\)"):
        m.get_intermediate_layers(torch.zeros(1, 4, 98, 98))
    with pytest.raises(TypeError, match="float32, float16 or bfloat16"):
        m.get_intermediate_layers(torch.zeros(1, 3, 98, 98, dtype=torch.uint8))
    with pytest.raises(AssertionError, match="blocks found"):
        m.get_intermediate_layers(torch.zeros(1, 3, 98, 98), n=[12])
    with pytest.raises(NotImplementedError, match="masks"):
        m.forward_features(torch.zeros(1, 3, 98, 98), masks=torch.zeros(1, 49, dtype=torch.bool))
    with pytest.raises(NotImplementedError, match="is_training"):
        m(torch.zeros(1, 3, 98, 98), is_training=True)
    with pytest.raises(NotImplementedError, match="list"):
        m.forward_features([torch.zeros(1, 3, 98, 98)])
    with pytest.raises(NotImplementedError):
        m.init_weights()
    with pytest.raises(NotImplementedError):
        m.onnx_compatible_mode = True
    m.onnx_compatible_mode = False
    assert m.get_intermediate_layers(torch.zeros(1, 3, 98, 98), n=0) == ()     # nothing asked, nothing run
    with pytest.raises(capi.MogeError, match="no CPU path"):                  # valid arguments reach the engine
        m.get_intermediate_layers(torch.zeros(1, 3, 98, 98))


def test_c_abi_group_signatures():
    for n in ("moge_dino_create", "moge_dino_workspace_bytes_groups", "moge_dino_forward_groups"):
        assert n in capi.SIGNATURES and n in capi.EXPORTS
    c = capi.DinoConfig()
    c.interpolate_offset = 0.1
    assert C.sizeof(c) == 9 * 4


def test_c_group_checks_without_a_device():
    """The entry points' own checks: a null config or engine fails before anything touches a device."""
    L = capi.lib()
    h = C.c_void_p()
    assert L.moge_dino_create(None, 0, C.byref(h)) != 0 and b"null argument" in L.moge_last_error()
    n = C.c_size_t()
    lay = (C.c_int * 1)(11)
    g = (capi.DinoGroup * 1)()
    g[0].B, g[0].H, g[0].W = 1, 98, 98
    assert L.moge_dino_workspace_bytes_groups(None, g, 1, lay, 1, 1, C.byref(n)) != 0 and b"null argument" in L.moge_last_error()
    assert L.moge_dino_forward_groups(None, g, 1, lay, 1, 1, None, 0, None) != 0 and b"null argument" in L.moge_last_error()
