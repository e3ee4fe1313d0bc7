"""CPU: MoGe-1 host logic -- resize arithmetic, the bicubic filter of the library against torch, config validation, the
deprecated constructor argument, strict state-dict loading and the C-ABI plumbing (no device needed)."""
import ctypes as C
import warnings

import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from moge_b200.configs import v1_model_config, v1_resized_size
from moge_b200.synthetic import make_v1_state_dict, v1_expected_keys


@pytest.mark.parametrize("H", [70, 98, 126, 331, 518, 768, 1024, 1036, 2160])
@pytest.mark.parametrize("W", [70, 140, 357, 518, 1036, 1920])
@pytest.mark.parametrize("tokens", [120, 1200, 1713, 2500])
def test_resize_arithmetic_matches_reference_formula(H, W, tokens):
    # /root/reference/moge/model/v1.py:273-279
    f = ((tokens * 14 ** 2) / (H * W)) ** 0.5
    rw, rh = int(W * f), int(H * f)
    assert v1_resized_size(H, W, tokens) == (rh, rw)
    assert (rh // 14) * (rw // 14) <= tokens


def test_resize_examples():
    assert v1_resized_size(518, 518, 2500) == (700, 700)
    assert v1_resized_size(518, 1036, 2500) == (494, 989)
    assert v1_resized_size(1024, 768, 2500) == (808, 606)


@pytest.mark.parametrize("n_in,n_out", [(518, 700), (1036, 700), (518, 350), (98, 140), (126, 181), (600, 350), (800, 466),
                                        (1024, 808), (7, 3), (3, 11), (4000, 700)])
def test_bicubic_aa_weights_match_torch(n_in, n_out):
    # one-hot rows through torch's antialiased bicubic resize give its weight matrix column by column
    eye = torch.eye(n_in, dtype=torch.float64).reshape(n_in, 1, 1, n_in)
    ref = F.interpolate(eye, (1, n_out), mode="bicubic", align_corners=False, antialias=True)[:, 0, 0, :]      # [in, out]
    L = capi.lib()
    w = (C.c_float * 64)()
    lo = C.c_int()
    got = torch.zeros(n_in, n_out, dtype=torch.float64)
    for i in range(n_out):
        n = L.moge_bicubic_aa_weights(n_in, n_out, i, C.byref(lo), w, 64)
        assert n > 0
        got[lo.value:lo.value + n, i] = torch.tensor(list(w)[:n], dtype=torch.float64)
    assert float((got - ref).abs().max()) < 2e-6
    assert L.moge_bicubic_aa_weights(n_in, n_out, n_out, C.byref(lo), w, 64) < 0


def _create_error(cfg):
    h = C.c_void_p()
    rc = capi.lib().moge_engine_create_v1(C.byref(capi.make_v1_config(cfg, capi.F16)), 0, C.byref(h))
    assert rc != 0
    return capi.lib().moge_last_error().decode()


@pytest.mark.parametrize("override,msg", [
    ({"last_res_blocks": 1}, "last_res_blocks"),
    ({"last_conv_size": 3}, "last_conv_size"),
    ({"last_conv_channels": 48}, "last_conv_channels"),
    ({"dim_upsample": [256, 128, 96]}, "dim_upsample[2]"),
    ({"dim_proj": 320}, "dim_proj"),
    ({"intermediate_layers": [3, 2]}, "intermediate_layers"),
])
def test_v1_config_validation(override, msg):
    cfg = {**v1_model_config("vitl"), **override}
    assert msg in _create_error(cfg)


def test_v1_valid_config_passes_validation():
    L = capi.lib()
    h = C.c_void_p()
    rc = L.moge_engine_create_v1(C.byref(capi.make_v1_config(v1_model_config("vitl"), capi.F16)), 0, C.byref(h))
    if torch.cuda.is_available():                  # on an H100 the engine is created
        assert rc == 0, L.moge_last_error().decode()
        L.moge_engine_destroy(h)
        return
    # without a device creation gets past the config checks and fails looking for it
    assert rc != 0
    err = L.moge_last_error().decode()
    assert "CUDA device" in err, err


def test_v1_config_struct():
    c = capi.make_v1_config(v1_model_config("vitl"), capi.BF16)
    assert (c.embed_dim, c.depth, c.num_heads, c.num_taps) == (1024, 24, 16, 4)
    assert list(c.taps)[:4] == [20, 21, 22, 23]            # intermediate_layers=4: the last four blocks
    assert (c.dim_proj, c.num_levels, list(c.dim_upsample)[:3]) == (512, 3, [256, 128, 64])
    assert (c.hidden_mult, c.num_res_blocks, c.hidden_norm, c.remap_output, c.compute_dtype) == (2, 2, 0, 2, capi.BF16)
    with pytest.raises(ValueError):
        capi.make_v1_config({**v1_model_config("vits"), "encoder": "dinov2_vitg14"}, capi.F16)
    with pytest.raises(ValueError):
        capi.make_v1_config({**v1_model_config("vits"), "res_block_norm": "batch_norm"}, capi.F16)


def test_v1_deprecated_trained_area_range():
    from moge.model.v1 import MoGeModel
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        m = MoGeModel(encoder="dinov2_vits14", trained_area_range=[196 * 1000, 196 * 2000 + 13])
    assert m.num_tokens_range == [1000, 2000]
    assert any("deprecated" in str(r.message) for r in rec)


def test_v1_strict_load_and_keys():
    from moge.model.v1 import MoGeModel
    cfg = v1_model_config("vits")
    sd = make_v1_state_dict(cfg, 0)
    assert list(sd.keys()) == v1_expected_keys(cfg)
    assert "head.upsample_blocks.2.1.layers.5.weight" in sd and sd["head.upsample_blocks.0.0.0.weight"].shape == (258, 128, 2, 2)
    m = MoGeModel(**cfg)
    r = m.load_state_dict(sd)
    assert not r.missing_keys and not r.unexpected_keys
    bad = dict(sd)
    bad.pop("head.projects.0.bias")
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad)
    with pytest.raises(NotImplementedError):
        m.infer(torch.rand(3, 28, 28), use_fp16=False)
    with pytest.raises(capi.MogeError):
        m.forward(torch.rand(1, 3, 28, 28), 4)           # no CPU path


def test_import_model_class_by_version_names_v1_class():
    from moge.model import import_model_class_by_version
    with pytest.raises(NotImplementedError, match="moge.model.v1.MoGeModel"):
        import_model_class_by_version("v1")
