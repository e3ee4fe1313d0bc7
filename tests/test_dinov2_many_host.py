"""CPU: host side of the DINOv2 backbone's mixed-shape lists (get_intermediate_layers_many, forward_features_many, forward_many):
the packing of a list into engine calls (buckets by shape and dtype, input order, the group cap, chunking), the argument checks,
which all run before any device work, and the C checks of the group entry points (no device needed).  The engine call itself
is replaced by a stand-in that writes each image's index into its outputs, so the whole host path runs on the CPU."""
import ctypes as C

import pytest
import torch

from moge_b200 import capi, dinov2
from moge_b200.synthetic import make_dinov2_state_dict


def _model():
    m = dinov2.dinov2_vits14(pretrained=False)
    m.load_state_dict(make_dinov2_state_dict("vits", 0))
    return m


def _images(shapes, dtype=torch.float32, first=0):
    """Image i is filled with the value first + i, so that a stand-in engine call can tell the images apart."""
    return [torch.full((3, H, W), float(first + i), dtype=dtype) for i, (H, W) in enumerate(shapes)]


class _Recorder:
    """Stands in for `_dino_call`: records each call's groups as (B, H, W, dtype) and writes, for image j of a group, that image's
    value into all of its outputs."""

    def __init__(self, model):
        self.calls = []
        model._dino_call = self

    def __call__(self, groups, layers, flags):
        self.calls.append([(x.shape[0], x.shape[2], x.shape[3], x.dtype) for x, _ in groups])
        for x, (tokens, cls, prenorm) in groups:
            for j in range(x.shape[0]):
                v = float(x[j, 0, 0, 0])
                for t, dim in ((tokens, 1), (cls, 1), (prenorm, 0)):
                    if t is not None:
                        t.select(dim, j).fill_(v)


MIXED = [(98, 126), (14, 518), (42, 42), (98, 126), (126, 98), (42, 42), (70, 70), (98, 126)]


@pytest.mark.parametrize("call", ["gil", "gil_cls_reshape", "features", "forward"])
def test_one_call_per_list_in_input_order(call):
    m = _model()
    rec = _Recorder(m)
    images = _images(MIXED)
    images[4] = images[4].half()
    if call == "gil":
        out = m.get_intermediate_layers_many(images, n=2)
        assert all(len(o) == 2 for o in out)
        got = [(o[0], o[1]) for o in out]
    elif call == "gil_cls_reshape":
        out = m.get_intermediate_layers_many(images, n=[3, 11], reshape=True, return_class_token=True)
        got = [(t, c) for o in out for (t, c) in o]
        for o, (H, W) in zip(out, MIXED):
            assert o[0][0].shape == (384, H // 14, W // 14) and o[0][1].shape == (384,)
    elif call == "features":
        out = m.forward_features_many(images)
        for o, (H, W) in zip(out, MIXED):
            T = (H // 14) * (W // 14)
            assert o["x_norm_patchtokens"].shape == (T, 384) and o["x_prenorm"].shape == (T + 1, 384)
            assert o["x_norm_clstoken"].shape == (384,) and o["x_norm_regtokens"].shape == (0, 384) and o["masks"] is None
        got = [(o["x_norm_patchtokens"], o["x_norm_clstoken"], o["x_prenorm"]) for o in out]
    else:
        out = m.forward_many(images)
        assert all(o.shape == (384,) for o in out)
        got = [(o,) for o in out]
    # one engine call; one group per (H, W, dtype), its images in input order, the groups with the most token rows first
    assert len(rec.calls) == 1
    assert rec.calls[0] == [(3, 98, 126, torch.float32), (1, 126, 98, torch.float16), (1, 14, 518, torch.float32),
                            (1, 70, 70, torch.float32), (2, 42, 42, torch.float32)]
    # every output of entry i is image i's
    per_image = len(got) // len(images)
    for k, ts in enumerate(got):
        for t in ts:
            assert torch.all(t == float(k // per_image)), (k, t.flatten()[:4])


def test_group_cap_splits_a_many_shape_list():
    """More distinct shapes than a call may carry: the calls hold at most MOGE_DINO_MAX_GROUPS groups, and every image comes back
    in its place."""
    m = _model()
    rec = _Recorder(m)
    shapes = [(14 * (1 + i % 10), 14 * (1 + i // 10)) for i in range(70)]
    out = m.get_intermediate_layers_many(_images(shapes), n=1, return_class_token=True)
    assert [len(c) for c in rec.calls] == [capi.DINO_MAX_GROUPS, 70 - capi.DINO_MAX_GROUPS]
    assert sorted((H, W) for c in rec.calls for (_, H, W, _) in c) == sorted(shapes)
    for i, ((t, c),) in enumerate(out):
        assert t.shape == ((shapes[i][0] // 14) * (shapes[i][1] // 14), 384)
        assert torch.all(t == i) and torch.all(c == i)


def test_small_max_chunk_tokens_chunks_and_packs():
    m = _model()
    rec = _Recorder(m)
    m.max_chunk_tokens = 2 * 50                       # 98 x 98: 50 token rows per image, so at most 2 such images per call
    shapes = [(98, 98)] * 5 + [(42, 42)] * 3
    out = m.get_intermediate_layers_many(_images(shapes), n=1)
    for call in rec.calls:
        assert sum(B * ((H // 14) * (W // 14) + 1) for (B, H, W, _) in call) <= m.max_chunk_tokens
    assert sorted(B for call in rec.calls for (B, H, _, _) in call if H == 98) == [1, 2, 2]
    assert sum(B for call in rec.calls for (B, H, _, _) in call if H == 42) == 3
    for i, (t,) in enumerate(out):
        assert torch.all(t == i)


def test_pack_calls_cap():
    """The shared packer's unit cap on its own: at most max_units units per call, still largest first; no cap, one call."""
    m = _model()
    shapes = [(14 * (1 + i), 14) for i in range(10)]
    geometry = lambda H, W: ((H // 14, W // 14), (H // 14) * (W // 14) + 1)      # noqa: E731
    calls = m._pack_calls(_images(shapes), geometry, max_units=3)
    assert [len(c) for c in calls] == [3, 3, 3, 1]
    assert [H for c in calls for (H, _, _, _) in c] == [14 * (10 - i) for i in range(10)]
    assert len(m._pack_calls(_images(shapes), geometry)) == 1


def test_bad_arguments_raise_before_device_work():
    m = _model()                                      # on the CPU: anything past the checks raises MogeError (no CPU path)
    good = _images([(98, 98)])[0]
    with pytest.raises(TypeError, match="a list"):
        m.get_intermediate_layers_many(torch.zeros(2, 3, 98, 98))
    with pytest.raises(TypeError, match="a list"):
        m.forward_features_many((good,))
    with pytest.raises(ValueError, match=r"images\[1\] must be \(3, H, W\)"):
        m.get_intermediate_layers_many([good, torch.zeros(1, 3, 98, 98)])
    with pytest.raises(ValueError, match=r"images\[1\] must be \(3, H, W\)"):
        m.forward_many([good, torch.zeros(4, 98, 98)])
    with pytest.raises(TypeError, match=r"images\[1\] must be float32, float16 or bfloat16"):
        m.get_intermediate_layers_many([good, torch.zeros(3, 98, 98, dtype=torch.uint8)])
    with pytest.raises(AssertionError, match="height 100 is not a multiple of patch height 14"):
        m.get_intermediate_layers_many([good, torch.zeros(3, 100, 98)])
    with pytest.raises(AssertionError, match="width 100 is not a multiple"):
        m.forward_features_many([good, torch.zeros(3, 98, 100)])
    with pytest.raises(AssertionError, match="blocks found"):
        m.get_intermediate_layers_many([good], n=[12])
    with pytest.raises(AssertionError, match="only 12 / 13"):
        m.get_intermediate_layers_many([good], n=13)
    with pytest.raises(NotImplementedError, match="list.*forward_features_many"):
        m.forward_features([good[None]])
    assert m.get_intermediate_layers_many([]) == [] and m.forward_features_many([]) == [] and m.forward_many([]) == []
    assert m.get_intermediate_layers_many([good, good], n=0) == [(), ()]            # nothing asked, nothing run
    with pytest.raises(capi.MogeError, match="no CPU path"):                       # valid arguments reach the engine
        m.get_intermediate_layers_many([good])


def test_c_abi_signatures():
    for n in ("moge_dino_workspace_bytes_groups", "moge_dino_forward_groups"):
        assert n in capi.SIGNATURES and n in capi.EXPORTS
    assert [name for name, _ in capi.DinoGroup._fields_] == ["x", "x_dtype", "B", "H", "W", "out_tokens", "out_cls",
                                                             "out_prenorm"]
    assert C.sizeof(capi.DinoGroup) == 8 + 4 * 4 + 3 * 8            # x, four ints, three pointers: no padding


@pytest.mark.parametrize("n,msg", [(0, "out of range"), (capi.DINO_MAX_GROUPS + 1, "out of range"), (1, "null argument")])
def test_c_group_entries_reject_bad_calls(n, msg):
    L = capi.lib()
    groups = (capi.DinoGroup * (capi.DINO_MAX_GROUPS + 1))()
    for g in groups:
        g.B, g.H, g.W = 1, 98, 126
    lay = (C.c_int * 1)(11)
    nbytes = C.c_size_t()
    assert L.moge_dino_workspace_bytes_groups(None, groups, n, lay, 1, 1, C.byref(nbytes)) != 0
    assert msg in L.moge_last_error().decode()
    ws = torch.empty(2048, dtype=torch.uint8)
    assert L.moge_dino_forward_groups(None, groups, n, lay, 1, 1, ws.data_ptr(), ws.numel(), None) != 0
    assert msg in L.moge_last_error().decode()
    assert L.moge_dino_workspace_bytes_groups(None, groups, 1, lay, 1, 1, None) != 0
    assert "null argument" in L.moge_last_error().decode()
    assert L.moge_dino_workspace_bytes_groups(None, None, 1, lay, 1, 1, C.byref(nbytes)) != 0
    assert "null argument" in L.moge_last_error().decode()
