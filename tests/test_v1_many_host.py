"""CPU: the mixed-shape batching shared by both models' `infer_many` (bucketing by shape and dtype, chunking, packing into
engine calls), MoGe-1's `infer_many` argument checks and the C-ABI checks of the MoGe-1 group entry points (no device needed)."""
import ctypes as C

import pytest
import torch

from moge_b200 import capi
from moge_b200.configs import token_grid, v1_model_config, v1_resized_size
from moge_b200.model._engine import EngineModel


def _images(shapes, dtype=torch.float32):
    return [torch.empty(3, H, W, dtype=dtype) for H, W in shapes]


def _v2_geometry(num_tokens):
    def geometry(H, W):
        h, w = token_grid(H, W, num_tokens)
        return (h, w), h * w + 1
    return geometry


def _v1_geometry(num_tokens):
    def geometry(H, W):
        rh, rw = v1_resized_size(H, W, num_tokens)
        return (rh, rw), (rh // 14) * (rw // 14) + 1
    return geometry


def _packer(max_chunk_tokens):
    m = EngineModel()
    m.max_chunk_tokens = max_chunk_tokens
    return m


def _old_v2_calls(model, images, num_tokens):
    """MoGe-2's infer_many packing as it was written inside v2.py before the helper existed."""
    buckets = {}
    for i, im in enumerate(images):
        buckets.setdefault((int(im.shape[1]), int(im.shape[2]), im.dtype), []).append(i)
    units = []
    for (H, W, _), idx in buckets.items():
        h, w = token_grid(H, W, int(num_tokens))
        for lo, n in model._chunks(len(idx), h * w + 1):
            units.append((n * (h * w + 1), H, W, h, w, idx[lo:lo + n]))
    units.sort(key=lambda u: -u[0])
    calls, cur, cur_tok = [], [], 0
    for u in units:
        if cur and cur_tok + u[0] > model.max_chunk_tokens:
            calls.append(cur); cur, cur_tok = [], 0
        cur.append(u); cur_tok += u[0]
    if cur:
        calls.append(cur)
    return calls


# the shape sets of the MoGe-2 infer_many GPU tests, with their token counts and call bounds
V2_CASES = [
    ([(98, 196), (126, 168), (140, 140), (168, 126), (196, 98), (126, 168), (98, 196), (140, 140), (140, 140)], 130, 48 * 1370),
    ([(70 + 14 * (i % 3), 98) for i in range(7)], 60, 3 * 61),
    ([(518, 1036)] * 7 + [(518, 777)] * 7 + [(518, 518)] * 6 + [(777, 518)] * 6 + [(1036, 518)] * 6, 700, 48 * 1370),
    ([(518, 1036)] * 7 + [(518, 777)] * 7 + [(518, 518)] * 6 + [(777, 518)] * 6 + [(1036, 518)] * 6, 700, 5 * 701),
]


@pytest.mark.parametrize("shapes,num_tokens,bound", V2_CASES)
def test_v2_packs_as_before(shapes, num_tokens, bound):
    model = _packer(bound)
    images = _images(shapes)
    old = _old_v2_calls(model, images, num_tokens)
    new = model._pack_calls(images, _v2_geometry(num_tokens))
    assert [[(H, W, (h, w), idx) for (_, H, W, h, w, idx) in call] for call in old] == new


def _check_calls(model, images, geometry, calls):
    seen = []
    for call in calls:
        tokens = [len(idx) * geometry(H, W)[1] for (H, W, _, idx) in call]
        assert len(call) == 1 or sum(tokens) <= model.max_chunk_tokens, (call, tokens)
        for (H, W, geom, idx) in call:
            assert geom == geometry(H, W)[0]
            assert idx == sorted(idx)                              # a bucket keeps its images in input order
            for i in idx:
                assert tuple(images[i].shape[1:]) == (H, W)
            seen += idx
    assert sorted(seen) == list(range(len(images)))                # every image exactly once
    units = [len(idx) * geometry(H, W)[1] for call in calls for (H, W, _, idx) in call]
    assert units == sorted(units, reverse=True)                    # largest units first


@pytest.mark.parametrize("bound", [48 * 1370, 4000, 1500, 100])
def test_pack_calls_bound_cover_order(bound):
    model = _packer(bound)
    shapes = [(518, 1036), (518, 518), (1024, 768), (518, 1036), (98, 126), (518, 777), (1024, 768), (518, 518), (98, 126),
              (777, 518), (518, 1036)]
    images = _images(shapes)
    geometry = _v1_geometry(1200)
    calls = model._pack_calls(images, geometry)
    _check_calls(model, images, geometry, calls)
    if bound == 48 * 1370:
        assert len(calls) == 1 and len(calls[0]) == 6               # every shape group in one call


def test_pack_calls_separates_dtypes():
    model = _packer(48 * 1370)
    images = _images([(98, 126)] * 2) + _images([(98, 126)], torch.float16) + _images([(98, 126)])
    calls = model._pack_calls(images, _v1_geometry(120))
    assert len(calls) == 1
    assert sorted(idx for (_, _, _, idx) in calls[0]) == [[0, 1, 3], [2]]


@pytest.mark.parametrize("bad", [torch.empty(1, 3, 28, 28), torch.empty(4, 28, 28), torch.empty(28, 28)])
def test_v1_infer_many_rejects_non_chw_before_the_device(bad):
    from moge.model.v1 import MoGeModel
    m = MoGeModel(**v1_model_config("vits"))         # on the CPU without weights: anything past the checks raises MogeError
    with pytest.raises(ValueError, match=r"images\[1\]"):
        m.infer_many([torch.empty(3, 28, 28), bad])
    with pytest.raises(NotImplementedError):
        m.infer_many([torch.empty(3, 28, 28)], use_fp16=False)


def test_v1_group_struct_matches_header():
    fields = [name for name, _ in capi.V1Group._fields_]
    assert fields == ["image", "image_dtype", "B", "H", "W", "rh", "rw", "points", "mask"]
    assert C.sizeof(capi.V1Group) == 8 + 4 + 5 * 4 + 8 + 8       # image, dtype, five ints, two pointers: no padding


@pytest.mark.parametrize("n,msg", [(0, "out of range"), (65, "out of range"), (1, "null argument")])
def test_v1_group_entries_reject_bad_calls(n, msg):
    L = capi.lib()
    groups = (capi.V1Group * 65)()
    for g in groups:
        g.B, g.H, g.W, g.rh, g.rw = 1, 98, 126, 98, 126
    nbytes = C.c_size_t()
    assert L.moge_v1_workspace_bytes_groups(None, groups, n, C.byref(nbytes)) != 0
    assert msg in L.moge_last_error().decode()
    ws = torch.empty(2048, dtype=torch.uint8)
    assert L.moge_v1_forward_groups(None, groups, n, ws.data_ptr(), ws.numel(), None) != 0
    assert msg in L.moge_last_error().decode()
    assert L.moge_v1_workspace_bytes_groups(None, groups, 1, None) != 0
    assert L.moge_v1_forward_groups(None, None, 1, None, 0, None) != 0
    assert "null argument" in L.moge_last_error().decode()
