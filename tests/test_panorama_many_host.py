"""Mixed-size panorama inference, host side (no GPU): infer_panoramas_many's argument checks fail with MogeError before any
device work and name the offending panorama, the merge schedule lines up pyramids of different depths at their finest level,
and the `_groups` C entry points are in the ABI table and reject null arguments and out-of-range counts without a device."""
import ctypes as C

import pytest
import torch

from moge_b200 import capi
from moge_b200 import panorama as P
from moge_b200.capi import MogeError


class _NoModel:
    """A model that fails the test if the views ever reach it."""
    def infer(self, *args, **kwargs):
        raise AssertionError("argument errors must be raised before the view pass")


def _img(H=64, W=128, dtype=torch.uint8):
    return torch.zeros(H, W, 3, dtype=dtype)


@pytest.mark.parametrize("images,msg", [
    (torch.zeros(2, 64, 128, 3, dtype=torch.uint8), "must be a list"),
    ([], r"a list of 0 panoramas is outside \[1, 64\]"),
    ([_img(2, 2)] * 65, r"a list of 65 panoramas is outside \[1, 64\]"),
    ([_img(dtype=torch.float32)], "panorama 0 must be a .*uint8"),
    ([_img()[..., :2]], r"panorama 0 must be a \(H, W, 3\)"),
    ([_img()[0]], r"panorama 0 must be a \(H, W, 3\)"),
    ([_img(), "not a tensor"], "panorama 0 operates on CUDA"),       # the first offending panorama is named
    ([_img()], "panorama 0 operates on CUDA tensors only"),
])
def test_infer_panoramas_many_checks(images, msg):
    with pytest.raises(MogeError, match=msg):
        P.infer_panoramas_many(_NoModel(), images)


def test_infer_panoramas_many_batch_size_checked_first():
    with pytest.raises(MogeError, match="batch_size 0 must be positive"):
        P.infer_panoramas_many(_NoModel(), "not a list", batch_size=0)


def test_check_list_names_the_index():
    # the element checks run in input order; a CPU model device is ignored
    with pytest.raises(MogeError, match="infer_panoramas_many: panorama 0 operates on CUDA"):
        P._check_list("infer_panoramas_many", [_img(), _img(dtype=torch.int16)], None)
    with pytest.raises(MogeError, match="panorama 0 must be"):
        P._check_list("infer_panoramas_many", [_img(dtype=torch.int16), _img()], None)


def test_schedule_lines_up_pyramids_at_the_finest_level():
    sizes = [(1920, 960), (1536, 768), (200, 100), (1000, 300), (1920, 960)]
    levels, launches = P._schedule(sizes)
    assert levels[0] == [(240, 120), (480, 240), (960, 480), (1920, 960)]
    assert levels[1] == [(192, 96), (384, 192), (768, 384), (1536, 768)]
    assert levels[2] == [(200, 100)]                                       # under 256 px: one level
    assert levels[3] == [(250, 75), (500, 150), (1000, 300)]               # not 2:1
    assert launches == [
        [(0, 0), (1, 0), (4, 0)],
        [(0, 1), (1, 1), (3, 0), (4, 1)],
        [(0, 2), (1, 2), (3, 1), (4, 2)],
        [(0, 3), (1, 3), (2, 0), (3, 2), (4, 3)],
    ]
    # each panorama sees its own levels in order, in consecutive launches, and every panorama is in the last launch
    for i, lv in enumerate(levels):
        seen = [(k, j) for k, members in enumerate(launches) for (m, j) in members if m == i]
        assert [j for _, j in seen] == list(range(len(lv)))
        assert [k for k, _ in seen] == list(range(len(launches) - len(lv), len(launches)))


def test_schedule_one_size_is_the_plain_pyramid():
    levels, launches = P._schedule([(1920, 960)] * 3)
    assert all(lv == P._levels(1920, 960) for lv in levels)
    assert launches == [[(i, k) for i in range(3)] for k in range(4)]
    levels, launches = P._schedule([(128, 64)])
    assert levels == [[(128, 64)]] and launches == [[(0, 0)]]


GROUPS = ("moge_panorama_split_groups", "moge_panorama_workspace_bytes_groups", "moge_panorama_rhs_groups",
          "moge_panorama_lsmr_groups", "moge_panorama_resize_groups", "moge_panorama_finish_groups")


def test_group_entry_points_registered():
    for name in GROUPS:
        assert name in capi.SIGNATURES and name in capi.EXPORTS
    assert [f for f, _ in capi.PanoramaSplit._fields_] == ["image", "H", "W", "view0"]
    assert [f for f, _ in capi.PanoramaLevel._fields_] == ["h", "w", "view0", "directions", "b", "row_mask", "pano_mask", "init",
                                                           "depth", "stats"]
    assert C.sizeof(capi.PanoramaLevel) == 4 * 4 + 7 * 8                   # three ints, padding, seven pointers
    assert C.sizeof(capi.PanoramaResize) == 8 + 4 * 4 + 8
    assert C.sizeof(capi.PanoramaFinish) == 2 * 8 + 4 * 4 + 3 * 8


def _error(rc):
    assert rc != 0
    return capi.lib().moge_last_error().decode()


def _levels_array(sizes, **ptrs):
    lv = (capi.PanoramaLevel * max(len(sizes), 1))()
    for k, (h, w) in enumerate(sizes):
        lv[k].h, lv[k].w, lv[k].view0 = h, w, 12 * k
        for name, value in ptrs.items():
            setattr(lv[k], name, value)
    return lv


@pytest.mark.parametrize("n", [0, 65])
def test_group_counts_rejected_without_device(n):
    L = capi.lib()
    lv = (capi.PanoramaLevel * 66)()
    for k in range(66):
        lv[k].h, lv[k].w = 8, 16
    nbytes = C.c_size_t()
    want = rf"a batch of {n} panoramas is outside \[1, 64\]"
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_workspace_bytes_groups(lv, n, 12, C.byref(nbytes))).match(want)
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_lsmr_groups(lv, n, 256, 256, None)).match(want)
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_rhs_groups(8, 1, 8, 12, 4, 4, None, lv, n, 256, 256, None)).match(want)
    splits = (capi.PanoramaSplit * 66)()
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_split_groups(splits, n, None, 12, 8, 4, 8, None, None)).match(want)
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_resize_groups((capi.PanoramaResize * 66)(), n, None)).match(want)
    assert pytest.raises(MogeError, capi.check, L.moge_panorama_finish_groups((capi.PanoramaFinish * 66)(), n, None)).match(want)


def test_group_null_arguments_rejected_without_device():
    L = capi.lib()
    assert _error(L.moge_panorama_lsmr_groups(None, 1, 256, 256, None)) == "null argument"
    assert _error(L.moge_panorama_split_groups(None, 1, None, 12, 8, 4, 8, None, None)) == "null argument"
    assert _error(L.moge_panorama_resize_groups(None, 1, None)) == "null argument"
    assert _error(L.moge_panorama_finish_groups(None, 1, None)) == "null argument"
    # a null pointer of one entry names that entry
    lv = _levels_array([(8, 16), (4, 8)], b=8, row_mask=8, depth=8, stats=8)
    lv[1].depth = None
    assert _error(L.moge_panorama_lsmr_groups(lv, 2, 256, 256, None)) == "panorama_lsmr_groups: panorama 1: null argument"
    lv = _levels_array([(8, 16), (4, 8)], directions=8, b=8, row_mask=8, pano_mask=8)
    lv[0].pano_mask = None
    assert _error(L.moge_panorama_rhs_groups(8, 1, 8, 12, 4, 4, None, lv, 2, 256, 256, None)) \
        == "panorama_rhs_groups: panorama 0: null argument"
    lv = _levels_array([(8, 16), (1, 8)], b=8, row_mask=8, depth=8, stats=8)
    assert "panorama 1: a 1 x 8 map is too small" in _error(L.moge_panorama_lsmr_groups(lv, 2, 256, 256, None))


def test_group_workspace_bytes_grow_with_entries():
    L = capi.lib()

    def nbytes(sizes):
        out = C.c_size_t()
        capi.check(L.moge_panorama_workspace_bytes_groups(_levels_array(sizes), len(sizes), 12, C.byref(out)))
        return out.value

    mixed = [(960, 1920), (384, 768), (100, 200)]
    assert nbytes(mixed) > nbytes(mixed[1:]) > nbytes(mixed[2:]) > 0
    # a call whose entries are each no larger fits in the workspace: every coarser level of a pyramid does
    assert nbytes([(480, 960), (192, 384), (100, 200)]) <= nbytes(mixed)
