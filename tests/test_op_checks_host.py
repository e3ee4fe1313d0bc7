"""The argument checks of the op libraries' C entry points (align, metrics, mesh, panorama, losses): out-of-range batches, sizes
and counts, null arguments, and undersized or misaligned workspaces each return -1 with the operation's name and the reason in
moge_last_error().  Every case fails in a check that runs before the device check and any launch (the pointers are stand-ins),
except the align workspace cases: align sizes its workspace from the device, so without one they fail at the device check."""
import ctypes as C

import pytest
import torch

from moge_b200 import capi

L = capi.lib()
HAS_DEVICE = torch.cuda.is_available()
BIG = 1 << 40                 # workspace bytes: enough for every case below
NB = C.c_size_t()
NOBYTES = C.POINTER(C.c_size_t)()
P = 8                         # a non-null stand-in pointer; never reaches a launch


def camera():
    c = (capi.PanoramaCamera * 1)()
    c[0].fx = c[0].fy = 1.0
    return c


def split():
    e = (capi.PanoramaSplit * 1)()
    e[0].image, e[0].H, e[0].W = P, 8, 8
    return e


def level(h=8, w=8, **ptrs):
    """One panorama's h x w merge level; every pointer but init is the stand-in unless `ptrs` gives it."""
    lv = (capi.PanoramaLevel * 1)()
    lv[0].h, lv[0].w = h, w
    for name in ("directions", "b", "row_mask", "pano_mask", "depth", "stats"):
        setattr(lv[0], name, ptrs.get(name, P))
    return lv


def resize():
    m = (capi.PanoramaResize * 1)()
    m[0].src, m[0].h, m[0].w, m[0].H, m[0].W, m[0].dst = P, 8, 8, 16, 16, P
    return m


def maps(kind=capi.MESH_F32, channels=1):
    m = (capi.MeshMap * 1)()
    m[0].src, m[0].kind, m[0].channels, m[0].dst = P, kind, channels, P
    return m


# (operation named in the message, call, message substring)
CASES = {
    # align
    "align_bytes_null": ("", lambda: L.moge_align_workspace_bytes(0, 0, 1, 8, NOBYTES), "null argument"),
    "align_batch": ("align", lambda: L.moge_align_workspace_bytes(capi.ALIGN_PLAIN, 1, 0, 8, C.byref(NB)), "batch must be positive"),
    "align_mode": ("align", lambda: L.moge_align_workspace_bytes(7, 1, 1, 8, C.byref(NB)), "unknown mode"),
    "align_plain_n": ("align", lambda: L.moge_align_workspace_bytes(capi.ALIGN_PLAIN, 1, 1, 12289, C.byref(NB)), "outside"),
    "align_anchored_n": ("align", lambda: L.moge_align_workspace_bytes(capi.ANCHOR_DEPTH, 1, 1, 4097, C.byref(NB)), "outside"),
    "align_null": ("", lambda: L.moge_align(P, None, P, P, 0, 1, 8, P, P, P, P, BIG, None), "null argument"),
    "align_anchored_mode": ("align_anchored", lambda: L.moge_align_anchored(P, P, P, capi.ALIGN_PLAIN, 1.0, 1, 8, P, P, P, P, BIG, None),
                            "mode must be one of"),
    "lstsq_shape": ("align_affine_lstsq", lambda: L.moge_align_affine_lstsq(P, P, None, 0, 8, P, P, None), "bad shape"),
    "lstsq_batch": ("align_affine_lstsq", lambda: L.moge_align_affine_lstsq(P, P, None, 1 << 31, 8, P, P, None), "too large"),
    # metrics
    "metrics_batch": ("metrics", lambda: L.moge_metrics_workspace_bytes(65536, 8, 8, 0, C.byref(NB)), "outside"),
    "metrics_size": ("metrics", lambda: L.moge_metrics_workspace_bytes(1, 0, 8, 0, C.byref(NB)), "size"),
    "metrics_too_large": ("metrics", lambda: L.moge_metrics_workspace_bytes(1, 40000, 30000, 0, C.byref(NB)), "too large"),
    "metrics_segments": ("metrics", lambda: L.moge_metrics_workspace_bytes(1, 8, 8, 257, C.byref(NB)), "outside"),
    "metrics_resize_null": ("", lambda: L.moge_metrics_resize(None, 1, 8, 8, 4, 4, P, P, P, P, P, None), "null argument"),
    "metrics_resize_target": ("masked_nearest_resize", lambda: L.moge_metrics_resize(P, 1, 8, 8, 0, 4, P, P, P, P, P, None),
                              "bad target size"),
    "metrics_stats_slots": ("metrics_stats", lambda: L.moge_metrics_stats(P, P, P, None, 0, P, P, P, 300, 1, 8, 8, P, P, P, BIG, None),
                            "outside"),
    "metrics_stats_ws_small": ("metrics_stats", lambda: L.moge_metrics_stats(P, P, P, P, 0, None, None, None, 0, 1, 8, 8, P, None, 256,
                                                                             16, None),
                                     "bytes needed"),
    "metrics_stats_ws_null": ("metrics_stats", lambda: L.moge_metrics_stats(P, P, P, P, 0, None, None, None, 0, 1, 8, 8, P, None, None,
                                                                            BIG, None), "bytes needed"),
    "metrics_stats_ws_align": ("metrics_stats", lambda: L.moge_metrics_stats(P, P, P, P, 0, None, None, None, 0, 1, 8, 8, P, None, 264,
                                                                             BIG, None), "256-byte aligned"),
    "metrics_eval_variants": ("metrics_eval", lambda: L.moge_metrics_eval(P, P, P, (capi.MetricVariant * 1)(), 9, None, None, None, None,
                                                                          0, None, None, 1, 8, 8, P, 40, P, BIG, None), "outside"),
    "metrics_eval_ws_small": ("metrics_eval", lambda: L.moge_metrics_eval(P, P, P, None, 0, None, None, None, None, 0, None, None, 1, 8, 8,
                                                                          P, 40, 256, 16, None), "bytes needed"),
    "metrics_eval_ws_align": ("metrics_eval", lambda: L.moge_metrics_eval(P, P, P, None, 0, None, None, None, None, 0, None, None, 1, 8, 8,
                                                                          P, 40, 264, BIG, None), "256-byte aligned"),
    # mesh
    "mesh_batch": ("mesh", lambda: L.moge_mesh_workspace_bytes(0, 8, 8, C.byref(NB)), "outside"),
    "mesh_size": ("mesh", lambda: L.moge_mesh_workspace_bytes(1, 8, -1, C.byref(NB)), "size"),
    "mesh_too_large": ("mesh", lambda: L.moge_mesh_workspace_bytes(1, 40000, 30000, C.byref(NB)), "too large"),
    "mesh_bytes_null": ("", lambda: L.moge_mesh_workspace_bytes(1, 8, 8, NOBYTES), "null argument"),
    "depth_edge_null": ("", lambda: L.moge_depth_edge(None, None, None, 1, 8, 8, 3, None, None, P, None), "null argument"),
    "depth_edge_kernel": ("depth_map_edge", lambda: L.moge_depth_edge(P, None, None, 1, 8, 8, 4, None, None, P, None), "kernel_size"),
    "normal_map_batch": ("point_map_to_normal_map", lambda: L.moge_normal_map(P, None, 70000, 8, 8, P, None, None), "outside"),
    "normal_edge_rows": ("normal_map_edge", lambda: L.moge_normal_edge(P, None, None, None, 1, 65535 * 32 + 1, 1, 3, 0.1, P, None, None),
                         "rows"),
    "mesh_count_ws_small": ("mesh_count", lambda: L.moge_mesh_count(None, 1, 8, 8, P, 256, 16, None), "bytes needed"),
    "mesh_count_ws_align": ("mesh_count", lambda: L.moge_mesh_count(None, 1, 8, 8, P, 264, BIG, None), "256-byte aligned"),
    "mesh_build_maps": ("mesh_build", lambda: L.moge_mesh_build(None, 1, 8, 8, 1, maps(), 9, P, P, 256, BIG, None), "outside"),
    "mesh_build_channels": ("mesh_build", lambda: L.moge_mesh_build(None, 1, 8, 8, 1, maps(channels=5), 1, P, P, 256, BIG, None),
                            "channels"),
    "mesh_build_ws_small": ("mesh_build", lambda: L.moge_mesh_build(None, 1, 8, 8, 1, maps(), 1, P, P, 256, 16, None), "bytes needed"),
    "mesh_build_ws_align": ("mesh_build", lambda: L.moge_mesh_build(None, 1, 8, 8, 1, maps(), 1, P, P, 264, BIG, None),
                            "256-byte aligned"),
    # panorama: the `_groups` entry points, with one entry except for the count
    "panorama_groups_count": ("panorama_workspace_bytes_groups",
                              lambda: L.moge_panorama_workspace_bytes_groups(level(), 65, 1, C.byref(NB)), "batch of 65 panoramas"),
    "panorama_groups_views": ("panorama_workspace_bytes_groups",
                              lambda: L.moge_panorama_workspace_bytes_groups(level(), 1, 21, C.byref(NB)), "outside"),
    "panorama_groups_small": ("panorama_workspace_bytes_groups",
                              lambda: L.moge_panorama_workspace_bytes_groups(level(1, 8), 1, 1, C.byref(NB)), "too small"),
    "panorama_groups_too_large": ("panorama_workspace_bytes_groups",
                                  lambda: L.moge_panorama_workspace_bytes_groups(level(40000, 30000), 1, 1, C.byref(NB)), "too large"),
    "panorama_groups_split_res": ("panorama_split_groups",
                                  lambda: L.moge_panorama_split_groups(split(), 1, camera(), 1, P, 0, P, None, None), "outside"),
    "panorama_groups_split_views": ("panorama_split_groups",
                                    lambda: L.moge_panorama_split_groups(split(), 1, camera(), 0, P, 8, P, None, None), "outside"),
    "panorama_groups_split_cams": ("panorama_split_groups", lambda: L.moge_panorama_split_groups(split(), 1, None, 1, P, 8, P, None, None),
                                   "null cameras"),
    "panorama_groups_rhs_null": ("panorama_rhs_groups",
                                 lambda: L.moge_panorama_rhs_groups(P, 1, P, 1, 8, 8, camera(), level(b=None), 1, 256, BIG, None),
                                 "null argument"),
    "panorama_groups_rhs_ws_small": ("panorama_rhs_groups",
                                     lambda: L.moge_panorama_rhs_groups(P, 1, P, 1, 8, 8, camera(), level(), 1, 256, 16, None),
                                     "bytes needed"),
    "panorama_groups_rhs_ws_align": ("panorama_rhs_groups",
                                     lambda: L.moge_panorama_rhs_groups(P, 1, P, 1, 8, 8, camera(), level(), 1, 264, BIG, None),
                                     "256-byte aligned"),
    "panorama_groups_lsmr_ws_small": ("panorama_lsmr_groups", lambda: L.moge_panorama_lsmr_groups(level(), 1, 256, 16, None),
                                      "bytes needed"),
    "panorama_groups_lsmr_ws_align": ("panorama_lsmr_groups", lambda: L.moge_panorama_lsmr_groups(level(), 1, 264, BIG, None),
                                      "256-byte aligned"),
    # losses
    "loss_batch": ("loss", lambda: L.moge_loss_workspace_bytes(0, 8, 8, C.byref(NB)), "outside"),
    "loss_size": ("loss", lambda: L.moge_loss_workspace_bytes(1, 8, 0, C.byref(NB)), "size"),
    "loss_too_large": ("loss", lambda: L.moge_loss_workspace_bytes(1, 40000, 30000, C.byref(NB)), "too large"),
    "loss_mask_null": ("", lambda: L.moge_loss_mask(capi.LOSS_MASK_L2, P, None, P, 1, 8, 8, None, None, P, 256, BIG, None),
                       "null argument"),
    "loss_mask_kind": ("loss_mask", lambda: L.moge_loss_mask(9, P, P, P, 1, 8, 8, None, None, P, 256, BIG, None), "unknown kind"),
    "loss_stencil_batch": ("loss_stencil", lambda: L.moge_loss_stencil(capi.LOSS_EDGE, P, P, 65536, 8, 8, None, None, P, 256, BIG, None),
                           "outside"),
    "loss_global_pass": ("loss_global", lambda: L.moge_loss_global(P, P, P, 0.0, 3, 1, 8, 8, None, P, 256, BIG, None), "unknown pass"),
    "loss_global_beta": ("loss_global", lambda: L.moge_loss_global(P, P, P, -1.0, 1, 1, 8, 8, None, P, 256, BIG, None), "beta"),
    "loss_mask_ws_small": ("loss_mask", lambda: L.moge_loss_mask(capi.LOSS_MASK_L2, P, P, P, 1, 8, 8, None, None, P, 256, 16, None),
                           "bytes needed"),
    "loss_stencil_ws_null": ("loss_stencil", lambda: L.moge_loss_stencil(capi.LOSS_NORMAL, P, P, 1, 8, 8, None, None, P, None, BIG, None),
                             "bytes needed"),
    "loss_global_sums_null": ("loss_global", lambda: L.moge_loss_global(P, P, P, 0.0, 1, 1, 8, 8, None, None, 256, BIG, None), "null sums"),
    "loss_global_ws_align": ("loss_global", lambda: L.moge_loss_global(P, P, P, 0.0, 1, 1, 8, 8, None, P, 264, BIG, None),
                             "256-byte aligned"),
}

# align derives its workspace size from the device's SM count, so its workspace checks come after the device check
ALIGN_WS = {
    "align_ws_small": ("align", lambda: L.moge_align(P, P, P, P, 0, 1, 8, P, P, P, 256, 16, None), "bytes needed"),
    "align_ws_null": ("align", lambda: L.moge_align(P, P, P, P, 0, 1, 8, P, P, P, None, BIG, None), "bytes needed"),
    "align_ws_align": ("align", lambda: L.moge_align(P, P, P, P, 0, 1, 8, P, P, P, 264, BIG, None), "256-byte aligned"),
    "align_anchored_ws_small": ("align", lambda: L.moge_align_anchored(P, P, P, capi.ANCHOR_DEPTH, -1.0, 1, 8, P, P, P, 256, 16, None),
                                "bytes needed"),
    "align_anchored_ws_align": ("align", lambda: L.moge_align_anchored(P, P, P, capi.ANCHOR_DEPTH, -1.0, 1, 8, P, P, P, 264, BIG, None),
                                "256-byte aligned"),
}

# calls whose arguments pass every check: without a device they stop at the device check
NO_DEVICE = {
    "align": ("align", lambda: L.moge_align_workspace_bytes(capi.ALIGN_PLAIN, 1, 1, 8, C.byref(NB))),
    "align_affine_lstsq": ("align_affine_lstsq", lambda: L.moge_align_affine_lstsq(P, P, None, 1, 8, P, P, None)),
    "masked_nearest_resize": ("masked_nearest_resize", lambda: L.moge_metrics_resize(P, 1, 8, 8, 4, 4, P, P, P, P, P, None)),
    "mesh_count": ("mesh_count", lambda: L.moge_mesh_count(None, 1, 8, 8, P, 256, BIG, None)),
    "panorama_groups_resize": ("panorama_resize_groups", lambda: L.moge_panorama_resize_groups(resize(), 1, None)),
    "loss_mask": ("loss_mask", lambda: L.moge_loss_mask(capi.LOSS_MASK_L2, P, P, P, 1, 8, 8, None, None, P, 256, BIG, None)),
}


def expect_error(what, call, substring):
    assert call() == -1
    msg = L.moge_last_error().decode()
    assert msg.startswith(what + ": " if what else "null argument"), msg
    assert substring in msg, msg


@pytest.mark.parametrize("case", sorted(CASES))
def test_bad_arguments_are_rejected_before_any_launch(case):
    expect_error(*CASES[case])


@pytest.mark.parametrize("case", sorted(ALIGN_WS))
def test_align_workspace(case):
    what, call, substring = ALIGN_WS[case]
    expect_error(what, call, substring if HAS_DEVICE else "no CPU fallback")


# the library's own device query (align's workspace size needs the SM count) must agree that there is no device
@pytest.mark.skipif(HAS_DEVICE or L.moge_align_workspace_bytes(capi.ALIGN_PLAIN, 1, 1, 8, C.byref(C.c_size_t())) == 0,
                    reason="the no-device message needs a machine without a CUDA device")
@pytest.mark.parametrize("case", sorted(NO_DEVICE))
def test_no_device(case):
    expect_error(*NO_DEVICE[case], "no CUDA device: moge_b200 has no CPU fallback")
