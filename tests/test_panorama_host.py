"""Panorama inference, host side (no GPU): the golden file, the utils3d restatement's cameras, the drop-in's import and the
argument checks that fail before any device work."""
import os

import cv2
import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "panorama.pt")


def _gold():
    return torch.load(GOLDEN, weights_only=False)


def test_golden_split_is_cv2_remap():
    """The golden views are cv2.remap of the seeded panoramas at the reference's pixel coordinates, rebuilt from the utils3d
    restatement and the drop-in's spherical-uv function."""
    from moge_b200.panorama import directions_to_spherical_uv
    from moge_b200.synthetic import array_digest, synthetic_panorama
    from oracle.utils3d_panorama import unproject_cv, uv_map, uv_to_pixel
    g = _gold()
    extr, intr = g["extrinsics"].numpy(), g["intrinsics"].numpy()
    assert extr.dtype == np.float32 and extr.shape == (12, 4, 4) and intr.shape == (12, 3, 3)
    for case in g["split"]:
        img, res = synthetic_panorama(case["H"], case["W"], case["seed"]), case["resolution"]
        uv = uv_map((res, res))
        views = []
        for k in range(12):
            rays = unproject_cv(uv, np.ones_like(uv[..., 0]), extrinsics=extr[k], intrinsics=intr[k])
            px = uv_to_pixel(directions_to_spherical_uv(rays), img.shape[:2]).astype(np.float32)
            views.append(cv2.remap(img, px[..., 0], px[..., 1], interpolation=cv2.INTER_LINEAR))
        views = np.stack(views)
        if "views" in case:
            np.testing.assert_array_equal(views, case["views"].numpy())
        assert array_digest(views) == case["views_sha256"]


def test_golden_room_inputs_regenerate():
    from moge_b200.synthetic import array_digest, synthetic_room_views
    room = _gold()["room"]
    dist, masks = synthetic_room_views(room["resolution"], room["seed"])
    assert dist.dtype == np.float32 and masks.dtype == bool and dist.shape == (12, 96, 96)
    assert array_digest(dist, masks) == room["inputs_sha256"]


def test_cameras_match_restatement_and_are_look_at():
    from moge_b200.panorama import get_panorama_cameras
    from oracle.utils3d_panorama import create_icosahedron_mesh, extrinsics_look_at, intrinsics_from_fov
    g = _gold()
    extr, intr = get_panorama_cameras()
    np.testing.assert_array_equal(extr, g["extrinsics"].numpy())
    np.testing.assert_array_equal(np.stack(intr), g["intrinsics"].numpy())
    vertices, faces = create_icosahedron_mesh()
    assert vertices.shape == (12, 3) and faces.shape == (20, 3)
    np.testing.assert_array_equal(extrinsics_look_at([0, 0, 0], vertices, [0, 0, 1]).astype(np.float32), extr)
    np.testing.assert_array_equal(intrinsics_from_fov(fov_x=np.deg2rad(90), fov_y=np.deg2rad(90)), intr[0])
    R = extr[:, :3, :3].astype(np.float64)
    np.testing.assert_allclose(R @ R.transpose(0, 2, 1), np.broadcast_to(np.eye(3), R.shape), atol=1e-6)
    fwd = R[:, 2]
    np.testing.assert_allclose(np.linalg.norm(fwd, axis=-1), 1, atol=1e-6)
    v = vertices / np.linalg.norm(vertices, axis=-1, keepdims=True)
    np.testing.assert_allclose(fwd, v, atol=1e-6)              # each camera looks at its vertex
    assert len({tuple(np.round(f, 4)) for f in fwd}) == 12
    np.testing.assert_array_equal(extr[:, :3, 3], 0)


def test_uv_map_matches_linspace_restatement():
    from moge_b200.panorama import uv_map
    from oracle.utils3d_panorama import uv_map as ref_uv_map
    for h, w in ((1, 512), (75, 150), (960, 1920), (127, 251)):
        np.testing.assert_array_equal(uv_map(h, w), ref_uv_map(h, w))
        np.testing.assert_array_equal(uv_map(h, w), ref_uv_map((h, w)))


def test_dropin_imports():
    import moge.utils.panorama as p
    for name in ("get_panorama_cameras", "spherical_uv_to_directions", "directions_to_spherical_uv", "split_panorama_image",
                 "merge_panorama_depth"):
        assert callable(getattr(p, name))
    assert not hasattr(p, "poisson_equation") and not hasattr(p, "grad_equation")
    uv = np.random.RandomState(0).uniform(0.01, 0.99, (50, 2))
    np.testing.assert_allclose(p.directions_to_spherical_uv(p.spherical_uv_to_directions(uv)), uv, atol=1e-12)


def test_golden_levels_are_consistent():
    from moge_b200.panorama import num_rows
    g = _gold()
    for case in g["merge"]:
        for lv in case["levels"]:
            h, w = lv["height"], lv["width"]
            assert lv["rows"] == num_rows(h, w)
            rm = np.unpackbits(lv["row_mask"].numpy())[:lv["rows"]].astype(bool)
            if "b" in lv:
                assert lv["b"].numel() == rm.sum()
            assert lv["istop"] in (1, 2, 3, 4, 5, 6, 7) and lv["itn"] > 0
        assert case["sensitivity"] > 0


def test_argument_checks_without_device():
    from moge_b200 import panorama as P
    from moge_b200.capi import MogeError
    img = torch.zeros(64, 128, 3, dtype=torch.uint8)
    with pytest.raises(MogeError, match="CUDA"):
        P.split_panorama(img)
    with pytest.raises(MogeError, match="uint8"):
        P.split_panorama(img.float())
    with pytest.raises(MogeError, match="uint8"):
        P.split_panorama(img[..., :2])
    with pytest.raises(MogeError, match="outside"):
        P.split_panorama(torch.zeros(1, 128, 3, dtype=torch.uint8))
    dist = torch.ones(12, 8, 8)
    with pytest.raises(MogeError, match="CUDA"):
        P.merge_panorama(64, 32, dist, torch.ones(12, 8, 8, dtype=torch.bool))
    with pytest.raises(MogeError, match="mask"):
        P.merge_panorama(64, 32, dist, torch.ones(12, 8, 7, dtype=torch.bool))
    with pytest.raises(MogeError, match="float32"):
        P.merge_panorama(64, 32, dist.double(), torch.ones(12, 8, 8, dtype=torch.bool))
    with pytest.raises(MogeError, match="outside"):
        P.merge_panorama(1, 32, dist, torch.ones(12, 8, 8, dtype=torch.bool))
    with pytest.raises(MogeError, match="views"):
        P._cameras(np.zeros((21, 4, 4), np.float32), np.zeros((21, 3, 3)))
    with pytest.raises(MogeError, match="intrinsics"):
        P._cameras(np.zeros((12, 4, 4), np.float32), np.zeros((11, 3, 3)))
    with pytest.raises(MogeError, match="batch_size"):
        P.infer_panorama(None, img, batch_size=0)
