"""Colourisation and CLI on the host: the Spectral table and matplotlib's index rules (oracle/vis_port.py), the quantile arithmetic
the kernels use against np.nanquantile, the CLI's planning (files, paths, --resize, fov.json, usage errors) and the C entry
points' argument checks."""
import ctypes as C
import json
import warnings

import numpy as np
import pytest
import torch
from click.testing import CliRunner

from moge_b200 import capi, cli, vis
from oracle import utils3d_panorama, vis_port


def test_table():
    lut = vis_port.lut_u8()
    assert lut.shape == (256, 3) and lut.dtype == np.uint8
    assert np.array_equal(vis.spectral_table(), lut)
    assert tuple(lut[0]) == vis_port.SPECTRAL_COLORS[0] and tuple(lut[-1]) == vis_port.SPECTRAL_COLORS[-1]
    # each of the 10 segments between control colours is monotone in every channel
    knots = np.round(np.linspace(0, 255, 11)).astype(int)
    for a, b in zip(knots[:-1], knots[1:]):
        seg = lut[a:b + 1].astype(int)
        for c in range(3):
            d = np.diff(seg[:, c])
            assert (d >= 0).all() or (d <= 0).all(), (a, b, c)


def test_index_rules():
    below_one = np.nextafter(np.float32(1), np.float32(0))
    x = np.array([0.0, 1.0, below_one, 0.5, -0.0, -1e-7, -5.0, np.inf, -np.inf, np.nan, 1.0 + 1e-6, 0.99999], dtype=np.float32)
    idx = vis_port.colormap_index(x)
    assert list(idx) == [0, 255, 255, 128, 0, 256, 256, 257, 256, 258, 257, 255]
    rgba = vis_port.spectral(x)
    assert np.array_equal(rgba[5], rgba[0]) and np.array_equal(rgba[7], rgba[1]) and (rgba[9] == 0).all()


def test_restatement_against_matplotlib():
    matplotlib = pytest.importorskip("matplotlib")
    cmap = matplotlib.colormaps["Spectral"]
    x = np.concatenate([np.linspace(-0.1, 1.1, 5001, dtype=np.float32), np.array([np.nan, np.inf, -np.inf, 1.0], np.float32)])
    assert np.array_equal(cmap(x), vis_port.spectral(x))
    assert np.array_equal((cmap(np.arange(256) / 255)[:, :3].clip(0, 1) * 255).astype(np.uint8), vis.spectral_table()[np.arange(256)])


@pytest.mark.parametrize("seed", range(6))
def test_quantile_arithmetic_matches_nanquantile(seed):
    rng = np.random.default_rng(seed)
    n = [1, 2, 57, 1000, 4097, 1 << 17][seed]
    v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4)).astype(np.float32)
    v[rng.random(n) < 0.1] = np.nan
    if seed % 2:
        v[rng.random(n) < 0.05] = np.inf
        v[:: 7] = v[0]                                        # ties
    valid = np.sort(v[~np.isnan(v)])
    for q in (0.0, 0.001, 0.5, 0.99, 0.999, 1.0):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = np.nanquantile(v, q)
            got = vis_port.nanquantile_from_sorted(valid, q)
        assert np.array_equal(np.float32(want), got, equal_nan=True), (n, q, want, got)


# ------------------------------------------------------------------------------------------------------------ CLI planning
def test_image_list_and_output_paths(tmp_path):
    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    for name in ("b.jpg", "a.PNG", "sub/c.jpeg", "notes.txt", "d.gif"):
        (src / name).write_bytes(b"x")
    paths = cli.list_images(src)
    assert [p.relative_to(src).as_posix() for p in paths] == ["a.PNG", "b.jpg", "sub/c.jpeg"]
    assert cli.save_dir("out", src, src / "sub" / "c.jpeg").as_posix() == "out/sub/c"
    assert cli.save_dir("out", src / "b.jpg", src / "b.jpg").as_posix() == "out/b"
    (tmp_path / "empty").mkdir()
    with pytest.raises(FileNotFoundError):
        cli.list_images(tmp_path / "empty")


def test_output_files():
    assert cli.output_files(True, True, True, normal=True) == ["image.jpg", "depth_vis.png", "depth.exr", "mask.png", "points.exr",
                                                               "normal.png", "fov.json", "mesh.glb", "pointcloud.ply"]
    assert cli.output_files(True, False, False, normal=False) == ["image.jpg", "depth_vis.png", "depth.exr", "mask.png", "points.exr",
                                                                  "fov.json"]
    assert cli.output_files(False, False, True, normal=True) == ["pointcloud.ply"]
    with pytest.warns(UserWarning, match="No output format"):
        assert cli.formats(False, False, False) == (True, True, True)


def test_resize_sizes():
    assert cli.resized_size(768, 1024, None) == (768, 1024)
    assert cli.resized_size(768, 1024, 512) == (384, 512)
    assert cli.resized_size(1024, 768, 512) == (512, 384)
    assert cli.resized_size(1365, 2048, 1000) == (666, 1000)
    assert cli.resized_size(100, 100, 64) == (64, 64)


def test_resize_interpolates_bilinearly():
    import cv2
    img = np.random.default_rng(0).integers(0, 256, (97, 131, 3), dtype=np.uint8)
    got = cv2.resize(img, (65, 48), cv2.INTER_AREA)             # INTER_AREA lands in `dst`: the default INTER_LINEAR is used
    assert np.array_equal(got, cv2.resize(img, (65, 48), interpolation=cv2.INTER_LINEAR))


def test_fov_json():
    rng = np.random.default_rng(1)
    for _ in range(20):
        K = np.array([[rng.uniform(0.3, 3), 0, 0.5], [0, rng.uniform(0.3, 3), 0.5], [0, 0, 1]], dtype=np.float32)
        fx, fy = utils3d_panorama.intrinsics_to_fov(K)
        want = {'fov_x': round(float(np.rad2deg(fx)), 2), 'fov_y': round(float(np.rad2deg(fy)), 2)}
        assert json.dumps(cli.fov_json(K)) == json.dumps(want)


@pytest.mark.parametrize("command", ["infer", "infer_panorama"])
@pytest.mark.parametrize("args,message", [(["--device", "cpu"], "CUDA devices only"), (["--show"], "--show is not provided")])
def test_usage_errors(tmp_path, command, args, message):
    from moge.scripts import infer, infer_panorama
    (tmp_path / "a.png").write_bytes(b"x")
    main = {"infer": infer.main, "infer_panorama": infer_panorama.main}[command]
    res = CliRunner().invoke(main, ["-i", str(tmp_path / "a.png"), "-o", str(tmp_path / "out")] + args)
    assert res.exit_code == 2, res.output
    assert message in res.output
    assert not (tmp_path / "out").exists()


def test_help_names_the_fp16_behaviour():
    from moge.scripts import cli as entry, infer
    res = CliRunner().invoke(infer.main, ["--help"])
    assert res.exit_code == 0 and "no fp32 pass" in res.output
    entry.cli.add_command(infer.main, name="infer")
    assert "infer" in CliRunner().invoke(entry.cli, ["--help"]).output


# ------------------------------------------------------------------------------------------------------------ C entry points
L = capi.lib()
NB = C.c_size_t()
P = 8                         # a non-null stand-in pointer; never reaches a launch
BIG = 1 << 40
Q2 = (C.c_float * 2)(0.001, 0.99)

CASES = {
    "bytes_null": ("", lambda: L.moge_vis_workspace_bytes(1, 8, 8, C.POINTER(C.c_size_t)()), "null argument"),
    "batch": ("vis", lambda: L.moge_vis_workspace_bytes(0, 8, 8, C.byref(NB)), "outside"),
    "size": ("vis", lambda: L.moge_vis_workspace_bytes(1, 0, 8, C.byref(NB)), "size"),
    "too_large": ("vis", lambda: L.moge_vis_workspace_bytes(1, 40000, 30000, C.byref(NB)), "too large"),
    "quantiles_null": ("", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, Q2, 2, None, P, BIG, None), "null argument"),
    "quantiles_kind": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 5, None, 1, 8, 8, Q2, 2, P, P, BIG, None), "unknown value kind"),
    "quantiles_count": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, Q2, 5, P, P, BIG, None), "outside"),
    "quantiles_q": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, (C.c_float * 1)(1.5), 1, P, P, BIG, None),
                    "outside [0, 1]"),
    "quantiles_batch": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 65536, 8, 8, Q2, 2, P, P, BIG, None), "outside"),
    "quantiles_ws_small": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, Q2, 2, P, 256, 16, None), "bytes needed"),
    "quantiles_ws_null": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, Q2, 2, P, None, BIG, None), "bytes needed"),
    "quantiles_ws_align": ("vis_quantiles", lambda: L.moge_vis_quantiles(P, 0, None, 1, 8, 8, Q2, 2, P, 264, BIG, None), "256-byte aligned"),
    "colorize_null": ("", lambda: L.moge_vis_colorize(P, 0, 1, None, 1, 8, 8, None, None, 0, P, None), "null argument"),
    "colorize_kind": ("vis_colorize", lambda: L.moge_vis_colorize(P, 2, 1, None, 1, 8, 8, None, P, 0, P, None), "unknown value kind"),
    "colorize_size": ("vis_colorize", lambda: L.moge_vis_colorize(P, 0, 1, None, 1, 8, -3, None, P, 0, P, None), "size"),
    "normal_null": ("", lambda: L.moge_vis_normal(None, None, 1, 8, 8, 0, P, None), "null argument"),
    "normal_batch": ("vis_normal", lambda: L.moge_vis_normal(P, None, 70000, 8, 8, 0, P, None), "outside"),
}


def expect_error(what, call, substring):
    assert call() == -1
    msg = L.moge_last_error().decode()
    assert msg.startswith(what + ": " if what else "null argument"), msg
    assert substring in msg, msg


@pytest.mark.parametrize("case", sorted(CASES))
def test_bad_arguments_are_rejected_before_any_launch(case):
    expect_error(*CASES[case])


@pytest.mark.skipif(torch.cuda.is_available(), reason="the no-device message needs a machine without a CUDA device")
def test_no_device():
    expect_error("vis_normal", lambda: L.moge_vis_normal(P, None, 1, 8, 8, 0, P, None), "no CUDA device: moge_b200 has no CPU fallback")
    with pytest.raises(capi.MogeError):
        vis.colorize_depth(torch.ones(4, 4))                     # a CPU tensor: no fallback


def test_only_spectral():
    with pytest.raises(capi.MogeError, match="only 'Spectral'"):
        vis.colorize_depth(torch.ones(4, 4), cmap="viridis")
    with pytest.raises(ValueError), np.errstate(invalid="ignore"):
        vis_port.colorize_depth(np.ones((4, 4), np.float32), cmap="viridis")
