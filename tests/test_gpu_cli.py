"""`moge infer` and `moge infer_panorama` end to end on the GPU, through click's CliRunner, on random-init ViT-S checkpoints.  Every
file is rebuilt from the same model's outputs by the reference script's lines, with oracle/vis_port.py and oracle/utils3d_mesh.py
in place of matplotlib and utils3d, cv2 for the encodes and moge_b200.export for GLB / PLY."""
import os
os.environ['OPENCV_IO_ENABLE_OPENEXR'] = '1'
import contextlib
import json
from pathlib import Path

import cv2
import numpy as np
import pytest
import torch
from click.testing import CliRunner

from moge_b200 import cli
from moge_b200.export import save_glb, save_ply
from oracle import utils3d_mesh, vis_port
from oracle.utils3d_panorama import intrinsics_to_fov

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EXR = [cv2.IMWRITE_EXR_TYPE, cv2.IMWRITE_EXR_TYPE_FLOAT]
NUM_TOKENS = 120


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    from moge_b200.configs import model_config, v1_model_config
    from moge_b200.synthetic import make_state_dict, make_v1_state_dict
    d = tmp_path_factory.mktemp("ckpt")
    cfg = model_config("vits", True)
    torch.save({"model_config": cfg, "model": make_state_dict(cfg, 0, well_posed=True)}, d / "v2.pt")
    cfg1 = v1_model_config("vits")
    torch.save({"model_config": cfg1, "model": make_v1_state_dict(cfg1, 7, well_posed=True)}, d / "v1.pt")
    return {"v2": d / "v2.pt", "v1": d / "v1.pt"}


@pytest.fixture(scope="module")
def images(tmp_path_factory):
    """Three images of different sizes: one in a subfolder, one with an upper-case .PNG suffix."""
    d = tmp_path_factory.mktemp("images")
    (d / "sub").mkdir()
    rng = np.random.default_rng(0)
    for name, (h, w) in (("a.jpg", (120, 160)), ("sub/b.png", (98, 126)), ("C.PNG", (140, 112))):
        i, j = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        img = np.stack([128 + 90 * np.sin(j / 9 + c) * np.cos(i / 7 + 2 * c) for c in range(3)], -1) + rng.integers(-20, 21, (h, w, 3))
        cv2.imwrite(str(d / name), np.clip(img, 0, 255).astype(np.uint8))
    return d


def load(version, path, fp16):
    if version == "v1":
        from moge.model.v1 import MoGeModel
    else:
        from moge.model.v2 import MoGeModel
    m = MoGeModel.from_pretrained(str(path)).to(DEV).eval()
    return m.half() if fp16 else m


def expected_infer(model, input_path, image_path, out_dir, resize_to, maps, glb, ply, threshold):
    """moge/scripts/infer.py:93-156 with the oracle's colourisers and mesh."""
    image = cv2.cvtColor(cv2.imread(str(image_path)), cv2.COLOR_BGR2RGB)
    height, width = image.shape[:2]
    if resize_to is not None:
        height, width = min(resize_to, int(resize_to * height / width)), min(resize_to, int(resize_to * width / height))
        image = cv2.resize(image, (width, height), cv2.INTER_AREA)
    image_tensor = torch.tensor(image / 255, dtype=torch.float32, device=DEV).permute(2, 0, 1)
    output = model.infer(image_tensor, fov_x=None, resolution_level=9, num_tokens=NUM_TOKENS, use_fp16=True)
    points, depth, mask, intrinsics = (output[k].cpu().numpy() for k in ("points", "depth", "mask", "intrinsics"))
    normal = output["normal"].cpu().numpy() if "normal" in output else None
    save_path = Path(out_dir, image_path.relative_to(input_path).parent, image_path.stem)
    save_path.mkdir(exist_ok=True, parents=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        if maps:
            cv2.imwrite(str(save_path / 'image.jpg'), cv2.cvtColor(image, cv2.COLOR_RGB2BGR))
            cv2.imwrite(str(save_path / 'depth_vis.png'), cv2.cvtColor(vis_port.colorize_depth(depth), cv2.COLOR_RGB2BGR))
            cv2.imwrite(str(save_path / 'depth.exr'), depth, EXR)
            cv2.imwrite(str(save_path / 'mask.png'), (mask * 255).astype(np.uint8))
            cv2.imwrite(str(save_path / 'points.exr'), cv2.cvtColor(points, cv2.COLOR_RGB2BGR), EXR)
            if normal is not None:
                cv2.imwrite(str(save_path / 'normal.png'), cv2.cvtColor(vis_port.colorize_normal(normal), cv2.COLOR_RGB2BGR))
            fov_x, fov_y = intrinsics_to_fov(intrinsics)
            with open(save_path / 'fov.json', 'w') as f:
                json.dump({'fov_x': round(float(np.rad2deg(fov_x)), 2), 'fov_y': round(float(np.rad2deg(fov_y)), 2)}, f)
        if glb or ply:
            mesh = utils3d_mesh.mesh_from_output(points, depth, mask, image, normal, threshold=threshold)
            if glb:
                save_glb(save_path / 'mesh.glb', mesh["vertices"], mesh["faces"], mesh["vertex_uvs"], image, mesh.get("vertex_normals"))
            if ply:
                save_ply(save_path / 'pointcloud.ply', mesh["vertices"], np.zeros((0, 3), dtype=np.int32), mesh["vertex_colors"],
                         mesh.get("vertex_normals"))


def compare_trees(got: Path, want: Path):
    files = sorted(p.relative_to(want) for p in want.rglob("*") if p.is_file())
    assert files and sorted(p.relative_to(got) for p in got.rglob("*") if p.is_file()) == files
    for rel in files:
        a, b = got / rel, want / rel
        if rel.suffix in (".png", ".jpg", ".exr"):
            x, y = cv2.imread(str(a), cv2.IMREAD_UNCHANGED), cv2.imread(str(b), cv2.IMREAD_UNCHANGED)
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), rel
        elif rel.suffix == ".json":
            assert json.loads(a.read_text()) == json.loads(b.read_text()), rel
        else:
            assert a.read_bytes() == b.read_bytes(), rel
    return files


# The random-init models' depth is rough at the pixel scale, so the default 4 % edge rule would clean away the whole mesh (and
# save_glb rejects an empty one): the mesh runs keep every edge with --threshold inf, and one maps run checks the default.
RUNS = [("v2", ["--maps", "--glb", "--ply"], None, False), ("v1", ["--maps", "--glb", "--ply"], None, False),
        ("v2", [], None, False), ("v2", ["--maps"], 96, False), ("v1", ["--glb", "--ply"], None, True), ("v2", ["--maps", "--ply"], None, True)]


@pytest.mark.parametrize("version,flags,resize_to,fp16", RUNS)
def test_infer_cli(tmp_path, checkpoints, images, version, flags, resize_to, fp16):
    from moge.scripts import infer
    args = ["-i", str(images), "-o", str(tmp_path / "got"), "--pretrained", str(checkpoints[version]), "--version", version,
            "--num_tokens", str(NUM_TOKENS)] + (["--threshold", "inf"] if flags != ["--maps"] else []) + flags + (["--resize", str(resize_to)] if resize_to else []) + (["--fp16"] if fp16 else [])
    with pytest.warns(UserWarning, match="No output format") if not flags else contextlib.nullcontext():
        res = CliRunner().invoke(infer.main, args, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    maps, glb, ply = ("--maps" in flags, "--glb" in flags, "--ply" in flags) if flags else (True, True, True)
    model = load(version, checkpoints[version], fp16)
    for path in cli.list_images(images):
        expected_infer(model, images, path, tmp_path / "want", resize_to, maps, glb, ply, 0.04 if flags == ["--maps"] else np.inf)
    files = compare_trees(tmp_path / "got", tmp_path / "want")
    per_image = cli.output_files(maps, glb, ply, normal=version == "v2")
    assert len(files) == 3 * len(per_image) and Path("sub", "b", per_image[-1]) in files


def test_infer_panorama_cli(tmp_path, checkpoints):
    from moge.scripts import infer_panorama as script
    from moge_b200.mesh import mesh_from_panorama
    from moge_b200.panorama import infer_panorama
    from moge_b200.synthetic import synthetic_panorama
    src = tmp_path / "in"
    src.mkdir()
    image = synthetic_panorama(256, 512, 3)
    cv2.imwrite(str(src / "pano.png"), cv2.cvtColor(image, cv2.COLOR_RGB2BGR))
    args = ["-i", str(src), "-o", str(tmp_path / "got"), "--pretrained", str(checkpoints["v1"]), "--maps", "--glb", "--ply", "--splitted",
            "--threshold", "inf"]
    res = CliRunner().invoke(script.main, args, catch_exceptions=False)
    assert res.exit_code == 0, res.output

    model = load("v1", checkpoints["v1"], False)
    dimg = torch.from_numpy(image).to(DEV)
    out = infer_panorama(model, dimg, batch_size=4, return_views=True)
    plain = infer_panorama(model, dimg, batch_size=4)
    assert sorted(plain) == ["depth", "mask", "points"]
    for k in plain:
        assert torch.equal(plain[k], out[k]), k
    host = {k: v.cpu().numpy() for k, v in out.items()}
    want = tmp_path / "want"
    split = want / "pano" / "splitted"
    split.mkdir(parents=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(len(host["views"])):
            cv2.imwrite(str(split / f'{i:02d}.jpg'), cv2.cvtColor(host["views"][i], cv2.COLOR_RGB2BGR))
            cv2.imwrite(str(split / f'{i:02d}_distance_vis.png'),
                        cv2.cvtColor(vis_port.colorize_depth(host["view_distance"][i], host["view_mask"][i]), cv2.COLOR_RGB2BGR))
        d, m, p = host["depth"], host["mask"], host["points"]
        cv2.imwrite(str(want / "pano" / 'image.jpg'), cv2.cvtColor(image, cv2.COLOR_RGB2BGR))
        cv2.imwrite(str(want / "pano" / 'depth_vis.png'), cv2.cvtColor(vis_port.colorize_depth(d, mask=m), cv2.COLOR_RGB2BGR))
        cv2.imwrite(str(want / "pano" / 'depth.exr'), d, EXR)
        cv2.imwrite(str(want / "pano" / 'points.exr'), p, EXR)
        cv2.imwrite(str(want / "pano" / 'mask.png'), (m * 255).astype(np.uint8))
    # the mesh: the engine's mesh_from_panorama (checked against the utils3d restatement in test_gpu_panorama_mesh.py)
    mesh = {k: v.cpu().numpy() for k, v in mesh_from_panorama(out, dimg, float("inf")).items()}
    save_glb(want / "pano" / 'mesh.glb', mesh["vertices"], mesh["faces"], mesh["vertex_uvs"], image)
    save_ply(want / "pano" / 'mesh.ply', mesh["vertices"], mesh["faces"], mesh["vertex_colors"])
    files = compare_trees(tmp_path / "got", want)
    assert len(files) == 24 + 7
