"""moge_b200.mesh on the GPU, bitwise against the numpy restatement of utils3d in oracle/utils3d_mesh.py: depth_map_edge over
shapes, kernel sizes, tolerances, masks, inf holes and negative depths; build_mesh_from_map over masks and tri; mesh_from_output
on synthetic infer()-style outputs and on the real infer() output of MoGe-2 (with normals) and MoGe-1 (without); batch against
single-image calls; one host synchronisation per call; inputs left unmodified and repeated calls identical."""
import numpy as np
import pytest
import torch

from moge_b200 import mesh as M
from moge_b200.synthetic import synthetic_images, synthetic_mesh_case
from oracle import utils3d_mesh as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def depth_case(B, H, W, seed):
    """(B, H, W) depths: a gently varying surface with box steps, ~4 % +inf holes and ~1 % negative depths; a ~80 % mask."""
    g = torch.Generator().manual_seed(seed)
    d = 2 + 0.05 * torch.rand(B, H, W, generator=g)
    for _ in range(3):
        i, j = int(torch.randint(0, H, (), generator=g)), int(torch.randint(0, W, (), generator=g))
        d[:, i:i + max(1, H // 3), j:j + max(1, W // 3)] += 1.5 * torch.rand((), generator=g).item()
    d = torch.where(torch.rand(B, H, W, generator=g) < 0.04, torch.tensor(float("inf")), d)
    d = torch.where(torch.rand(B, H, W, generator=g) < 0.01, -d, d)
    return d, torch.rand(B, H, W, generator=g) < 0.8


TOLS = [(None, None), (0.3, None), (None, 0.04), (0.3, 0.04)]


@pytest.mark.parametrize("H,W", [(1, 1), (1, 57), (43, 1), (37, 53), (480, 640), (1365, 2048)])
@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("masked", [False, True])
def test_depth_map_edge_bitwise(H, W, k, masked):
    d, m = depth_case(1, H, W, H * W + k)
    d, m = d[0], m[0]
    dg, mg = d.to(DEV), (m.to(DEV) if masked else None)
    for atol, rtol in TOLS:
        got = M.depth_map_edge(dg, atol=atol, rtol=rtol, kernel_size=k, mask=mg)
        want = O.depth_map_edge(d.numpy(), atol=atol, rtol=rtol, kernel_size=k, mask=m.numpy() if masked else None)
        assert got.dtype == torch.bool and got.shape == (H, W)
        assert np.array_equal(got.cpu().numpy(), want), (atol, rtol, int((got.cpu().numpy() != want).sum()))
        if atol is not None or rtol is not None:
            assert H * W < 100 or want.any()
    assert torch.equal(dg.cpu(), d)                                # the input is not modified


def test_depth_map_edge_batch():
    d, m = depth_case(3, 37, 53, 11)
    for mask in (None, m):
        got = M.depth_map_edge(d.to(DEV)[None], rtol=0.04, kernel_size=5, mask=None if mask is None else mask.to(DEV)[None])
        want = O.depth_map_edge(d.numpy(), rtol=0.04, kernel_size=5, mask=None if mask is None else mask.numpy())
        assert got.shape == (1, 3, 37, 53) and np.array_equal(got[0].cpu().numpy(), want)
        for b in range(3):
            one = M.depth_map_edge(d[b].to(DEV), rtol=0.04, kernel_size=5, mask=None if mask is None else mask[b].to(DEV))
            assert torch.equal(one, got[0, b])


def mask_case(kind, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "none":
        return None
    if kind == "random":
        return torch.rand(H, W, generator=g) < 0.7
    if kind == "empty":
        return torch.zeros(H, W, dtype=torch.bool)
    return torch.rand(H, W, generator=g) < 0.15        # "sparse": mostly isolated pixels, a few quads


def maps_case(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(H, W, 3, generator=g), torch.randn(H, W, generator=g), torch.rand(H, W, 2, generator=g)]


def assert_mesh_equal(got, want):
    assert len(got) == len(want)
    assert got[0].dtype == torch.int32 and np.array_equal(got[0].cpu().numpy(), want[0]) and got[0].shape == want[0].shape
    for g, w in zip(got[1:], want[1:]):
        assert g.dtype == torch.float32 and g.shape == w.shape and g.cpu().numpy().tobytes() == np.ascontiguousarray(w).tobytes()


@pytest.mark.parametrize("H,W", [(1, 1), (1, 9), (9, 1), (2, 3), (37, 53), (480, 640)])
@pytest.mark.parametrize("kind", ["none", "random", "empty", "sparse"])
@pytest.mark.parametrize("tri", [False, True])
def test_build_mesh_from_map_bitwise(H, W, kind, tri):
    maps = maps_case(H, W, H + W)
    mask = mask_case(kind, H, W, H * W)
    got = M.build_mesh_from_map(*[x.to(DEV) for x in maps], mask=None if mask is None else mask.to(DEV), tri=tri)
    want = O.build_mesh_from_map(*[x.numpy() for x in maps], mask=None if mask is None else mask.numpy(), tri=tri)
    assert_mesh_equal(got, want)
    if kind == "empty":
        assert got[0].shape == (0, 3 if tri else 4) and got[1].shape == (0, 3) and got[2].shape == (0,)


def oracle_output(out, image, b, remove_edge=True, normals=True):
    n = out["normal"][b].cpu().numpy() if normals and "normal" in out else None
    return O.mesh_from_output(out["points"][b].cpu().numpy(), out["depth"][b].cpu().numpy(), out["mask"][b].cpu().numpy(),
                              image[b].cpu().numpy(), n, remove_edge=remove_edge)


def assert_output_equal(got, want):
    assert set(got) == set(want), (sorted(got), sorted(want))
    assert np.array_equal(got["mask_cleaned"].cpu().numpy(), want["mask_cleaned"])
    assert got["faces"].dtype == torch.int32 and np.array_equal(got["faces"].cpu().numpy(), want["faces"])
    for k in ("vertices", "vertex_colors", "vertex_uvs", "vertex_normals"):
        if k in want:
            g = got[k].cpu().numpy()
            assert g.dtype == np.float32 and g.shape == want[k].shape and g.tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("remove_edge", [True, False])
def test_mesh_from_output_synthetic_2048x1365(remove_edge):
    out, image = synthetic_mesh_case(0, 2, 1365, 2048)
    dev_out = {k: v.to(DEV) for k, v in out.items()}
    res = M.mesh_from_output(dev_out, image.to(DEV), remove_edge=remove_edge)
    for b in range(2):
        want = oracle_output(out, image, b, remove_edge)
        assert want["faces"].shape[0] > 1_000_000
        assert_output_equal(res[b], want)
    # the float32 (3, H, W) image given to infer(): colours are taken as they are
    chw = torch.from_numpy(image.numpy().astype(np.float32) / np.float32(255)).permute(0, 3, 1, 2)
    one = M.mesh_from_output({k: v[0] for k, v in dev_out.items()}, chw[0].to(DEV), remove_edge=remove_edge)
    assert torch.equal(one["vertex_colors"], res[0]["vertex_colors"]) and torch.equal(one["faces"], res[0]["faces"])


def _infer_image(H, W, seed):
    img = synthetic_images(1, H, W, seed)[0]
    return img, (img.permute(1, 2, 0) * 255).round().to(torch.uint8)


def test_mesh_from_output_real_moge2_infer():
    from moge.model.v2 import MoGeModel
    from moge_b200.configs import model_config
    from moge_b200.synthetic import make_state_dict
    cfg = model_config("vits", True)
    model = MoGeModel(**cfg)
    model.load_state_dict(make_state_dict(cfg, 0, well_posed=True))
    model = model.to(DEV).eval()
    img, img_u8 = _infer_image(196, 252, 0)
    out = model.infer(img.to(DEV), num_tokens=300)
    assert "normal" in out and torch.isinf(out["depth"][~out["mask"]]).all()
    check_real_output(out, img_u8, normals=True)


def check_real_output(out, img_u8, normals):
    """The random-init models' depth is rough at the pixel scale, so the 4 % edge rule may clean away most of the mask: the
    output is also checked with the edges kept, where the mesh covers the whole mask."""
    for remove_edge in (True, False):
        res = M.mesh_from_output(out, img_u8.to(DEV), remove_edge=remove_edge)
        want = oracle_output({k: v[None] for k, v in out.items()}, img_u8[None], 0, remove_edge)
        assert ("vertex_normals" in res) == normals
        assert remove_edge or res["faces"].shape[0] > 1000
        assert_output_equal(res, want)


def test_mesh_from_output_real_moge1_infer():
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vits")
    model = MoGeModel(**cfg)
    model.load_state_dict(make_v1_state_dict(cfg, 7, well_posed=True))
    model = model.to(DEV).half()
    img, img_u8 = _infer_image(126, 168, 7)
    out = model.infer(img.to(DEV), num_tokens=192)
    assert "normal" not in out
    check_real_output(out, img_u8, normals=False)


def test_batch_equals_single_calls_and_offsets_agree():
    B, H, W = 4, 97, 131
    maps = [torch.stack(x) for x in zip(*[maps_case(H, W, 40 + b) for b in range(B)])]
    mask = torch.stack([mask_case("random", H, W, 50 + b) for b in range(B)])
    mask[2] = False                                                 # an image without faces inside the batch
    for tri in (False, True):
        batch = M.build_mesh_from_map_batch(*[x.to(DEV) for x in maps], mask=mask.to(DEV), tri=tri)
        assert len(batch) == B
        nv = nf = 0
        for b in range(B):
            single = M.build_mesh_from_map(*[x[b].to(DEV) for x in maps], mask=mask[b].to(DEV), tri=tri)
            for g, s in zip(batch[b], single):
                assert torch.equal(g, s)
            # every result is a view of one allocation, images in order (an empty view has no data pointer)
            if batch[b][0].numel():
                assert batch[b][0].data_ptr() == batch[0][0].data_ptr() + 4 * nf
                assert batch[b][1].data_ptr() == batch[0][1].data_ptr() + 4 * 3 * nv
            nv += batch[b][1].shape[0]
            nf += batch[b][0].numel()
        assert batch[2][0].shape[0] == 0
    out, image = synthetic_mesh_case(3, 3, 120, 160)
    dev_out, dev_img = {k: v.to(DEV) for k, v in out.items()}, image.to(DEV)
    res = M.mesh_from_output(dev_out, dev_img)
    for b in range(3):
        one = M.mesh_from_output({k: v[b] for k, v in dev_out.items()}, dev_img[b])
        assert one.keys() == res[b].keys()
        for k in one:
            assert torch.equal(one[k], res[b][k]), (b, k)


def test_one_host_sync_inputs_unmodified_and_repeatable():
    out, image = synthetic_mesh_case(5, 2, 200, 300)
    dev_out, dev_img = {k: v.to(DEV) for k, v in out.items()}, image.to(DEV)
    first = M.mesh_from_output(dev_out, dev_img)                    # warm-up: library load, allocator
    torch.cuda.synchronize()
    d, m = dev_out["depth"].contiguous(), dev_out["mask"].contiguous().view(torch.uint8)
    B, H, W = d.shape
    maps = M._output_maps(dev_out["points"], M._Map(dev_img, M.capi.MESH_U8_UNIT, 3), dev_out["normal"])
    torch.cuda.set_sync_debug_mode("error")
    try:                                                            # edge, count and the counts copy: no synchronisation
        cleaned = M._edge(d, None, m, None, 0.04, 3)
        counted = M._count(cleaned, B, H, W, d.device)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    counted[3].synchronize()                                        # the one wait: for the counts
    torch.cuda.set_sync_debug_mode("error")
    try:                                                            # allocation and the emit passes: no synchronisation
        res = M._build(cleaned, B, H, W, maps, True, counted)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for b in range(B):
        f, v, c, uv, n = res[b]
        assert torch.equal(f, first[b]["faces"]) and torch.equal(v, first[b]["vertices"]) and torch.equal(c, first[b]["vertex_colors"])
        assert torch.equal(uv, first[b]["vertex_uvs"]) and torch.equal(n, first[b]["vertex_normals"])
    for k, v in out.items():
        assert torch.equal(dev_out[k].cpu(), v), k
    assert torch.equal(dev_img.cpu(), image)
    for _ in range(3):
        again = M.mesh_from_output(dev_out, dev_img)
        for b in range(B):
            for k in first[b]:
                assert again[b][k].cpu().numpy().tobytes() == first[b][k].cpu().numpy().tobytes(), (b, k)
