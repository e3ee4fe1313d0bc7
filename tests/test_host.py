"""CPU: host-side logic and the C-ABI surface (no compute calls)."""
import ctypes as C
import os
import re

import pytest
import torch

from moge_b200 import capi
from moge_b200.configs import model_config, v1_model_config


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(os.path.dirname(capi._HERE), "include", "moge_b200.h")).read()
    declared = set(re.findall(r"\b(moge_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(capi.EXPORTS), declared ^ set(capi.EXPORTS)
    L = capi.lib()
    for name in declared:
        assert hasattr(L, name), name
    assert b"sm_90a" in L.moge_version()


def test_config_struct_roundtrip():
    c = capi.make_config(model_config("vitl"), capi.F16)
    assert (c.embed_dim, c.depth, c.num_heads) == (1024, 24, 16)
    assert list(c.taps)[:4] == [5, 11, 17, 23]
    assert list(c.neck.dim_in)[:5] == [1026, 2, 2, 2, 2]
    assert list(c.points_head.dim_out)[:5] == [0, 0, 0, 0, 3]
    assert list(c.neck.resamplers)[:4] == [0, 0, 0, 1]
    assert c.scale_head_layers == 3 and c.remap_output == 2
    c2 = capi.make_config(model_config("vitb", with_normal=False), capi.BF16)
    assert c2.normal_head.present == 0 and c2.compute_dtype == capi.BF16


def test_no_cpu_fallback():
    from moge.model.v2 import MoGeModel
    from moge_b200.synthetic import make_state_dict, synthetic_images
    cfg = model_config("vits")
    m = MoGeModel(**cfg)
    with pytest.raises(ValueError):
        MoGeModel(**{**cfg, "remap_output": "bogus"})
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="Missing key"):
        m.load_state_dict({"x": torch.zeros(1)})                    # strict=True like nn.Module
    rep = m.load_state_dict({"x": torch.zeros(1)}, strict=False)    # the reference's from_pretrained uses strict=False (v2.py:105)
    assert rep.unexpected_keys == ["x"] and "neck.input_blocks.0.weight" in rep.missing_keys
    with pytest.raises(NotImplementedError, match="use_fp16=False"):
        m.infer(synthetic_images(1, 28, 28, 0), use_fp16=False)
    with pytest.raises(capi.MogeError):
        m.infer(synthetic_images(1, 28, 28, 0))
    h = C.c_void_p()
    c = capi.make_config(cfg, capi.F16)
    assert capi.lib().moge_engine_create(C.byref(c), 0, C.byref(h)) != 0
    assert b"no CPU fallback" in capi.lib().moge_last_error()


def test_import_model_class_by_version():
    from moge.model import import_model_class_by_version
    from moge.model.v2 import MoGeModel
    assert import_model_class_by_version("v2") is MoGeModel
    with pytest.raises(NotImplementedError):
        import_model_class_by_version("v1")


def test_make_config_rejects_unsupported_decoders():
    cfg = model_config("vits")
    bad = {**cfg, "neck": {**cfg["neck"], "res_block_in_norm": "layer_norm"}}
    with pytest.raises(capi.MogeError):
        capi.make_config(bad, capi.F16)
    bad = {**cfg, "points_head": {**cfg["points_head"], "resamplers": ["pixel_shuffle"] * 4}}
    with pytest.raises(capi.MogeError):
        capi.make_config(bad, capi.F16)
    with pytest.raises(ValueError):
        capi.make_config({**cfg, "encoder": {**cfg["encoder"], "backbone": "dinov2_vitg14"}}, capi.F16)


def _with_last_width(cfg, width):
    stacks = [k for k in ("neck", "points_head", "normal_head", "mask_head") if k in cfg]
    return {**cfg, **{k: {**cfg[k], "dim_res_blocks": cfg[k]["dim_res_blocks"][:-1] + [width]} for k in stacks}}


@pytest.mark.parametrize("change,msg", [
    (lambda c: {k: v for k, v in c.items() if not k.endswith("_head") or k == "scale_head"}, "without points, normal and mask heads"),
    (lambda c: {**c, "neck": {**c["neck"], "resamplers": ["conv_transpose"] * 4}}, "bilinear only"),
    (lambda c: {**c, "neck": {**c["neck"], "num_res_blocks": [0, 2, 2, 2, 1]}}, "residual blocks at the last level"),
    (lambda c: _with_last_width(c, 64), "last-level width 64"),
], ids=["no_heads", "neck_convT_last", "neck_res_blocks_last", "last_width_64"])
def test_create_rejects_configs_the_neck_fold_cannot_cover(change, msg):
    """The neck's last level always runs folded through the heads (EPI_NECKOUT); a config of another shape fails at create,
    before the device is looked for."""
    h = C.c_void_p()
    c = capi.make_config(change(model_config("vits")), capi.F16)
    assert capi.lib().moge_engine_create(C.byref(c), 0, C.byref(h)) != 0
    err = capi.lib().moge_last_error().decode()
    assert msg in err, err


def _check_model_plumbing(MoGeModel, cfg):
    """nn.Module-like surface both drop-in classes share (EngineModel): dtype/device bookkeeping, training-only stubs."""
    m = MoGeModel(**cfg)
    assert m.dtype == torch.float32 and m.half().dtype == torch.float16 and m.bfloat16().dtype == torch.bfloat16
    assert m.eval() is m and m.device.type == "cpu"
    assert m.to(dtype=torch.float16).dtype == torch.float16 and m.float().dtype == torch.float32 and m.cpu() is m
    assert m.train(False) is m and m.requires_grad_(False) is m and m.state_dict() == {}
    with pytest.raises(NotImplementedError):
        m.train()
    with pytest.raises(TypeError):
        m.to(torch.float64)
    with pytest.raises(NotImplementedError):
        m.init_weights()
    with pytest.raises(NotImplementedError):
        m.enable_gradient_checkpointing()
    with pytest.warns(UserWarning):
        MoGeModel(**cfg, deprecated_thing=3)          # v2.py:42-43, v1.py:166-172
    return m


def test_model_plumbing_without_gpu():
    """nn.Module-like surface of the drop-in class (v2.py:59-74,109-120): dtype/device bookkeeping, training-only stubs."""
    from moge.model.v2 import MoGeModel
    m = _check_model_plumbing(MoGeModel, model_config("vits", with_normal=False))
    assert not hasattr(m, "normal_head") and hasattr(m, "points_head") and hasattr(m, "scale_head")
    with pytest.raises(NotImplementedError):
        m.onnx_compatible_mode = True
    assert m.onnx_compatible_mode is False


def test_v1_model_plumbing_without_gpu():
    """The same surface on the MoGe-1 class (v1.py:206-251)."""
    from moge.model.v1 import MoGeModel
    _check_model_plumbing(MoGeModel, v1_model_config("vits"))


def test_public_signatures():
    """forward / infer / infer_many keep the parameter names, order and defaults of the reference classes (v2.py:138,194,
    v1.py:269,301).  The two models take infer's arguments in different orders, behind one shared body."""
    import inspect
    from moge.model.v1 import MoGeModel as V1
    from moge.model.v2 import MoGeModel as V2
    E = inspect.Parameter.empty

    def params(f):
        ps = inspect.signature(f).parameters.values()
        assert all(p.kind == inspect.Parameter.POSITIONAL_OR_KEYWORD for p in ps), f
        return [(p.name, p.default) for p in ps]

    v2_args = [("num_tokens", None), ("resolution_level", 9), ("force_projection", True), ("apply_mask", True),
               ("fov_x", None), ("use_fp16", True)]
    v1_args = [("fov_x", None), ("resolution_level", 9), ("num_tokens", None), ("apply_mask", True),
               ("force_projection", True), ("use_fp16", True)]
    for M, args in ((V2, v2_args), (V1, v1_args)):
        assert params(M.forward) == [("self", E), ("image", E), ("num_tokens", E)]
        assert M.__call__ is M.forward
        assert params(M.infer) == [("self", E), ("image", E)] + args
        assert params(M.infer_many) == [("self", E), ("images", E)] + args


def test_synthetic_checkpoint_roundtrip(tmp_path):
    """The synthetic checkpoint is a reference-format file: {'model_config', 'model'} loadable with weights_only=True."""
    from moge.model.v2 import MoGeModel
    from moge_b200.synthetic import save_checkpoint, make_state_dict
    cfg = model_config("vits")
    path = tmp_path / "model.pt"
    save_checkpoint(path, cfg, seed=3)
    ck = torch.load(path, map_location="cpu", weights_only=True)
    assert set(ck) == {"model_config", "model"}
    m = MoGeModel.from_pretrained(path)
    sd = make_state_dict(cfg, 3)
    assert set(m.state_dict()) == set(sd) and all(torch.equal(m.state_dict()[k], sd[k]) for k in sd)
    assert m.num_tokens_range == [1200, 3600] and m.remap_output == "exp"


def test_layernorm_fold_algebra():
    """The identity behind the engine's fused LayerNorm + GEMM (moge_b200/csrc/elementwise.cu, ln_fold_kernel):
    LN(x) W^T + b == rstd * (x W''^T) + b'  with W'' = rows of (W diag(gamma)) centred, b' = b + W beta  (block.py:90,93)."""
    g = torch.Generator().manual_seed(5)
    M, K, N = 37, 96, 24
    x = (torch.randn(M, K, generator=g, dtype=torch.float64) * 3 + torch.randn(M, 1, generator=g, dtype=torch.float64))
    gamma = 1 + 0.3 * torch.randn(K, generator=g, dtype=torch.float64)
    beta = 0.2 * torch.randn(K, generator=g, dtype=torch.float64)
    W = torch.randn(N, K, generator=g, dtype=torch.float64) / K ** 0.5
    b = torch.randn(N, generator=g, dtype=torch.float64)
    ref = torch.nn.functional.linear(torch.nn.functional.layer_norm(x, (K,), gamma, beta, 1e-6), W, b)
    Wg = W * gamma[None, :]
    W2 = Wg - Wg.mean(dim=1, keepdim=True)                 # centred rows: (x - mean(x) 1) Wg^T == x W2^T
    b2 = b + W @ beta
    s1, s2 = x.sum(1), (x * x).sum(1)                      # what the producing epilogues accumulate per row
    mean = s1 / K
    rstd = 1.0 / torch.sqrt(s2 / K - mean * mean + 1e-6)
    out = rstd[:, None] * (x @ W2.T) + b2[None, :]
    assert torch.allclose(out, ref, rtol=1e-9, atol=1e-9)


def test_serving_pipeline_needs_a_cuda_model():
    from moge.model.v2 import MoGeModel
    from moge_b200.serving import InferPipeline
    m = MoGeModel(**model_config("vits", True))
    with pytest.raises(RuntimeError, match="CUDA"):
        InferPipeline(m)
    with pytest.raises(ValueError):
        InferPipeline(m, depth=0)


@pytest.mark.parametrize("tag", ["h100"])
def test_committed_bench_lines_follow_the_contract(tag):
    """profiles/<tag>_bench_n1.json and <tag>_bench_reference_arm.json are real bench.py lines: check the keys the driver parses."""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    eng = json.load(open(os.path.join(root, "profiles", f"{tag}_bench_n1.json")))
    ref = json.load(open(os.path.join(root, "profiles", f"{tag}_bench_reference_arm.json")))
    for line in (eng, ref):
        for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                  "dtype", "data", "config", "e2e", "cpu_baseline", "gpu_launches"):
            assert k in line, k
        assert "workload" in line["config"] and "model" not in line["config"]
        for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
            assert k in line["e2e"], k
        for k in ("value", "unit", "cores", "kind", "sample"):
            assert k in line["cpu_baseline"], k
    assert eng["metric"] == ref["metric"] and eng["unit"] == ref["unit"] and eng["config"]["workload"] == ref["config"]["workload"]
    assert ref["impl"] == "reference" and ref["e2e"]["h2d_bytes_per_step"] == 0 and ref["gpu_launches"] == 0
    assert eng["gpu_launches"] > 0 and eng["e2e"]["h2d_bytes_per_step"] > 0 and eng["e2e"]["value"] != eng["value"]
    r = eng["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(eng["clocks"])
    gb = eng["gpu_baseline"]                              # same-box PyTorch-CUDA comparator, both 16-bit modes of the reference
    for mode in ("half", "autocast"):
        assert gb[mode]["batch1_iters"] >= 200 and gb[mode]["images_per_s"] > 0
    assert eng["latency"]["iters"] >= 200
    assert "SURVEY" in eng["roofline_decoder"]["bytes_definition"] and eng["roofline_decoder"]["frac_engine_bytes"] < eng["roofline_decoder"]["frac"]


def test_all_committed_profile_json_files_parse():
    import glob
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for f in glob.glob(os.path.join(root, "profiles", "*.json")):
        json.load(open(f))


def _work_list(n_tokens, heads, n_ctas):
    L = capi.lib()
    n = (C.c_int * len(n_tokens))(*n_tokens)
    ni, nr = C.c_int(), C.c_int()
    capi.check(L.moge_attention_work_list(n, len(n_tokens), heads, n_ctas, None, 0, None, C.byref(ni), C.byref(nr)))
    items = (C.c_int * (4 * max(ni.value, 1)))()
    ranges = (C.c_int * (2 * n_ctas))()
    capi.check(L.moge_attention_work_list(n, len(n_tokens), heads, n_ctas, items, ni.value, ranges, C.byref(ni), C.byref(nr)))
    it = [tuple(items[4 * i:4 * i + 4]) for i in range(ni.value)]
    rg = [tuple(ranges[2 * i:2 * i + 2]) for i in range(nr.value)]
    return it, rg


@pytest.mark.parametrize("n_tokens,heads,n_ctas", [
    ([1370] * 32, 16, 148),                  # the benchmark batch
    ([1370], 16, 148),                       # batch 1: fewer items than CTAs
    ([3601] * 8, 16, 148),                   # API-default grid
    ([704, 1370, 704, 3601, 1226, 1370], 12, 148),   # mixed-shape batch (shape groups)
    ([1], 6, 148), ([256, 257, 512, 513], 6, 7), ([129] * 5, 16, 1),
])
def test_attention_work_list_partition(n_tokens, heads, n_ctas):
    """Plan-time host logic of the persistent attention kernel (attention.cu attention_work_list): every (image, head, 256-query
    tile) exactly once, the per-CTA ranges contiguous and non-empty, the modelled cost balanced."""
    it, rg = _work_list(n_tokens, heads, n_ctas)
    row0 = [sum(n_tokens[:i]) for i in range(len(n_tokens))]
    want = {(row0[i], n_tokens[i], q0, h) for i in range(len(n_tokens)) for h in range(heads) for q0 in range(0, n_tokens[i], 256)}
    assert len(it) == len(want) and set(it) == want
    assert len(rg) == min(n_ctas, len(it))
    assert rg[0][0] == 0 and rg[-1][1] == len(it)
    for (b0, e0), (b1, e1) in zip(rg, rg[1:]):
        assert e0 == b1
    assert all(e > b for b, e in rg)
    # cost model of the kernel: kv tiles x query groups per item (+ a constant); no CTA above mean + one largest item
    cost = [-(-n // 128) * (2 if q0 + 128 < n else 1) + 0.5 for (_, n, q0, _) in it]
    per_cta = [sum(cost[b:e]) for b, e in rg]
    assert max(per_cta) <= sum(cost) / len(rg) + max(cost) + 1e-9


def test_attention_work_list_rejects_bad_arguments():
    L = capi.lib()
    n = (C.c_int * 2)(1370, 0)
    ni = C.c_int()
    assert L.moge_attention_work_list(n, 2, 16, 148, None, 0, None, C.byref(ni), None) != 0
    assert b"tokens" in L.moge_last_error()
    n = (C.c_int * 1)(1370)
    items = (C.c_int * 4)()
    assert L.moge_attention_work_list(n, 1, 16, 148, items, 1, None, C.byref(ni), None) != 0      # items_cap too small


@pytest.mark.parametrize("compiler,std,lang", [("gcc", "-std=c99", "c"), ("g++", "-std=c++11", "c++")])
def test_header_is_plain_c_and_cxx(tmp_path, compiler, std, lang):
    """The drop-in boundary is a C ABI: include/moge_b200.h must compile as strict C99 and as C++ with nothing but the standard headers."""
    import shutil
    import subprocess
    if shutil.which(compiler) is None:
        pytest.skip(compiler + " not installed")
    src = tmp_path / "use_header.c"
    src.write_text('#include "moge_b200.h"\nint main(void) { moge_config_t c; moge_group_t g; (void)c; (void)g; return moge_version() == 0; }\n')
    inc = os.path.join(os.path.dirname(capi._HERE), "include")
    r = subprocess.run([compiler, std, "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", inc, "-x", lang, "-fsyntax-only", str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
