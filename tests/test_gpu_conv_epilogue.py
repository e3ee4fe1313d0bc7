"""-m gpu: the EPI_DEC epilogues of the 3x3 convs in every output combination moge_op_conv reaches -- ReLU copy only, raw +
skip, raw + ReLU + skip, raw + ReLU, raw only, ReLU + skip -- against F.conv2d on replicate padding, with the replicated 1-pixel
border checked on every output, and tile by tile.  In the halo modes (CONV64: C_in = 64, CONVH: C_in >= 128) the first four run
the direct epilogue (a compile-time output mask, stores from the consumers' registers).  Raw only and ReLU + skip, which neither
mode specialises (MoGe-1's decoder convs write only the raw map), run the staged epilogue instead: in CONV64 its run-time-flag
variant, while at C_in >= 128 the conv leaves CONVH, which has no such variant, for the per-tap GEMM mode (raw only there is
its specialised DF_RAW, ReLU + skip the run-time flags).  A map 6 pixels tall (padded height 8, under one halo box) takes the
per-tap GEMM mode for every output.  The shapes mix interior tiles (TMA stores) with ragged edge tiles (H % 8 != 0,
W % 16 != 0), a map one halo box tall, and more than one image.  The two epilogues are also compared on the same inputs: bit
for bit where they share the main loop."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, to_padded_nhwc, empty_padded, from_padded_nhwc, border_ok, check_tiles, tile_conv

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}
# direct epilogue in the halo modes: relu, raw_skip, raw_relu_skip, raw_relu; staged: raw, relu_skip
OUTPUTS = ["relu", "raw_skip", "raw_relu_skip", "raw_relu", "raw", "relu_skip"]
SHAPES = [(2, 37, 53, 64, 64),      # CONV64, ragged, two images
          (1, 8, 40, 64, 128),      # CONV64, one box tall, two channel tiles
          (2, 29, 70, 128, 128),    # CONVH, ragged, two images
          (1, 8, 33, 256, 256),     # CONVH, one box tall
          (1, 48, 64, 128, 256),    # CONVH, whole tiles, interior tiles in both directions
          (1, 6, 37, 128, 128)]     # per-tap GEMM (under one halo box)


def _inputs(B, H, W, Cin, Cout, dtype):
    g = torch.Generator(device="cpu").manual_seed(B * H * W + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(DEV)
    b = torch.randn(Cout, generator=g).to(DEV)
    skip = torch.randn(B, Cout, H, W, generator=g).to(DEV).to(dtype)
    return x, w, b, skip


def _conv(x, w, b, skip, outputs, B, H, W, Cin, Cout, dtype):
    """moge_op_conv with the outputs (and the skip operand) that `outputs` names: (raw, relu) padded maps, None if not written"""
    has_raw, has_relu, has_skip = "raw" in outputs, "relu" in outputs, "skip" in outputs
    xp, sp = to_padded_nhwc(x, dtype), to_padded_nhwc(skip, dtype)
    raw = empty_padded(B, H, W, Cout, dtype, DEV) if has_raw else None
    relu = empty_padded(B, H, W, Cout, dtype, DEV) if has_relu else None
    capi.check(capi.lib().moge_op_conv(xp.data_ptr(), w.data_ptr(), b.data_ptr(), sp.data_ptr() if has_skip else None,
                                       raw.data_ptr() if has_raw else None, relu.data_ptr() if has_relu else None,
                                       B, H, W, Cin, Cout, 9, 0, dt(dtype), stream()))
    torch.cuda.synchronize()
    return raw, relu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("outputs", OUTPUTS)
@pytest.mark.parametrize("B,H,W,Cin,Cout", SHAPES)
def test_conv3x3_direct_epilogue(B, H, W, Cin, Cout, outputs, dtype):
    x, w, b, skip = _inputs(B, H, W, Cin, Cout, dtype)
    has_skip = "skip" in outputs
    raw, relu = _conv(x, w, b, skip, outputs, B, H, W, Cin, Cout, dtype)
    ref = F.conv2d(F.pad(x.float(), (1, 1, 1, 1), mode="replicate"), w.to(dtype).float(), b)
    if has_skip:
        ref = ref + skip.float()
    for out, r in ((raw, ref), (relu, F.relu(ref))):
        if out is None:
            continue
        got = from_padded_nhwc(out, H, W)
        assert torch.isfinite(got).all()
        assert rel_l2(got, r) < TOL[dtype]
        assert border_ok(out, H, W)
        check_tiles(got, r, tile_conv(Cout), TOL[dtype], f"conv {outputs} {dtype}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W,Cin,Cout", SHAPES)
def test_conv3x3_epilogue_variants_bitwise(B, H, W, Cin, Cout, dtype):
    """The same conv through two epilogues: the raw map of raw only (staged) against that of raw + ReLU, and the ReLU map of
    ReLU + skip (staged) against that of raw + ReLU + skip (both direct in the halo modes).  Both epilogues add bias, then skip,
    in fp32 before one rounding.  In CONV64 and in the per-tap mode the two share the main loop and its k-order, so the maps,
    borders included, are equal bit for bit.  In CONVH the staged outputs run the per-tap GEMM main loop, which sums the k
    blocks tap by tap (each tap over the channel blocks) where CONVH sums them channel block by channel block (each over the 9
    taps): the fp32 sums differ in the last bits, so there the two maps are held to each other tile by tile."""
    x, w, b, skip = _inputs(B, H, W, Cin, Cout, dtype)
    convh = Cin >= 128 and H + 2 >= 10
    pairs = ((("raw", 0), ("raw_relu", 0)), (("relu_skip", 1), ("raw_relu_skip", 1)))
    for (flags, i), (spec, j) in pairs:
        a = _conv(x, w, b, skip, flags, B, H, W, Cin, Cout, dtype)[i]
        s = _conv(x, w, b, skip, spec, B, H, W, Cin, Cout, dtype)[j]
        if convh:
            assert border_ok(a, H, W) and border_ok(s, H, W)
            check_tiles(from_padded_nhwc(a, H, W), from_padded_nhwc(s, H, W), tile_conv(Cout), TOL[dtype],
                        f"conv {flags} against {spec} {dtype}")
            continue
        a, s = a[:, :H + 2, :W + 2], s[:, :H + 2, :W + 2]
        diff = (a.float() - s.float()).abs().max().item()
        assert torch.equal(a, s), f"{flags} and {spec} differ: max |diff| {diff:.3e}"
