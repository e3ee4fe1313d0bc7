"""-m gpu: the direct EPI_DEC epilogue of the halo conv modes (CONV64: C_in = 64, CONVH: C_in >= 128) in every output
combination moge_op_conv reaches -- ReLU copy only, raw + skip, raw + ReLU + skip, raw + ReLU -- against F.conv2d on
replicate padding, with the replicated 1-pixel border checked on every output.  The shapes mix interior tiles (TMA stores) with
ragged edge tiles (H % 8 != 0, W % 16 != 0), a map one halo box tall, and more than one image."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, to_padded_nhwc, empty_padded, from_padded_nhwc, border_ok

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}
OUTPUTS = ["relu", "raw_skip", "raw_relu_skip", "raw_relu"]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("outputs", OUTPUTS)
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 37, 53, 64, 64),      # CONV64, ragged, two images
                                               (1, 8, 40, 64, 128),      # CONV64, one box tall, two channel tiles
                                               (2, 29, 70, 128, 128),    # CONVH, ragged, two images
                                               (1, 8, 33, 256, 256),     # CONVH, one box tall
                                               (1, 48, 64, 128, 256)])   # CONVH, whole tiles, interior tiles in both directions
def test_conv3x3_direct_epilogue(B, H, W, Cin, Cout, outputs, dtype):
    g = torch.Generator(device="cpu").manual_seed(B * H * W + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(DEV)
    b = torch.randn(Cout, generator=g).to(DEV)
    skip = torch.randn(B, Cout, H, W, generator=g).to(DEV).to(dtype)
    has_raw, has_relu, has_skip = "raw" in outputs, "relu" in outputs, "skip" in outputs
    xp, sp = to_padded_nhwc(x, dtype), to_padded_nhwc(skip, dtype)
    raw = empty_padded(B, H, W, Cout, dtype, DEV) if has_raw else None
    relu = empty_padded(B, H, W, Cout, dtype, DEV) if has_relu else None
    capi.check(capi.lib().moge_op_conv(xp.data_ptr(), w.data_ptr(), b.data_ptr(), sp.data_ptr() if has_skip else None,
                                       raw.data_ptr() if has_raw else None, relu.data_ptr() if has_relu else None,
                                       B, H, W, Cin, Cout, 9, 0, dt(dtype), stream()))
    torch.cuda.synchronize()
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
