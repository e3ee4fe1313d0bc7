"""-m gpu: the persistent attention kernel where one CTA walks many work items.  The second consumer warpgroup skips a query
tile that lies past the image, and the barrier phases carry from item to item, so these cases run several items per CTA, with
dead tiles among them, against an fp32 SDPA, and check that an image's result does not depend on the batch around it."""
import pytest
import torch
import torch.nn.functional as F

from moge_b200 import capi
from gpu_util import rel_l2, stream, dt, TILE_ATTENTION, TILE_C, worst_tile

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float16: 3e-3, torch.bfloat16: 1.5e-2}


def _qkv(B, N, heads, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(B, N, 3 * heads * 64, generator=g) * 1.5).to(DEV).to(dtype)


def _attention(qkv, heads):
    B, N, D3 = qkv.shape
    D = D3 // 3
    out = torch.full((B, N, D), float("nan"), dtype=qkv.dtype, device=DEV)
    capi.check(capi.lib().moge_op_attention(qkv.data_ptr(), out.data_ptr(), B, N, D, heads, dt(qkv.dtype), stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,N,heads", [
    (16, 1370, 16),   # 1536 items, about 12 per CTA; the last item of every (image, head) has a dead second query tile
    (24, 129, 16),    # one valid key in the last K/V tile; the second query tile holds one row
    (12, 384, 12),    # the dead query tile starts exactly at the image's end
    (40, 100, 16),    # every item is half dead and holds a single K/V tile
])
def test_attention_many_items_per_cta(B, N, heads, dtype):
    qkv = _qkv(B, N, heads, dtype, B * N + heads)
    out = _attention(qkv, heads)
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4).unbind(0)
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, heads * 64)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < TOL[dtype]
    # block by block: (image, 64 query rows, head), half of a consumer warpgroup's query tile; the last block of an image lies
    # in or next to the item's dead query tile
    err, (img, qb, head) = worst_tile(out, ref, TILE_ATTENTION)
    whole = rel_l2(out, ref)
    last = qb == (N + 63) // 64 - 1
    print(f"tile-check attention {dtype} {(B, N, heads)}: whole {whole:.3e} worst {err:.3e} at image {img} head {head} "
          f"query block {qb}{' (last)' if last else ''} ratio {err / whole:.2f}")
    assert err < TILE_C * TOL[dtype], (f"image {img}, head {head}, query block {qb} (rows {64 * qb}..{min(64 * qb + 64, N) - 1}"
                                       f"{', the last block of the image' if last else ''}): error {err:.3e}, whole tensor "
                                       f"{whole:.3e}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_attention_image_independent_of_batch(dtype):
    """Image i computed in a batch of 9 (432 items over the SMs, other neighbours on its CTA) is bitwise equal to the same
    image computed alone (48 items)."""
    B, N, heads = 9, 1370, 16
    qkv = _qkv(B, N, heads, dtype, 11)
    batch = _attention(qkv, heads)
    for i in range(B):
        alone = _attention(qkv[i:i + 1].contiguous(), heads)
        assert torch.equal(alone[0], batch[i]), f"image {i}"
