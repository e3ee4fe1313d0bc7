"""Micro-benchmark of decoder convolutions / attention through the C ABI at the ViT-L batch-32 shapes."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from moge_b200 import capi
L = capi.lib(); dev = "cuda"
B = int(os.environ.get("B", 32))
what = os.environ.get("WHAT", "conv,attn")
def timeit(fn, iters=3):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters
if "conv" in what:
    for (H, W, C, skip, both) in [(74, 74, 256, False, False), (74, 74, 256, True, True), (148, 148, 128, False, False), (148, 148, 128, True, True), (296, 296, 64, False, False), (296, 296, 64, True, True)]:
        Hp, Wp = H + 2, W + 2
        x = torch.randn(B, Hp, Wp, C, device=dev).half()
        w = (torch.randn(C, C, 3, 3, device=dev) / (9 * C) ** 0.5)
        b = torch.randn(C, device=dev)
        sk = torch.randn(B, Hp, Wp, C, device=dev).half() if skip else None
        o0 = torch.empty(B, Hp, Wp, C, device=dev, dtype=torch.float16)
        o1 = torch.empty(B, Hp, Wp, C, device=dev, dtype=torch.float16) if both else None
        st = capi.current_stream()
        f = lambda: capi.check(L.moge_op_conv(x.data_ptr(), w.data_ptr(), b.data_ptr(), capi.ptr(sk), capi.ptr(o0) if (both or not skip) else None, capi.ptr(o1) if both else (None if not skip else capi.ptr(o0)), B, H, W, C, C, 9, 0, capi.F16, st))
        ms = timeit(f)
        fl = 2.0 * B * H * W * C * C * 9
        by = B * H * W * C * 2 * (1 + (1 if skip else 0) + (2 if both else 1))
        print(f"conv3x3 {H}x{W} C={C} skip={skip} both={both}: {ms:.3f} ms {fl/ms/1e9:.0f} TF/s {by/ms/1e6:.0f} GB/s (incl. weight pack)", flush=True)
if "attn" in what:
    N, heads = 1370, 16
    D = heads * 64
    qkv = torch.randn(B, N, 3 * D, device=dev).half()
    out = torch.empty(B, N, D, device=dev, dtype=torch.float16)
    st = capi.current_stream()
    ms = timeit(lambda: capi.check(L.moge_op_attention(qkv.data_ptr(), out.data_ptr(), B, N, D, heads, capi.F16, st)))
    print(f"attention B={B} N={N} heads={heads}: {ms:.3f} ms {4.0*B*N*N*D/ms/1e9:.0f} TF/s", flush=True)
    import torch.nn.functional as F
    q, k, v = qkv.reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4).unbind(0)
    ms = timeit(lambda: F.scaled_dot_product_attention(q, k, v))
    print(f"  torch SDPA (library) : {ms:.3f} ms {4.0*B*N*N*D/ms/1e9:.0f} TF/s", flush=True)
