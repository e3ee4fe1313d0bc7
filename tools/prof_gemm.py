"""Micro-benchmark of the wgmma GEMM kernel through the C ABI (moge_op_linear): encoder shapes of ViT-L at
batch 32 x 1370 tokens.  Prints TFLOP/s per epilogue."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from moge_b200 import capi

L = capi.lib()
dev = "cuda"
M = int(os.environ.get("M", 43840))
shapes = [("qkv", 3072, 1024, 0), ("fc1+gelu", 4096, 1024, 1), ("fc2+resid", 1024, 4096, 2), ("proj+resid", 1024, 1024, 2)]
iters = int(os.environ.get("ITERS", 5))
for name, N, K, epi in shapes:
    x = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev)
    g = torch.randn(N, device=dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if epi == 2 else torch.float16)
    st = capi.current_stream()
    for _ in range(2):
        capi.check(L.moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), g.data_ptr(), out.data_ptr(), M, N, K, epi, capi.F16, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        capi.check(L.moge_op_linear(x.data_ptr(), w.data_ptr(), b.data_ptr(), g.data_ptr(), out.data_ptr(), M, N, K, epi, capi.F16, st))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"{name:12s} M={M} N={N} K={K}: {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)
    if os.environ.get("CUBLAS"):
        ref = torch.empty(M, N, device=dev, dtype=torch.float16)
        for _ in range(2): torch.matmul(x, w.t(), out=ref)
        torch.cuda.synchronize(); e0.record()
        for _ in range(iters): torch.matmul(x, w.t(), out=ref)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        print(f"   cuBLAS fp16 (no epilogue)        : {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)
