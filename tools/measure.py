"""Measurement helpers shared by the tools/ scripts: which card the timings ran on, one CUDA-event timing loop and its
summary."""
import os
import subprocess
import sys

import torch


def gpu_identity(device=0):
    """{"gpu": name, "power_limit_w": float or None} of `device`, the card the timings run on.

    The power limit is asked of nvidia-smi by the device's UUID: nvidia-smi ignores CUDA_VISIBLE_DEVICES, so a row index
    could name another card.  It is None when nvidia-smi is missing or does not answer.  Exits with one message when no
    CUDA device is visible."""
    if not torch.cuda.is_available():
        sys.exit(f"{os.path.basename(sys.argv[0])} measures on an H100; no CUDA device is visible")
    uuid = str(torch.cuda.get_device_properties(device).uuid)
    uuid = uuid if uuid.startswith("GPU-") else "GPU-" + uuid
    try:
        q = subprocess.run(["nvidia-smi", f"--id={uuid}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip())
    except (OSError, subprocess.SubprocessError, ValueError):
        power = None
    return {"gpu": torch.cuda.get_device_name(device), "power_limit_w": power}


def cuda_samples(fn, iters, warmup=1):
    """Milliseconds of each of `iters` calls of fn: `warmup` untimed calls and a device synchronise first, then per call a
    CUDA event pair around fn() and a device synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    samples = []
    for _ in range(iters):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        torch.cuda.synchronize()
        samples.append(start.elapsed_time(end))
    return samples


def summary(samples, per=1):
    """{median, min, max, samples} of the samples divided by `per` (e.g. images per call); the median is sorted[n // 2]."""
    s = sorted(x / per for x in samples)
    return {"median": s[len(s) // 2], "min": s[0], "max": s[-1], "samples": len(s)}
