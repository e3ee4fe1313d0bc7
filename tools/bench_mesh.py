"""Mesh export after infer(): `moge_b200.mesh.mesh_from_output` (edge cleaning, mesh, colours, UVs, normals, OpenGL flips) on
device-resident infer()-style outputs (synthetic_mesh_case: piecewise-planar scenes, +inf off the mask, unit normals, uint8
image) at 518x518, 1024x768 and 2048x1365, batch 1 and 8, against what the reference CLI does today.  Prints one JSON line with
the GPU name and power limit read in the same run.

    python tools/bench_mesh.py [--iters 20] [--host-iters 3]

Per row, in ms per image (median, min and max of separately timed calls after a warm-up call):
  - engine_device: CUDA events around the call's kernels and its counts copy enqueued back to back (outputs allocated at the
    sizes a previous call found), i.e. device time without the host's wait, allocation and launch work;
  - engine_end_to_end: a host clock around mesh_from_output plus the copy of every result array into pinned host memory,
    ended by a device synchronise;
  - host_numpy: the reference CLI's path: the dense maps (points, depth, mask, normal) copied to the host, then the numpy
    restatement of utils3d's depth_map_edge + build_mesh_from_map + the flips (oracle/utils3d_mesh.py) on the host cores, one
    image at a time.  It is a restatement of utils3d, not utils3d itself.
bytes: what the kernels must move (each input read once, each output written once; see kernel_bytes), and the rate over
engine_device against NVIDIA's 3.35 TB/s H100 SXM data-sheet figure (a fraction of that figure, not of a reached peak).
Agreement with the host path is checked bitwise for the first and last image at every timed size.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from measure import cuda_samples, gpu_identity, summary  # noqa: E402
from moge_b200 import mesh as M  # noqa: E402
from moge_b200.synthetic import synthetic_mesh_case  # noqa: E402
from oracle import utils3d_mesh as O  # noqa: E402

WORKLOADS = [(518, 518), (768, 1024), (1365, 2048)]
BATCHES = (1, 8)
HBM_BYTES_PER_S = 3.35e12


def kernel_bytes(B, H, W, nv, nq):
    """Bytes the passes must move: edge (depth 4 + mask 1 read, cleaned mask 1 written), count (mask 1), vertex pass (mask 1,
    index map 4 written; per kept vertex points 12 + colour 3 + normal 12 read, 12 + 12 + 8 + 12 written), face pass (mask 1,
    index map 4 read; 24 written per kept quad)."""
    px = B * H * W
    return px * (6 + 1 + 5 + 5) + nv * (27 + 44) + nq * 24


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-iters", type=int, default=3)
    a = ap.parse_args()
    result = {"metric": "mesh_from_output_ms_per_image", **gpu_identity(),
              "host_comparator": "numpy restatement of utils3d (oracle/utils3d_mesh.py), not utils3d itself",
              "host_cpus": os.cpu_count(), "hbm_data_sheet_bytes_per_s": HBM_BYTES_PER_S, "rows": []}
    for H, W in WORKLOADS:
        out_cpu, img_cpu = synthetic_mesh_case(0, max(BATCHES), H, W)
        host = None
        for B in BATCHES:
            out = {k: v[:B].to("cuda") for k, v in out_cpu.items()}
            image = img_cpu[:B].to("cuda")
            res = M.mesh_from_output(out, image)                                     # warm-up; sizes for the device chain
            torch.cuda.synchronize()
            nv = sum(r["vertices"].shape[0] for r in res)
            nq = sum(r["faces"].shape[0] for r in res) // 2

            d, m = out["depth"].contiguous(), out["mask"].contiguous().view(torch.uint8)
            maps = M._output_maps(out["points"], M._Map(image, M.capi.MESH_U8_UNIT, 3), out["normal"])
            faces = torch.empty(2 * nq, 3, dtype=torch.int32, device="cuda")
            rows = [torch.empty(nv, mp.channels, device="cuda") for mp in maps]

            def device_chain():
                cleaned = M._edge(d, None, m, None, 0.04, 3)
                ws, totals, _, _ = M._count(cleaned, B, H, W, d.device)
                M._emit(cleaned, B, H, W, maps, True, ws, totals, faces, rows)

            dev_s = summary(cuda_samples(device_chain, a.iters), B)

            def end_to_end():
                r = M.mesh_from_output(out, image)
                pinned = [{k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True).copy_(v, non_blocking=True) for k, v in x.items()}
                          for x in r]
                torch.cuda.synchronize()
                return pinned

            e2e = []
            for _ in range(a.iters):
                t0 = time.perf_counter()
                pinned = end_to_end()
                e2e.append((time.perf_counter() - t0) * 1e3 / B)

            if host is None:                         # the host path is per image: timed once per size
                hs = []
                for _ in range(a.host_iters):
                    t0 = time.perf_counter()
                    maps_h = {k: out[k][0].cpu().numpy() for k in ("points", "depth", "mask", "normal")}
                    want0 = O.mesh_from_output(maps_h["points"], maps_h["depth"], maps_h["mask"], img_cpu[0].numpy(), maps_h["normal"])
                    hs.append((time.perf_counter() - t0) * 1e3)
                host = summary(hs)
            agree = True
            for b in sorted({0, B - 1}):
                want = want0 if b == 0 else O.mesh_from_output(out_cpu["points"][b].numpy(), out_cpu["depth"][b].numpy(),
                                                               out_cpu["mask"][b].numpy(), img_cpu[b].numpy(), out_cpu["normal"][b].numpy())
                got = pinned[b]
                agree &= np.array_equal(got["faces"].numpy(), want["faces"]) and np.array_equal(got["mask_cleaned"].numpy(), want["mask_cleaned"])
                for k in ("vertices", "vertex_colors", "vertex_uvs", "vertex_normals"):
                    agree &= got[k].numpy().tobytes() == want[k].tobytes()
            nbytes = kernel_bytes(B, H, W, nv, nq)
            gbs = nbytes / B / (dev_s["median"] * 1e-3) / 1e9
            row = {"H": H, "W": W, "batch": B, "vertices_per_image": nv / B, "triangles_per_image": 2 * nq / B,
                   "engine_device_ms_per_image": dev_s, "engine_end_to_end_ms_per_image": summary(e2e),
                   "host_numpy_ms_per_image": host, "kernel_bytes_per_image": nbytes / B, "kernel_gb_per_s": gbs,
                   "fraction_of_3_35_tb_per_s": gbs * 1e9 / HBM_BYTES_PER_S, "bitwise_agreement": bool(agree)}
            result["rows"].append(row)
            print(json.dumps(row), file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
