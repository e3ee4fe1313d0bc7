"""Mesh export after infer_panorama(): `moge_b200.mesh.mesh_from_panorama` (normals, depth-and-normal edge cleaning, triangles,
colours, UVs) at 2048 x 1024 and 4096 x 2048, on the analytic room (synthetic_panorama_scene) and on infer_panorama() output of a
synthetic-weight MoGe-1 ViT-S, against the host path the reference script takes.  Prints one JSON line with the GPU name and
power limit read in the same run.

    python tools/bench_panorama_mesh.py [--iters 20] [--host-iters 2] [--out FILE]

Per row, in ms (median, min and max of separately timed calls after a warm-up call):
  - engine_device: CUDA events around the call's kernels and its counts copy enqueued back to back (outputs allocated at the
    sizes a previous call found), i.e. device time without the host's wait, allocation and launch work; split into `clean`
    (depth edge, normal map, normal edge with the fused cleaning) and `mesh` (count, scan, emit);
  - engine_end_to_end: a host clock around mesh_from_panorama plus the copy of every result array into pinned host memory,
    ended by a device synchronise;
  - host_numpy: the panorama script's path: the maps copied to the host, then the numpy restatement of utils3d's
    point_map_to_normal_map, depth_map_edge, normal_map_edge and build_mesh_from_map (oracle/utils3d_normals.py) on the host
    cores.  It is a restatement of utils3d, not utils3d itself.
Agreement: the engine's cleaned mask against the restatement's (pixels that differ, and pixels whose angle is within 1e-6 of
the threshold, where they may), and the mesh bitwise against build_mesh_from_map restated on the engine's own cleaned mask.
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

from measure import gpu_identity, summary  # noqa: E402
from moge_b200 import mesh as M  # noqa: E402
from moge_b200.synthetic import synthetic_panorama, synthetic_panorama_scene  # noqa: E402
from oracle import utils3d_mesh as OM  # noqa: E402
from oracle import utils3d_normals as O  # noqa: E402

SIZES = [(1024, 2048), (2048, 4096)]
DEV = "cuda"


def summary_ms(samples):
    """summary() to the microsecond"""
    return {k: round(v, 3) for k, v in summary(samples).items()}


def v1_model():
    from moge.model.v1 import MoGeModel
    from moge_b200.configs import v1_model_config
    from moge_b200.synthetic import make_v1_state_dict
    cfg = v1_model_config("vits")
    m = MoGeModel(**cfg)
    m.load_state_dict(make_v1_state_dict(cfg, 7, well_posed=True))
    return m.to(DEV).eval()


def measure(out, image, iters, host_iters):
    H, W = out["depth"].shape
    res = M.mesh_from_panorama(out, image)                  # warm-up; sizes for the device chain
    torch.cuda.synchronize()
    nv, nf = res["vertices"].shape[0], res["faces"].shape[0]
    d, p, m = out["depth"].contiguous()[None], out["points"].contiguous()[None], out["mask"].contiguous().view(torch.uint8)[None]
    maps = [M._Map(p, M.capi.MESH_F32, 3), M._Map(image.contiguous(), M.capi.MESH_U8_UNIT, 3), M._Map(None, M.capi.MESH_UV, 2)]
    faces = torch.empty(nf, 3, dtype=torch.int32, device=DEV)
    rows = [torch.empty(nv, mp.channels, device=DEV) for mp in maps]

    def device_chain(ev):
        ev[0].record()
        de = M._edge(d, None, None, None, 0.03, 3)
        normals, nmask = M._normal_map(p, m)
        cleaned = M._normal_edge(normals, nmask, de, m, M.PANORAMA_NORMAL_TOL, 3)
        ev[1].record()
        ws, totals, _, _ = M._count(cleaned, 1, H, W, d.device)
        M._emit(cleaned, 1, H, W, maps, True, ws, totals, faces, rows)
        ev[2].record()

    dev, clean, mesh = [], [], []
    for it in range(iters + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        device_chain(ev)
        torch.cuda.synchronize()
        if it:
            dev.append(ev[0].elapsed_time(ev[2]))
            clean.append(ev[0].elapsed_time(ev[1]))
            mesh.append(ev[1].elapsed_time(ev[2]))

    e2e = []
    for _ in range(iters):
        t0 = time.perf_counter()
        r = M.mesh_from_panorama(out, image)
        pinned = {k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True).copy_(v, non_blocking=True) for k, v in r.items()}
        torch.cuda.synchronize()
        e2e.append((time.perf_counter() - t0) * 1e3)

    hs = []
    for _ in range(host_iters):
        t0 = time.perf_counter()
        hp, hd, hm, hi = out["points"].cpu().numpy(), out["depth"].cpu().numpy(), out["mask"].cpu().numpy(), image.cpu().numpy()
        want = O.mesh_from_panorama(hp, hd, hm, hi)
        hs.append((time.perf_counter() - t0) * 1e3)

    cleaned = pinned["mask_cleaned"].numpy()
    normals, nm = O.point_map_to_normal_map(hp, hm)
    angle = O.normal_angle_map(normals, 3, nm)
    with np.errstate(invalid="ignore"):
        near = (angle > np.deg2rad(5 * (1 - 1e-6))) != (angle > np.deg2rad(5 * (1 + 1e-6)))
    mesh_want = OM.build_mesh_from_map(hp, hi.astype(np.float32) / 255, OM.uv_map(H, W), mask=cleaned, tri=True)
    bitwise = np.array_equal(pinned["faces"].numpy(), mesh_want[0]) and all(
        pinned[k].numpy().tobytes() == w.tobytes() for k, w in zip(("vertices", "vertex_colors", "vertex_uvs"), mesh_want[1:]))
    return {"size": f"{W}x{H}", "vertices": nv, "triangles": nf, "pixels_cleaned": int((hm & ~cleaned).sum()),
            "engine_device_ms": summary_ms(dev), "engine_device_clean_ms": summary_ms(clean),
            "engine_device_mesh_ms": summary_ms(mesh), "engine_end_to_end_ms": summary_ms(e2e), "host_numpy_ms": summary_ms(hs),
            "agreement": {"mask_cleaned_mismatch": int((cleaned != want["mask_cleaned"]).sum()), "pixels_near_threshold": int(near.sum()),
                          "mesh_bitwise_on_engine_mask": bool(bitwise),
                          "mesh_bitwise_vs_host": bool(np.array_equal(pinned["faces"].numpy(), want["faces"])
                                                       and pinned["vertices"].numpy().tobytes() == want["vertices"].tobytes())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-iters", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    result = {"metric": "mesh_from_panorama_ms", **gpu_identity(), "host_cpus": os.cpu_count(),
              "host_comparator": "numpy restatement of utils3d (oracle/utils3d_normals.py), not utils3d itself", "rows": []}
    model = None
    for H, W in SIZES:
        points, depth, mask, image = synthetic_panorama_scene(H, W, 3)
        out = {"points": torch.from_numpy(points).to(DEV), "depth": torch.from_numpy(depth).to(DEV), "mask": torch.from_numpy(mask).to(DEV)}
        row = dict(measure(out, torch.from_numpy(image).to(DEV), a.iters, a.host_iters), input="analytic room")
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        from moge_b200.panorama import infer_panorama
        model = model or v1_model()
        img = torch.from_numpy(synthetic_panorama(H, W, 1)).to(DEV)
        out = infer_panorama(model, img)
        row = dict(measure(out, img, a.iters, a.host_iters), input="infer_panorama, MoGe-1 ViT-S synthetic weights")
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
