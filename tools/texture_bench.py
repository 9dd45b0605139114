#!/usr/bin/env python
"""Time the textured mesh's selection (immesh_mesh_texture_select) on bench.py's workloads.

  python tools/texture_bench.py [--configs C100k,C3] [--scans 30] [--reps 3]

Each workload's stream is localized and meshed through the queued chain (step_async + push_frame_from_lio_async, inputs in HBM).
One camera per frame is posed from the frame's converged pose and a fixed extrinsic (looking along the sensor's +x, 10 cm ahead and
5 cm up), a pinhole with a 61-degree horizontal field of view, at 1224 x 1024 and at 2448 x 2048 (the paper's camera).  Then, on the
final mesh, the blocking call over every camera, timed with the host clock (median of --reps calls after a warm-up):
  ms_per_camera, total_s   the call's time over the number of cameras, and the whole call
  textured_share           textured facets over live facets
Prints one JSON line per workload with the GPU's name, power limit and SM clock limit.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R_EXT = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])   # OpenCV camera axes in the sensor frame: z ahead, x right, y down
T_EXT = np.array([0.1, 0.0, 0.05])


def run(config, n, reps):
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[config]
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]
    lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    poses = []
    for k in range(1, 1 + n):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        s = lio.get_state()
        poses.append((s[0:9].reshape(3, 3).copy(), s[9:12].copy()))
    lio.wait()
    mesh.wait()
    nt = mesh.counts()["n_triangles"]
    out = {"config": config, "frames": n, "cameras": n, "triangles": nt}
    for w, h in ((1224, 1024), (2448, 2048)):
        f = 0.85 * w
        cams = [(w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), R @ R_EXT, t + R @ T_EXT) for R, t in poses]
        r = mesh.texture_select(cams)   # warm-up
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            r = mesh.texture_select(cams)
            ts.append(time.perf_counter() - t0)
        sec = float(np.median(ts))
        out[f"{w}x{h}"] = dict(ms_per_camera=round(sec * 1e3 / n, 3), total_s=round(sec, 4),
                               textured_share=round(r["counts"]["textured"] / max(nt, 1), 4), cameras_used=r["counts"]["cameras_used"])
    lio.close()
    mesh.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C100k,C3")
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for c in args.configs.split(","):
        out = run(c, args.scans, args.reps)
        out["gpu"] = gpu
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
