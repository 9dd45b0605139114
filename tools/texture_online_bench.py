#!/usr/bin/env python
"""Time the texturing queued behind every frame (immesh_mesh_texture_enable) on bench.py's workloads.

  python tools/texture_online_bench.py [--configs C100k,C3] [--scans 30] [--reps 3]

Each workload's stream is localized and meshed through the queued chain (step_async + push_frame_from_lio_async, inputs in HBM) on
fresh handles, with the texturing off, on at 640 x 480 and on at 1224 x 1024 (rig: looking along the sensor's +x, 10 cm ahead and
5 cm up, a pinhole with a 61-degree horizontal field of view).  The three runs alternate --reps times in this one command; each run
is timed with the host clock from the first queued frame to the final wait, so a frame's time is that of the whole chain, which the
mesh stream paces.  Reported per setting: the median ms per frame, and for the texturing the median extra ms per frame over "off".
One JSON line per workload with the GPU's name, power limit and SM clock limit.  Writes nothing."""
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
SIZES = ((640, 480), (1224, 1024))


def chain(wl, scans, d_ds, d_full, size):
    """one run of the queued chain on fresh handles; size None: texturing off.  Returns (seconds, textured share)"""
    import torch
    import bench
    from immesh_b200 import api
    lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    if size:
        w, h = size
        f = 0.85 * w
        mesh.texture_enable((w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), R_EXT, T_EXT))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(1, len(scans)):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
    lio.wait()
    mesh.wait()
    sec = time.perf_counter() - t0
    share = None
    if size:
        c = mesh.texture_rows(vertices=False)["counts"]
        share = round(c["textured"] / max(c["textured"] + c["untextured"], 1), 4)
    lio.close()
    mesh.close()
    return sec, share


def run(config, n, reps):
    import torch
    import bench
    wl = bench.workloads()[config]
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]
    settings = [None] + list(SIZES)
    chain(wl, scans, d_ds, d_full, SIZES[-1])   # warm-up: modules, graphs of every shape
    times = {s: [] for s in settings}
    shares = {}
    for _ in range(reps):
        for s in settings:
            sec, share = chain(wl, scans, d_ds, d_full, s)
            times[s].append(sec * 1e3 / n)
            shares[s] = share
    out = {"config": config, "frames": n, "off_ms_per_frame": round(float(np.median(times[None])), 3)}
    for s in SIZES:
        extra = [a - b for a, b in zip(times[s], times[None])]
        out[f"{s[0]}x{s[1]}"] = dict(ms_per_frame=round(float(np.median(times[s])), 3), extra_ms_per_frame=round(float(np.median(extra)), 3),
                                     textured_share=shares[s])
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
