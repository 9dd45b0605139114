#!/usr/bin/env python
"""Time the LiDAR point-cloud reinforcement (immesh_mesh_reinforce_enable) on one of bench.py's workloads, reference camera (640 x 480,
focus 400, z range 0.1 .. 1500, win 1).

  python tools/reinforce_bench.py [--config C100k] [--scans 24] [--rounds 3]

Three numbers, each on the same scans:
  queued_ms / blocking_ms   per frame: the device time of the queued chain (sum of the k_rf_* kernels, CUDA events of the library's
                            profiler over a stream of direct launches) against the host clock around immesh_mesh_render_depth at the
                            same pose after the same frame, in a pass of its own without the profiler (the blocking call: waits for
                            the mesh stream, allocates, runs the same tiled kernels, copies the result back, frees)
  tiled_ms                  per image: the tiled rasteriser (k_rf_count + k_rf_scan + k_rf_fill + k_rf_tile), from the profiler run
  scans_per_s on / off      the pipelined, graph-replayed stream (step_async + push_frame_from_lio_async, inputs in HBM), timed with
                            pipeline_mark_begin / _end, reinforcement on and off alternated `rounds` times
Prints one JSON line with the GPU's name, power limit and SM clock limit.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C100k")
    ap.add_argument("--scans", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    n = args.scans
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]
    K = api.reinforce_intrinsics(640, 480)

    def handles(reinforce):
        lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        if reinforce:
            mesh.reinforce_enable()
        return lio, mesh

    # ---- the queued chain per frame, profiler on (direct launches)
    lio, mesh = handles(True)
    api.profile_enable(True)
    for k in range(1, 1 + n):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        mesh.reinforced_cloud()   # read every frame, as in the pass below
    lio.wait()
    mesh.wait()
    rep = api.profile_report()
    api.profile_enable(False)
    lio.close(); mesh.close()
    rf = {k: v for k, v in rep.items() if k.startswith("k_rf_")}
    tiled = sum(rep[k][0] for k in ("k_rf_count", "k_rf_scan", "k_rf_fill", "k_rf_tile")) / n   # k_rf_scan runs twice per frame

    # ---- the blocking call after every frame at the pose the frame used, profiler off
    lio, mesh = handles(True)
    blocking = []
    for k in range(1, 1 + n):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        d, p, x, R, t = mesh.reinforced_cloud()
        t0 = time.perf_counter()
        dr, pr, xr = mesh.render_depth(K, 640, 480, 0.1, 1500.0, R, t)
        blocking.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(d.view(np.uint32), dr.view(np.uint32)) and np.array_equal(x, xr), k
    lio.wait()
    mesh.wait()
    out = {
        "config": args.config, "frames": n, "points_last_frame": int(len(p)), "triangles_last_frame": mesh.counts()["n_triangles"],
        "queued_ms_per_frame": round(sum(v[0] for v in rf.values()) / n, 4),
        "blocking_ms_per_frame": round(float(np.median(blocking[n // 2:])), 4),
        "tiled_ms": round(tiled, 4),
        "rf_kernels_ms_per_frame": {k: round(v[0] / n, 4) for k, v in sorted(rf.items())},
    }
    lio.close(); mesh.close()

    # ---- pipelined stream, reinforcement on / off alternated
    def stream(reinforce):
        lio, mesh = handles(reinforce)
        W = 4
        for k in range(1, 1 + W):
            lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        lio.wait(); mesh.wait()
        torch.cuda.synchronize()
        api.pipeline_mark_begin(lio)
        for k in range(1 + W, 1 + n):
            lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        ms = api.pipeline_mark_end(lio, mesh)
        lio.wait(); mesh.wait()
        lio.close(); mesh.close()
        return (n - W) / ms * 1e3

    rates = {True: [], False: []}
    for _ in range(args.rounds):
        for on in (False, True):
            rates[on].append(stream(on))
    out["scans_per_s_off"] = [round(r, 2) for r in rates[False]]
    out["scans_per_s_on"] = [round(r, 2) for r in rates[True]]
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
