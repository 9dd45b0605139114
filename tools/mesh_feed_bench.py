#!/usr/bin/env python
"""What the mesh frame feed (immesh_mesh_feed_enable) costs the queued chain, on one of bench.py's workloads.

  python tools/mesh_feed_bench.py [--config C100k|C4] [--frames 30] [--rounds 3] [--no-profile]

The chain is the device front-end (immesh_lio_step_async_raw) on the full-resolution scans already in HBM, each scan handed to the
mesher with immesh_mesh_push_frame_from_lio_async.  Settings, each run with the feed off and on, alternated --rounds times in this
one process:
  plain           no reinforcement, no view; the feed records headers and poses only
  points          the reinforcement at the reference camera (640 x 480, focus 400); the feed also records its points and pixels
  images          the reinforcement and the queued view (640 x 480, height colour); the feed also records the view's rgba and depth
  frames_per_s    host clock from the first enqueue to the end of the last frame, over --frames frames after a warm-up; the records
                  are read once, after the timed window (the cost of recording)
  feed_kernels_us device time per frame of each kernel the feed adds (torch.profiler, CUDA activities, a run of its own per setting)
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

FEED_KERNELS = ("k_mfeed_begin", "k_mfeed_head", "k_mfeed_points", "k_mfeed_image", "k_mfeed_done")
SETTINGS = ("plain", "points", "images")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C100k", choices=["C100k", "C4"])
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    n = args.frames
    W = 4
    scans = bench.get_stream(wl, 1 + W + n)
    d_full = [torch.from_numpy(np.ascontiguousarray(s["body_full"])).cuda() for s in scans]
    leaf = wl["lio"].filter_size_surf
    max_pts = max(s["body_full"].shape[0] for s in scans)

    def run(setting, feed, profile=None):
        lio, vg, mesh = api.Lio(wl["lio"]), api.VoxelGrid(max_pts), api.Mesh(wl["mesh"])
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        if setting in ("points", "images"):
            mesh.reinforce_enable(width=640, height=480)
        if setting == "images":
            mesh.view_enable(width=640, height=480, color_by_height=True)
        if feed:
            mesh.feed_enable(max_frames=256, max_rows=(1 << 24) if setting != "plain" else 0, max_images=64 if setting == "images" else 0,
                             depth=setting == "images")

        def frame(k):
            vg.step_async_raw(lio, d_full[k].data_ptr(), leaf, scans[k]["dt"], n=d_full[k].shape[0], stride=3, on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)

        for k in range(1, 1 + W):
            frame(k)
        lio.wait()
        mesh.wait()
        torch.cuda.synchronize()
        if profile is not None:
            profile.start()
        t0 = time.perf_counter()
        for k in range(1 + W, 1 + W + n):
            frame(k)
        lio.wait()
        mesh.wait()
        ms = (time.perf_counter() - t0) * 1e3
        rows = 0
        if feed:
            f = mesh.feed(W, wait=True)
            assert f["frames"].shape[0] == n
            rows = f["points"].shape[0]
        if profile is not None:
            torch.cuda.synchronize()
            profile.stop()
        mesh.close(); lio.close(); vg.close()
        return n / ms * 1e3, rows / n

    for s in SETTINGS:   # warm-up: module loads, graph captures
        run(s, True)
        run(s, False)
    rates = {f"{s}_{m}": [] for s in SETTINGS for m in ("off", "on")}
    rows_per_frame = 0.0
    for _ in range(args.rounds):
        for s in SETTINGS:
            for m in ("off", "on"):
                r, rows = run(s, m == "on")
                rates[f"{s}_{m}"].append(r)
                if s == "points" and m == "on":
                    rows_per_frame = rows
    out = {"config": args.config, "frames": n, **{f"frames_per_s_{k}": [round(r, 2) for r in v] for k, v in rates.items()},
           "points_per_frame": round(rows_per_frame, 1),
           "record_bytes_per_frame": {"plain": 22 * 8 + 36 * 8, "points": int(22 * 8 + 36 * 8 + rows_per_frame * 16),
                                      "images": int(22 * 8 + 36 * 8 + rows_per_frame * 16 + 640 * 480 * 8)}}
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        out["feed_kernels_us"] = {}
        for s in SETTINGS:
            prof = profile(activities=[ProfilerActivity.CUDA])
            run(s, True, prof)
            per = {}
            for e in prof.key_averages():
                t = getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0)
                for name in FEED_KERNELS:
                    if e.key == name or e.key.startswith(name + "(") or f"::{name}(" in e.key:
                        per[name] = per.get(name, 0.0) + t
            out["feed_kernels_us"][s] = {k: round(v / n, 2) for k, v in per.items()}
            out["feed_kernels_us"][s]["total"] = round(sum(per.values()) / n, 2)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
