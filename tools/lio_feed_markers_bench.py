#!/usr/bin/env python
"""What recording the plane-map markers in the scan feed (immesh_lio_feed_markers_enable) costs the queued localization chain, on
bench.py's workloads, against what a node with voxel/pub_plane_en must do without it.

  python tools/lio_feed_markers_bench.py [--configs C100k,C4,C5] [--scans 30] [--rounds 3] [--no-profile]

The chain is the device front-end (immesh_lio_step_async_raw) on the full-resolution scans, already in HBM, with the scan feed on
(headers and states only, so that the markers are what differs).  After the map build one blocking immesh_voxelmap_plane_markers
publishes the first message, as a node does.  Numbers per configuration:
  scans_per_s off / on / blocking
                         the pipelined chain over --scans scans after a warm-up, host clock from the first enqueue to the end of the
                         last scan, alternated --rounds times in this one process: markers off; markers on, the records read after the
                         timed window; markers off with immesh_lio_wait and a blocking immesh_voxelmap_plane_markers after every scan
  rows_per_scan          marker rows the feed recorded per scan
  marker_kernels_us      device time per scan of each kernel the markers add (torch.profiler, CUDA activities, one run of its own)
Prints one JSON line with the GPU's name, power limit and SM clock limit, read in the same process.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MARKER_KERNELS = ("k_mark_begin", "k_pub_keys", "k_rs_hist_dev", "k_rs_scan_dev", "k_rs_scatter_dev", "k_pub_count", "k_pub_scan",
                  "k_mark_head", "k_pub_emit")


def bench_config(name, args):
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[name]
    n = args.scans
    W = 4
    scans = bench.get_stream(wl, 1 + W + n)
    d_full = [torch.from_numpy(np.ascontiguousarray(s["body_full"])).cuda() for s in scans]
    leaf = wl["lio"].filter_size_surf
    max_pts = max(s["body_full"].shape[0] for s in scans)

    def run(mode, profile=None):
        lio, vg = api.Lio(wl["lio"]), api.VoxelGrid(max_pts)
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        lio.feed_enable(max_scans=256, max_rows=0, effect=False, registered=0)
        if mode == "on":
            lio.feed_markers_enable(1 << 20)
        lio.plane_markers()

        def step(k):
            vg.step_async_raw(lio, d_full[k].data_ptr(), leaf, scans[k]["dt"], n=d_full[k].shape[0], stride=3, on_device=True)
            if mode == "blocking":
                lio.wait()
                lio.plane_markers()

        for k in range(1, 1 + W):
            step(k)
        lio.wait()
        torch.cuda.synchronize()
        if profile is not None:
            profile.start()
        t0 = time.perf_counter()
        for k in range(1 + W, 1 + W + n):
            step(k)
        lio.wait()
        ms = (time.perf_counter() - t0) * 1e3
        rows = 0
        if mode == "on":
            f = lio.feed_markers(W, wait=True)
            assert (f["scans"][:, 4] == 0).all(), "a scan lost its markers: enlarge the ring"
            rows = f["rows"].shape[0]
        if profile is not None:
            torch.cuda.synchronize()
            profile.stop()
        lio.close(); vg.close()
        return n / ms * 1e3, rows / n

    for mode in ("on", "off", "blocking"):   # warm-up: module loads, graph captures
        run(mode)
    rates = {"off": [], "on": [], "blocking": []}
    rows_per_scan = 0.0
    for _ in range(args.rounds):
        for mode in rates:
            r, rows = run(mode)
            rates[mode].append(r)
            if mode == "on":
                rows_per_scan = rows
    out = {**{f"scans_per_s_{m}": [round(r, 2) for r in v] for m, v in rates.items()}, "rows_per_scan": round(rows_per_scan, 1)}
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        prof = profile(activities=[ProfilerActivity.CUDA])
        run("on", prof)
        tot = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
                tot[e.key] = (getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0), e.count)

        def find(name):
            us = 0.0
            for key, (t, _) in tot.items():
                if key == name or key.startswith((name + "(", name + "<")) or f"::{name}(" in key:
                    us += t
            return us
        out["marker_kernels_us"] = {k: round(find(k) / n, 2) for k in MARKER_KERNELS}
        out["marker_kernels_us_total"] = round(sum(out["marker_kernels_us"].values()), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C100k,C4,C5")
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    out = {"scans": args.scans, "chain": "raw", "feed": "headers and states"}
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for name in args.configs.split(","):
        out[name] = bench_config(name, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
