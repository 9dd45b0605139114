#!/usr/bin/env python
"""What the scan feed (immesh_lio_feed_enable) costs the queued localization chain, on one of bench.py's workloads.

  python tools/lio_feed_bench.py [--config C100k|C4] [--scans 30] [--rounds 3] [--no-profile]

The chain is the device front-end (immesh_lio_step_async_raw: VoxelGrid + predict + IESKF + map update) on the full-resolution scans,
already in HBM, with the feed recording every scan at registered = 2 (the full scan) and effect = 1, point_skip 1.  Numbers:
  scans_per_s off / on / on_read
                         the pipelined chain over --scans scans after a warm-up, host clock from the first enqueue to the end of the
                         last scan (immesh_lio_wait), alternated --rounds times in this one process: feed off; feed on, the records
                         read after the timed window (the cost of recording); feed on, the finished scans read with wait = 0
                         after every enqueue, as a node would (the rows copied to the host every scan included)
  feed_kernels_us        device time per scan of each kernel the feed adds (torch.profiler, CUDA activities, one run of its own),
                         and k_rs_scan's extra launches; rows_per_scan and the bytes the record writes per scan
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

FEED_KERNELS = ("k_eff_count", "k_feed_head", "k_eff_emit", "k_reg_gather", "k_feed_done")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C100k", choices=["C100k", "C4"])
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    n = args.scans
    W = 4
    scans = bench.get_stream(wl, 1 + W + n)
    d_full = [torch.from_numpy(np.ascontiguousarray(s["body_full"])).cuda() for s in scans]
    leaf = wl["lio"].filter_size_surf
    max_pts = max(s["body_full"].shape[0] for s in scans)

    def run(feed, profile=None, read_each=True):
        lio, vg = api.Lio(wl["lio"]), api.VoxelGrid(max_pts)
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        if feed:
            lio.feed_enable(max_scans=256, max_rows=1 << 24, effect=True, registered=2, point_skip=1)

        def step(k):
            vg.step_async_raw(lio, d_full[k].data_ptr(), leaf, scans[k]["dt"], n=d_full[k].shape[0], stride=3, on_device=True)

        for k in range(1, 1 + W):
            step(k)
        lio.wait()
        since = W if feed else 0
        rows = 0
        torch.cuda.synchronize()
        if profile is not None:
            profile.start()
        t0 = time.perf_counter()
        for k in range(1 + W, 1 + W + n):
            step(k)
            if feed and read_each:
                f = lio.feed(since, wait=False)
                since = f["newest_finished"] if f["scans"].shape[0] else since
                rows += f["rows"].shape[0]
        lio.wait()
        ms = (time.perf_counter() - t0) * 1e3
        if feed:   # the scans not read yet; inside the timed window only when the loop reads as it goes
            f = lio.feed(since, wait=True)
            rows += f["rows"].shape[0]
            if read_each:
                ms = (time.perf_counter() - t0) * 1e3
        if profile is not None:
            torch.cuda.synchronize()
            profile.stop()
        lio.close(); vg.close()
        return n / ms * 1e3, rows / n

    run(True); run(False)   # warm-up: module loads, graph captures
    rates = {"off": [], "on": [], "on_read": []}
    rows_per_scan = 0.0
    for _ in range(args.rounds):
        for mode in rates:
            r, rows = run(mode != "off", read_each=mode == "on_read")
            rates[mode].append(r)
            if mode != "off":
                rows_per_scan = rows
    out = {"config": args.config, "scans": n, "registered": 2, "effect": 1,
           **{f"scans_per_s_{m}": [round(r, 2) for r in v] for m, v in rates.items()},
           "rows_per_scan": round(rows_per_scan, 1),
           "record_bytes_per_scan": int(348 * 8 + 12 * 8 + rows_per_scan * (16 + 4))}
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        per = {}
        for on in (False, True):
            prof = profile(activities=[ProfilerActivity.CUDA])
            run(on, prof, read_each=False)
            tot = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
                    tot[e.key] = (getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0), e.count)
            per[on] = tot

        def find(tot, name):
            us, cnt = 0.0, 0
            for key, (t, c) in tot.items():
                if key == name or key.startswith((name + "(", name + "<")) or f"::{name}(" in key:
                    us += t
                    cnt += c
            return us, cnt
        out["feed_kernels_us"] = {}
        for name in FEED_KERNELS:
            us, cnt = find(per[True], name)
            out["feed_kernels_us"][name] = round(us / n, 2)
        on_us, _ = find(per[True], "k_rs_scan")
        off_us, _ = find(per[False], "k_rs_scan")
        out["feed_kernels_us"]["k_rs_scan_extra"] = round((on_us - off_us) / n, 2)
        out["feed_kernels_us_total"] = round(sum(out["feed_kernels_us"].values()), 2)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
