#!/usr/bin/env python
"""Time the two scan publishers, immesh_lio_effect_cloud (publish_effect_world) and immesh_lio_registered_cloud
(publish_frame_world), on one of bench.py's workloads.

  python tools/scan_pub_bench.py --config C100k|C4|C5 [--scans 10]

The map is built and grown through the blocking step for the workload's warm-up scans.  Then every scan is followed by the calls a
node makes after map_incremental_grow: the effect cloud, the registered down-sampled scan (pts = NULL) and the registered dense scan
(the full-resolution host cloud, point_skip 1).  Median and p95 of the host clock around each blocking call, the count query and
the row copy included, and the rows per call.  Prints one JSON line with the GPU's name and power limit.  Writes nothing."""
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
    ap.add_argument("--config", default="C100k", choices=["C100k", "C1", "C2", "C3", "C4", "C5"])
    ap.add_argument("--scans", type=int, default=10)
    args = ap.parse_args()
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    warm = max(wl["map_warm"], 3)
    scans = bench.get_stream(wl, 1 + warm + args.scans)
    lio = api.Lio(wl["lio"])
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    k = 1
    for _ in range(warm):
        lio.step(scans[k]["body_ds"], scans[k]["dt"])
        k += 1
    calls = {"effect": lambda s: lio.effect_cloud()[0],
             "registered_ds": lambda s: lio.registered_cloud(None),
             "registered_dense": lambda s: lio.registered_cloud(s["body_full"])}
    ms = {c: [] for c in calls}
    rows = {c: [] for c in calls}
    for _ in range(args.scans):
        lio.step(scans[k]["body_ds"], scans[k]["dt"])
        for c, f in calls.items():
            t0 = time.perf_counter()
            r = f(scans[k])
            ms[c].append((time.perf_counter() - t0) * 1e3)
            rows[c].append(r.shape[0])
        k += 1
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"config": args.config, "gpu": gpu, "calls": args.scans,
                      **{c: {"median_ms": round(float(np.median(ms[c])), 4), "p95_ms": round(float(np.percentile(ms[c], 95)), 4),
                             "rows_per_call": round(float(np.mean(rows[c])), 1)} for c in calls}}))


if __name__ == "__main__":
    main()
