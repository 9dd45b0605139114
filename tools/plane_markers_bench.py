#!/usr/bin/env python
"""Time immesh_voxelmap_plane_markers (the plane-map publisher) on one of bench.py's workloads.

  python tools/plane_markers_bench.py --config C100k|C4|C5 [--scans 10]

The map is built and grown through the blocking step for the workload's warm-up scans with no marker call, so the first call
publishes every plane fitted since the build (`first_call`).  Then every scan is followed by one call: median and p95 of the
host clock around the blocking call (the row copy included), rows and roots walked per call.  Prints one JSON line with the
GPU's name and power limit.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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
    t0 = time.perf_counter()
    rows, c = lio.plane_markers()
    first = {"ms": round((time.perf_counter() - t0) * 1e3, 4), "rows": int(rows.shape[0]), "roots_walked": c["roots_walked"],
             "map_roots": lio.counts()["roots"], "scans_since_build": warm}
    ms, n, walked, roots = [], [], [], []
    for _ in range(args.scans):
        lio.step(scans[k]["body_ds"], scans[k]["dt"])
        k += 1
        t0 = time.perf_counter()
        rows, c = lio.plane_markers()
        ms.append((time.perf_counter() - t0) * 1e3)
        n.append(rows.shape[0])
        walked.append(c["roots_walked"])
        roots.append(lio.counts()["roots"])
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"config": args.config, "gpu": gpu, "calls": args.scans,
                      "median_ms": round(float(np.median(ms)), 4), "p95_ms": round(float(np.percentile(ms, 95)), 4),
                      "rows_per_call": round(float(np.mean(n)), 1), "roots_walked_per_call": round(float(np.mean(walked)), 1),
                      "map_roots": int(roots[-1]), "first_call": first}))


if __name__ == "__main__":
    main()
