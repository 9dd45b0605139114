"""Cost of growing the VoxelMap pools on the device (immesh_lio_reserve / immesh_lio_set_growth), on one GPU.

  1. One doubling per pool of `size` records on an EMPTY handle, by immesh_lio_reserve: the cost of the allocation, the clearing of
     the new table and the free (the records a full pool would copy are not measured here).
  2. The hdl64loop stream from small capacities with automatic growth against a pre-sized handle: scans/s, growths, the total and
     the largest pause (step latency above the pre-sized handle's median), p95 step latency, device bytes at the end.
Prints one JSON object; --out also writes it to a file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from immesh_b200 import api, synth  # noqa: E402
from pool_growth_common import first_scan_use, start, tiny_config  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the measurement itself does not depend on it
        return f"unavailable ({e})"


def one_doubling(lib, pool, size):
    """ms of immesh_lio_reserve doubling `pool` of `size` records (mean of 3), on a handle whose other pools are minimal"""
    mi = 1 << 20
    cfg = api.LioConfig(hash_capacity_log2=10, max_nodes=1024, max_chunks=1024, max_scan_points=1 << 16)
    if pool == "root_hash":
        cfg.hash_capacity_log2 = size.bit_length() - 1
    elif pool == "nodes":
        cfg.max_nodes = size
    else:
        cfg.max_chunks = size
    times = []
    for _ in range(3):
        h = api.Lio(cfg, lib=lib)
        c = h.capacity()
        t0 = time.perf_counter()
        if pool == "root_hash":
            h.reserve(c["root_slots"] * 2, 0, 0)
        elif pool == "nodes":
            h.reserve(0, c["nodes_cap"] * 2, 0)
        else:
            h.reserve(0, 0, c["chunks_cap"] * 2)
        times.append((time.perf_counter() - t0) * 1e3)
        h.close()
    # an empty pool: the time is the allocation, the clearing of the new table and the free -- no record is migrated, so no
    # migration bandwidth is derived from it
    return dict(pool=pool, records_mi=size // mi, ms=float(np.mean(times)), empty_pool=True)


def stream(lib, n_scans, n_points, grow):
    cfg = api.VELODYNE
    sensor, scans = synth.make_stream("hdl64loop", n_scans, seed=8, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    h = api.Lio(tiny_config(cfg, first_scan_use(lib, cfg, sensor, scans)) if grow else cfg, lib=lib)
    if grow:
        h.set_growth(1 << 40)
    start(h, sensor, scans)
    h.voxel_map_init(scans[0]["body_full"])
    lat, growth_at = [], []
    g0 = h.capacity()["growths"]
    t_all = time.perf_counter()
    for k in range(1, n_scans):
        t0 = time.perf_counter()
        h.step(scans[k]["body_ds"], dt=scans[k]["dt"])
        lat.append((time.perf_counter() - t0) * 1e3)
        if grow:
            g = h.capacity()["growths"]
            if g != g0:
                growth_at.append(k - 1)
                g0 = g
    wall = time.perf_counter() - t_all
    cap = h.capacity()
    h.close()
    return dict(lat=np.array(lat), growth_at=growth_at, wall=wall, cap=cap)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,16", help="Mi records per pool for the doubling times")
    ap.add_argument("--scans", type=int, default=300)
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = api.load_library()
    res = dict(gpu=gpu_info(), doubling=[], stream={})
    for s in [int(x) for x in a.sizes.split(",")]:
        for pool in ("root_hash", "nodes", "chunks"):
            res["doubling"].append(one_doubling(lib, pool, s << 20))
    ref = stream(lib, a.scans, a.points, grow=False)
    grw = stream(lib, a.scans, a.points, grow=True)
    med = float(np.median(ref["lat"]))
    pauses = [grw["lat"][i] - med for i in grw["growth_at"]]
    res["stream"] = dict(
        scans=a.scans, points=a.points,
        presized=dict(scans_per_s=(a.scans - 1) / ref["wall"], p95_ms=float(np.percentile(ref["lat"], 95)), device_bytes=ref["cap"]["device_bytes"]),
        growing=dict(scans_per_s=(a.scans - 1) / grw["wall"], p95_ms=float(np.percentile(grw["lat"], 95)), growths=len(grw["growth_at"]),
                     pause_total_ms=float(sum(pauses)), pause_max_ms=float(max(pauses)) if pauses else 0.0, device_bytes=grw["cap"]["device_bytes"],
                     final=grw["cap"]))
    txt = json.dumps(res, default=lambda o: o.tolist() if hasattr(o, "tolist") else str(o))
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
