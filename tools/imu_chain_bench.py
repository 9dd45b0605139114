"""Scans per second of the IMU-enabled scan loop (immesh_lio_step_async_imu, host and device input) and of the LiDAR-only raw chain
(immesh_lio_step_async_raw with Forward_without_imu) on the same Avia-shaped stream, every steady scan meshed through
immesh_mesh_push_frame_from_lio_async.  Before timing, a prefix of the stream is checked bit for bit against the CPU oracle chain.
Each timed run starts from fresh handles and covers the steady scans (after the initialisation and the first map), ending with the
waits; the three legs alternate over --rounds rounds.  Prints one JSON line per leg with the card's name and power limit.

  python tools/imu_chain_bench.py [--scans 120] [--points 100000] [--rounds 20] [--check 6]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests")]

from immesh_b200 import api  # noqa: E402
from imu_stream_common import OracleChain, imu_cfg, make_imu_stream, true_velocity  # noqa: E402

MAX_INI = 3   # mapping/imu_int_frame default
MESH_CFG = api.MeshConfig(max_vertices=1 << 22, max_triangles=1 << 23, max_voxels=1 << 20, max_frame_points=1 << 18)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, pl = out.strip().splitlines()[0].split(", ")
        return name, pl
    except Exception as e:   # the numbers are still printed; the card fields say why they are missing
        return f"unknown ({e})", "unknown"


def state0(sensor, scans):
    s = np.zeros(348)
    s[0:9] = np.eye(3).reshape(9)
    s[12:15] = true_velocity(sensor, scans[0]["beg"])
    for i in range(18):
        s[24 + i * 18 + i] = 1e-7
    return s


def run_imu(scans, s0, leaf, dev=None, timed_from=None):
    """the stream through the IMU chain; returns (lio, mesh, seconds from scan timed_from to the end of the waits)"""
    g = api.Lio(api.AVIA)
    g.set_state(s0)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 18, max_imu=64)
    vg = api.VoxelGrid(1 << 18)
    gm = api.Mesh(MESH_CFG)
    imu_h.init_begin(MAX_INI)
    t0 = None
    for k, sc in enumerate(scans):
        if k == timed_from:
            g.wait(); gm.wait()
            t0 = time.perf_counter()
        n = sc["pts"].shape[0]
        if dev is not None:
            br = vg.step_async_imu(g, imu_h, sc["imu"], dev[k].data_ptr(), sc["beg"], leaf, n=n, on_device=True)
        else:
            br = vg.step_async_imu(g, imu_h, sc["imu"], sc["pts"], sc["beg"], leaf)
        if br == 3:
            gm.push_frame_from_lio_async(g, vg.input_points(), n, on_device=True)
    g.wait(); gm.wait()
    sec = time.perf_counter() - t0 if t0 is not None else 0.0
    return g, gm, sec, (imu_h, vg)


def run_raw(scans, s0, leaf, timed_from):
    """the LiDAR-only chain on the same scans: the first scan (after the initialisation scans) builds the map, then
    immesh_lio_step_async_raw with the constant-velocity prediction"""
    g = api.Lio(api.AVIA)
    g.set_state(s0)
    vg = api.VoxelGrid(1 << 18)
    gm = api.Mesh(MESH_CFG)
    first = timed_from - 1
    g.voxel_map_init(np.ascontiguousarray(scans[first]["pts"][:, :3]))
    t0 = None
    for k in range(first + 1, len(scans)):
        if k == timed_from:
            g.wait(); gm.wait()
            t0 = time.perf_counter()
        pts = scans[k]["pts"]
        vg.step_async_raw(g, pts, leaf, dt=0.1, stride=4)
        gm.push_frame_from_lio_async(g, vg.input_points(), pts.shape[0], on_device=True)
    g.wait(); gm.wait()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=120)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--check", type=int, default=6)
    a = ap.parse_args()
    import torch
    leaf = api.AVIA.filter_size_surf
    sensor, scans = make_imu_stream(a.scans, seed=21, n_points=a.points, kind="avia100k")
    s0 = state0(sensor, scans)
    # parity of a prefix against the oracle chain
    o = OracleChain(api.AVIA, imu_cfg(), MESH_CFG, MAX_INI, s0, leaf)
    br_o = [o.step(sc["imu"], sc["pts"], sc["beg"]) for sc in scans[:a.check]]
    g, gm, _, _ = run_imu(scans[:a.check], s0, leaf)
    (v, t, f), (ov, ot, of) = gm.snapshot(), o.mesh.snapshot()
    ok = (np.array_equal(g.get_state(), o.lio.get_state()) and np.array_equal(g.dump_map(), o.lio.dump_map()) and v.shape == ov.shape
          and np.array_equal(v, ov) and t.shape == ot.shape and np.array_equal(t, ot) and np.array_equal(f, of))
    print(json.dumps({"parity_prefix_scans": a.check, "branches": br_o, "ok": bool(ok)}), flush=True)
    if not ok:
        sys.exit(1)
    g.close(); gm.close()
    timed_from = br_o.index(2) + 1   # the first steady scan
    steady = a.scans - timed_from
    dev = [torch.from_numpy(sc["pts"]).cuda() for sc in scans]
    torch.cuda.synchronize()
    # warm-up of every leg
    run_imu(scans[:timed_from + 5], s0, leaf, timed_from=timed_from)
    run_imu(scans[:timed_from + 5], s0, leaf, dev=dev, timed_from=timed_from)
    run_raw(scans[:timed_from + 5], s0, leaf, timed_from)
    tot = {"imu_host": 0.0, "imu_device": 0.0, "raw_lidar_only": 0.0}
    for r in range(a.rounds):
        legs = ["imu_host", "imu_device", "raw_lidar_only"]
        for leg in (legs if r % 2 == 0 else legs[::-1]):
            if leg == "raw_lidar_only":
                tot[leg] += run_raw(scans, s0, leaf, timed_from)
            else:
                tot[leg] += run_imu(scans, s0, leaf, dev=dev if leg == "imu_device" else None, timed_from=timed_from)[2]
    name, pl = card()
    for leg, sec in tot.items():
        n = steady * a.rounds
        print(json.dumps({"leg": leg, "scans": n, "points_per_scan": a.points, "seconds": round(sec, 3), "scans_per_s": round(n / sec, 1),
                          "gpu": name, "power_limit": pl}), flush=True)


if __name__ == "__main__":
    main()
