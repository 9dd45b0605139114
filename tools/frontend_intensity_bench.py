"""What carrying point intensity through the device front-end costs: scans per second of the plain chains against their
intensity-carrying (_i) twins on the same Avia-shaped stream, every steady scan meshed through immesh_mesh_push_frame_from_lio_async.
  raw_host / raw_i_host     immesh_lio_step_async_raw on [n][4] host scans / _raw_i on stride-12 PointXYZINormal host records
  imu_host / imu_i_host     immesh_lio_step_async_imu on [n][4] host scans / _imu_i on stride-12 host records (48 B per point over PCIe
                            instead of 16)
  imu_device / imu_i_device the same from device memory
Before timing, a prefix of the stream through the _i IMU chain is checked bit for bit against the CPU oracle chain (state, map, mesh)
and its published intensities against the stable time sort of the input's.  Each timed run starts from fresh handles, covers the
steady scans and ends with the waits; the legs alternate over --rounds rounds.  Prints one JSON line per leg with the card's name
and power limit.

  python tools/frontend_intensity_bench.py [--scans 60] [--points 100000] [--rounds 8] [--check 6]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests"), os.path.join(_ROOT, "tools")]

from immesh_b200 import api  # noqa: E402
from frontend_intensity_common import intensities, records  # noqa: E402
from imu_chain_bench import MAX_INI, MESH_CFG, card, state0  # noqa: E402
from imu_stream_common import OracleChain, imu_cfg, make_imu_stream  # noqa: E402

STRIDE, TIME_COL, INTENSITY_COL = 12, 9, 8   # pcl::PointXYZINormal: x y z pad intensity normal_xyz curvature ...


def run_imu(scans, s0, leaf, with_i, dev=None, timed_from=None):
    """the stream through the IMU chain; returns (lio, mesh, vg, seconds from scan timed_from to the end of the waits)"""
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
        src = sc["rec"] if with_i else sc["pts"]
        if with_i:
            if dev is not None:
                br = vg.step_async_imu_i(g, imu_h, sc["imu"], dev[k].data_ptr(), sc["beg"], leaf, TIME_COL, INTENSITY_COL, n=n, stride=STRIDE, on_device=True)
            else:
                br = vg.step_async_imu_i(g, imu_h, sc["imu"], src, sc["beg"], leaf, TIME_COL, INTENSITY_COL)
        elif dev is not None:
            br = vg.step_async_imu(g, imu_h, sc["imu"], dev[k].data_ptr(), sc["beg"], leaf, n=n, on_device=True)
        else:
            br = vg.step_async_imu(g, imu_h, sc["imu"], src, sc["beg"], leaf)
        if br == 3:
            gm.push_frame_from_lio_async(g, vg.input_points(), n, on_device=True)
    g.wait(); gm.wait()
    sec = time.perf_counter() - t0 if t0 is not None else 0.0
    return g, gm, vg, sec


def run_raw(scans, s0, leaf, timed_from, with_i):
    """the LiDAR-only chain on the same scans: the scan before timed_from builds the map, then the raw chain with the
    constant-velocity prediction"""
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
        n = scans[k]["pts"].shape[0]
        if with_i:
            vg.step_async_raw_i(g, scans[k]["rec"], leaf, INTENSITY_COL, dt=0.1)
        else:
            vg.step_async_raw(g, scans[k]["pts"], leaf, dt=0.1, stride=4)
        gm.push_frame_from_lio_async(g, vg.input_points(), n, on_device=True)
    g.wait(); gm.wait()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=60)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--check", type=int, default=6)
    a = ap.parse_args()
    import torch
    leaf = api.AVIA.filter_size_surf
    sensor, scans = make_imu_stream(a.scans, seed=21, n_points=a.points, kind="avia100k")
    for k, sc in enumerate(scans):
        sc["inten"] = intensities(sc["pts"].shape[0], k)
        sc["rec"] = records(sc["pts"][:, :3], sc["inten"], STRIDE, INTENSITY_COL, stamps=sc["pts"][:, 3], time_col=TIME_COL, seed=k)
    s0 = state0(sensor, scans)
    # parity of a prefix of the _i chain against the oracle chain, and the published intensities of its last scan
    o = OracleChain(api.AVIA, imu_cfg(), MESH_CFG, MAX_INI, s0, leaf)
    br_o = [o.step(sc["imu"], sc["pts"], sc["beg"]) for sc in scans[:a.check]]
    g, gm, vg, _ = run_imu(scans[:a.check], s0, leaf, True)
    (v, t, f), (ov, ot, of) = gm.snapshot(), o.mesh.snapshot()
    last = scans[a.check - 1]
    dense = g.frontend_cloud(vg, True)
    ok = (br_o[-1] == 3 and np.array_equal(g.get_state(), o.lio.get_state()) and np.array_equal(g.dump_map(), o.lio.dump_map())
          and v.shape == ov.shape and np.array_equal(v, ov) and t.shape == ot.shape and np.array_equal(t, ot) and np.array_equal(f, of)
          and np.array_equal(dense[:, 3], last["inten"][np.argsort(last["pts"][:, 3], kind="stable")]))
    print(json.dumps({"parity_prefix_scans": a.check, "branches": br_o, "ok": bool(ok)}), flush=True)
    if not ok:
        sys.exit(1)
    g.close(); gm.close()
    timed_from = br_o.index(2) + 1   # the first steady scan
    steady = a.scans - timed_from
    dev4 = [torch.from_numpy(sc["pts"]).cuda() for sc in scans]
    dev12 = [torch.from_numpy(sc["rec"]).cuda() for sc in scans]
    torch.cuda.synchronize()
    legs = {"raw_host": lambda s: run_raw(s, s0, leaf, timed_from, False),
            "raw_i_host": lambda s: run_raw(s, s0, leaf, timed_from, True),
            "imu_host": lambda s: run_imu(s, s0, leaf, False, timed_from=timed_from)[3],
            "imu_i_host": lambda s: run_imu(s, s0, leaf, True, timed_from=timed_from)[3],
            "imu_device": lambda s: run_imu(s, s0, leaf, False, dev=dev4, timed_from=timed_from)[3],
            "imu_i_device": lambda s: run_imu(s, s0, leaf, True, dev=dev12, timed_from=timed_from)[3]}
    for fn in legs.values():   # warm-up of every leg
        fn(scans[:timed_from + 5])
    tot = {leg: [] for leg in legs}
    names = list(legs)
    for r in range(a.rounds):
        for leg in (names if r % 2 == 0 else names[::-1]):
            tot[leg].append(legs[leg](scans))
    name, pl = card()
    for leg, secs in tot.items():
        rates = [steady / s for s in secs]
        print(json.dumps({"leg": leg, "scans": steady * a.rounds, "points_per_scan": a.points, "scans_per_s": round(steady * a.rounds / sum(secs), 1),
                          "round_min": round(min(rates), 1), "round_max": round(max(rates), 1), "gpu": name, "power_limit": pl}), flush=True)


if __name__ == "__main__":
    main()
