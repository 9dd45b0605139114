"""Cost of the mesh's change feed (immesh_mesh_changes).  Needs a GPU.

  python tools/mesh_changes_bench.py [--kinds avia100k,hdl64loop] [--scans 40] [--reps 3] [--out DIR]

For each stream (avia100k = bench.py C100k's sensor, hdl64loop = C4's), the graph-replayed chain (localization step +
push_frame_from_lio_async per scan):
  - scans/s with the feed off and on, alternated --reps times (host clock around the queued scans and a final wait);
  - per-frame host time of a mirror's changes(newest) read against a full snapshot(), both after the frame has finished, with the
    rows, vertices and live triangles each returns (the snapshot grows with the map, the changes stay with the frame);
  - the feed kernels' device time per frame (k_chg_*, the radix passes they launch) from torch.profiler in a run of its own.
The card's name and power limit are printed with the numbers."""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from immesh_b200 import api, synth  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def chain(kind, n_scans, seed=0):
    from lio_common import init_velocity
    cfg = api.AVIA if kind.startswith("avia") else dataclasses.replace(api.VELODYNE, calib_laser=1)   # bench.py's C100k / C4 configurations
    sensor, scans = synth.make_stream(kind, n_scans + 1, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg), api.Mesh(api.MeshConfig())
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    return lio, mesh, scans


def rate(kind, n_scans, feed):
    lio, mesh, scans = chain(kind, n_scans)
    if feed:
        mesh.changes_enable(1 << 22, 1024)
    t0 = time.perf_counter()
    for k in range(1, n_scans + 1):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
    lio.wait()
    mesh.wait()
    return n_scans / (time.perf_counter() - t0)


def read_costs(kind, n_scans):
    lio, mesh, scans = chain(kind, n_scans)
    mesh.changes_enable(1 << 22, 1024)
    newest = mesh.changes_newest()
    rows = []
    for k in range(1, n_scans + 1):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        mesh.wait()
        t0 = time.perf_counter()
        ch = mesh.changes(newest)
        t1 = time.perf_counter()
        v, t, _ = mesh.snapshot()
        t2 = time.perf_counter()
        newest = ch["newest"]
        rows.append(dict(frame=newest, changes_ms=(t1 - t0) * 1e3, rows=len(ch["rows"]), new_vertices=len(ch["vertices"]),
                         snapshot_ms=(t2 - t1) * 1e3, triangles=len(t), vertices=len(v)))
    return rows


def kernel_times(kind, n_scans):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lio, mesh, scans = chain(kind, n_scans)
    mesh.changes_enable(1 << 22, 1024)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(1, n_scans + 1):
            lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
            mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        lio.wait()
        mesh.wait()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.key_averages():
        if e.key.startswith("k_chg_") or "_dev" in e.key and "k_rs_" in e.key:
            tot[e.key] = tot.get(e.key, 0.0) + e.device_time_total / n_scans / 1e3   # ms per frame
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kinds", default="avia100k,hdl64loop")
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print("card, power limit:", res["card"])
    for kind in a.kinds.split(","):
        r = dict(off=[], on=[])
        rate(kind, 4, False)   # warm-up: module load, graph capture
        for _ in range(a.reps):
            r["off"].append(round(rate(kind, a.scans, False), 1))
            r["on"].append(round(rate(kind, a.scans, True), 1))
        reads = read_costs(kind, a.scans)
        r["reads"] = reads
        r["kernels_ms_per_frame"] = kernel_times(kind, a.scans)
        res[kind] = r
        print(kind, "scans/s off", r["off"], "on", r["on"])
        for x in reads[:: max(1, len(reads) // 8)] + reads[-1:]:
            print(f"  frame {x['frame']}: changes {x['changes_ms']:.3f} ms ({x['rows']} rows, {x['new_vertices']} vertices)  "
                  f"snapshot {x['snapshot_ms']:.3f} ms ({x['triangles']} triangles, {x['vertices']} vertices)")
        print("  feed kernels, ms per frame:", {k: round(v, 4) for k, v in sorted(r["kernels_ms_per_frame"].items())},
              "total", round(sum(r["kernels_ms_per_frame"].values()), 4))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mesh_changes_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
