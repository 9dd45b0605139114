"""Cost and effect of the VoxelMap's local map (immesh_lio_local_map), on one GPU.

  1. Pipelined localization rate on the C100k stream (avia100k, config/avia.yaml) with the local map off and on-but-not-moving
     (cube_side_length 1000: the box is placed and never moves on this stream), in alternating rounds.
  2. Device time of the eviction sweep (k_evict_roots) on the scans that move the box, and of the idle sweep and the box rule, from
     torch.profiler over an hdl64open drive with a small cube.
  3. immesh_lio_capacity device bytes along a long drive through the open-ended scene (synth "hdl64open", 1 m per scan), with and
     without the local map, from small capacities with automatic growth; beside them the bytes of a mesh handle meshing the same
     drive (immesh_mesh_capacity), which the local map does not bound.
  4. The card's name and power limit.
Prints one JSON object; --out also writes it to a file."""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

from immesh_b200 import api, synth  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the measurement itself does not depend on it
        return f"unavailable ({e})"


def start(h, scans):
    h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    s = h.get_state()
    s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
    h.set_state(s)
    h.voxel_map_init(scans[0]["body_full"])


def rate_round(cfg, scans, warm, local_map):
    h = api.Lio(cfg)
    if local_map:
        h.local_map(1000.0, 300.0, 1.5)
    start(h, scans)
    for k in range(1, warm + 1):
        h.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
    h.wait()
    t0 = time.perf_counter()
    for k in range(warm + 1, len(scans)):
        h.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
    h.wait()
    dt = time.perf_counter() - t0
    _, st = h.local_map_state()
    h.close()
    return (len(scans) - warm - 1) / dt, st


def sweep_cost(n_scans, n_points):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    cfg = api.VELODYNE
    _, scans = synth.make_stream("hdl64open", n_scans, seed=1, leaf=cfg.filter_size_surf, n_points=n_points)
    h = api.Lio(cfg)
    h.local_map(60.0, 20.0, 1.5)
    start(h, scans)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(1, n_scans):
            h.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        h.wait()
    _, st = h.local_map_state()
    ev = {"k_evict_roots": [], "k_local_map_box": []}
    for e in prof.events():
        for name in ev:
            if e.name.startswith(name) and e.device_type is not None and str(e.device_type).endswith("CUDA"):
                ev[name].append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    sw = np.sort(np.array(ev["k_evict_roots"], dtype=float))
    moves = st["moves"]
    out = dict(scans=n_scans - 1, moves=moves, roots_evicted=st["roots_evicted"], nodes_freed=st["nodes_freed"], root_slots=h.capacity()["root_slots"],
               sweeps=int(sw.size), box_rule_us_median=float(np.median(ev["k_local_map_box"])) if ev["k_local_map_box"] else None)
    if sw.size and moves:
        out["sweep_us_moving_mean"] = float(sw[-moves:].mean())     # the `moves` longest sweeps: the scans that moved the box
        out["sweep_us_idle_median"] = float(np.median(sw[:-moves])) if sw.size > moves else None
    h.close()
    return out


def capacity_drive(n_scans, n_points, every, local_map):
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=14, max_nodes=1 << 15, max_chunks=1 << 16, max_scan_points=1 << 17)
    h = api.Lio(cfg)
    h.set_growth(16 << 30)
    # the mesh handle fed the same drive (it is not bounded by the local map): its bytes beside the VoxelMap's
    gm = api.Mesh(api.MeshConfig(max_vertices=1 << 16, max_triangles=1 << 17, max_voxels=1 << 14, max_frame_points=1 << 17))
    gm.set_growth(16 << 30)
    if local_map:
        h.local_map(100.0, 30.0, 1.5)
    rows = []
    sensor = synth.make_sensor("hdl64open", n_points)
    first = [dict(zip(("body_full", "R_true", "t_true"), synth.make_scan(sensor, k, 1))) for k in (0, 1)]
    for f in first:
        f["dt"] = 1.0 / sensor.hz
    start(h, first)
    for k in range(1, n_scans):
        body, _, _ = synth.make_scan(sensor, k, 1)
        h.step_async(synth.voxel_grid_downsample(body, cfg.filter_size_surf), dt=1.0 / sensor.hz)
        gm.push_frame_from_lio_async(h, body)
        if k % every == 0 or k == n_scans - 1:
            h.wait()
            gm.wait()
            c = h.capacity()
            mc = gm.capacity()
            _, st = h.local_map_state()
            rows.append(dict(scan=k, metres=k * sensor.speed / sensor.hz, device_bytes=c["device_bytes"], roots=c["roots"], nodes=c["nodes"],
                             root_slots=c["root_slots"], growths=c["growths"], evicted=st["roots_evicted"], free_nodes=st["free_nodes"],
                             mesh_device_bytes=mc["device_bytes"], mesh_vertices=mc["vertices"], mesh_triangles=mc["triangles"]))
    gm.close()
    h.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rate-scans", type=int, default=60)
    ap.add_argument("--warm", type=int, default=10)
    ap.add_argument("--sweep-scans", type=int, default=80)
    ap.add_argument("--drive-scans", type=int, default=400)
    ap.add_argument("--drive-points", type=int, default=16384)
    ap.add_argument("--every", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info())
    _, scans = synth.make_stream("avia100k", a.rate_scans, seed=0, ext_T=api.AVIA.ext_T)
    rounds = []
    for _ in range(a.rounds):
        off, _ = rate_round(api.AVIA, scans, a.warm, False)
        on, st = rate_round(api.AVIA, scans, a.warm, True)
        assert st["moves"] == 0 and st["placed"] == 1
        rounds.append(dict(off_scans_per_s=round(off, 1), idle_scans_per_s=round(on, 1)))
    res["rate_c100k_pipelined"] = rounds
    res["sweep"] = sweep_cost(a.sweep_scans, 32768)
    res["drive_without_local_map"] = capacity_drive(a.drive_scans, a.drive_points, a.every, False)
    res["drive_with_local_map"] = capacity_drive(a.drive_scans, a.drive_points, a.every, True)
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
