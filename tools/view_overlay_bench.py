#!/usr/bin/env python
"""Time the queued view's overlays (immesh_mesh_view_overlay) on one of bench.py's workloads.

  python tools/view_overlay_bench.py [--config C3] [--scans 24] [--rounds 3]

The pipelined, graph-replayed stream (step_async + push_frame_from_lio_async, inputs in HBM, timed with pipeline_mark_begin / _end)
with the queued view at 640 x 480 (the reference's camera, follow mode, white), alternated `rounds` times over these settings:
  view          the faces only
  overlays      the faces and every overlay at the reference's defaults (scan and reinforced points 2 px, axis and grid, camera
                size 1, path width 4), with the reinforcement on so that its points are drawn
  wireframe     the same with the wireframe in place of the faces
  view_rf       the faces with the reinforcement on and no overlay (the baseline of `overlays`)
  scan_only, lines_only, reinforced_only   one group of layers alone, reinforcement on (which layer dominates the cost)
Reports scans/s for each, and the overlay's cost per frame against view_rf.  Prints one JSON line with the GPU's name, power limit and
SM clock limit.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULTS = dict(scan_point_size=2, reinforced_point_size=2, axis_and_grid=True, camera_size=1.0, path_width=4, path_capacity=1 << 16)
NONE = dict(scan_point_size=0, reinforced_point_size=0, axis_and_grid=False, camera_size=0.0, path_width=0)
SETTINGS = {
    "view": (False, None),
    "view_rf": (True, None),
    "overlays": (True, DEFAULTS),
    "wireframe": (True, dict(DEFAULTS, wireframe=True)),
    "scan_only": (True, dict(NONE, scan_point_size=2)),
    "reinforced_only": (True, dict(NONE, reinforced_point_size=2)),
    "lines_only": (True, dict(NONE, axis_and_grid=True, camera_size=1.0, path_width=4, path_capacity=1 << 16)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--scans", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    n = args.scans
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]
    R_follow = np.array([[0.0, 0.0, -1.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])   # looking along +x, behind and above the sensor

    def stream(name):
        rf, ov = SETTINGS[name]
        lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        if rf:
            mesh.reinforce_enable()
        mesh.view_enable()
        mesh.view_pose(R_follow, np.array([-15.0, 0.0, 8.0]), follow=True)
        if ov is not None:
            mesh.view_overlay(**ov)
        W = 4
        for k in range(1, 1 + W):
            lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        lio.wait(); mesh.wait()
        torch.cuda.synchronize()
        api.pipeline_mark_begin(lio)
        for k in range(1 + W, 1 + n):
            lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        ms = api.pipeline_mark_end(lio, mesh)
        lio.wait(); mesh.wait()
        rgba = mesh.view_image()[0]
        drawn = int((rgba[..., :3] != 0).any(axis=2).sum())
        lio.close(); mesh.close()
        return (n - W) / ms * 1e3, drawn

    rates = {k: [] for k in SETTINGS}
    drawn = {}
    for _ in range(args.rounds):
        for name in SETTINGS:
            r, d = stream(name)
            rates[name].append(round(r, 2))
            drawn[name] = d
    med = {k: float(np.median(v)) for k, v in rates.items()}
    out = {"config": args.config, "frames": n, "scans_per_s": rates, "drawn_pixels": drawn,
           "overlay_ms_per_frame": {k: round(1e3 / med[k] - 1e3 / med["view_rf"], 3) for k in ("overlays", "wireframe", "scan_only", "reinforced_only", "lines_only")}}
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
