#!/usr/bin/env python
"""Time the mesh viewer's shaded image (immesh_mesh_render_view, immesh_mesh_view_enable) on one of bench.py's workloads.

  python tools/view_bench.py [--config C3] [--scans 24] [--rounds 3] [--reps 20]

Numbers, each on the same scans:
  render_view_ms            the host clock around the blocking immesh_mesh_render_view on the mesh after the stream (median of --reps
                            calls after a warm-up; each call waits for the mesh stream, allocates, bins, shades, copies back, frees),
                            at 640 x 480 (the reference's camera) and 1920 x 1080 (focus scaled by 3), white and height-coloured,
                            from a camera behind and above the last sensor pose
  scans_per_s off / on      the pipelined, graph-replayed stream (step_async + push_frame_from_lio_async, inputs in HBM), timed with
                            pipeline_mark_begin / _end, the queued view (640 x 480, sensor-bound, height colour) off and on,
                            alternated `rounds` times
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


def look_at(eye, target):
    f = np.asarray(target, np.float64) - eye
    f /= np.linalg.norm(f)
    x = np.cross(f, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(x, f), -f], axis=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--scans", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    n = args.scans
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]

    def handles(view):
        lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        if view:
            mesh.view_enable(color_by_height=True)
        return lio, mesh

    # ---- the blocking call on the stream's mesh
    lio, mesh = handles(False)
    for k in range(1, 1 + n):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
    lio.wait()
    mesh.wait()
    pos = lio.get_state()[9:12].copy()
    eye = pos + np.array([-25.0, -10.0, 20.0])
    R = look_at(eye, pos)
    out = {"config": args.config, "frames": n, "triangles": mesh.counts()["n_triangles"], "render_view_ms": {}}
    for w, h, focus in ((640, 480, 400.0), (1920, 1080, 1200.0)):
        K = api.reinforce_intrinsics(w, h, focus)
        for color in (False, True):
            rgba, depth = mesh.render_view(K, w, h, 0.1, 1500.0, R, eye, color_by_height=color)   # warm-up
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                mesh.render_view(K, w, h, 0.1, 1500.0, R, eye, color_by_height=color)
                ts.append((time.perf_counter() - t0) * 1e3)
            key = f"{w}x{h}_{'height' if color else 'white'}"
            out["render_view_ms"][key] = round(float(np.median(ts)), 3)
            out.setdefault("drawn_pixels", {})[key] = int((rgba[..., :3] != 0).any(axis=2).sum())
    lio.close(); mesh.close()

    # ---- pipelined stream, queued view on / off alternated
    def stream(view):
        lio, mesh = handles(view)
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
        lio.close(); mesh.close()
        return (n - W) / ms * 1e3

    rates = {True: [], False: []}
    for _ in range(args.rounds):
        for on in (False, True):
            rates[on].append(stream(on))
    out["scans_per_s_off"] = [round(r, 2) for r in rates[False]]
    out["scans_per_s_on"] = [round(r, 2) for r in rates[True]]
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
