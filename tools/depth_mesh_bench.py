#!/usr/bin/env python
"""Meshing a depth-camera stream: immesh_mesh_push_depth_async against a host unprojection + immesh_mesh_push_frame, and the
Experiment-3 metrics of the result.

  python tools/depth_mesh_bench.py [--frames 60] [--rounds 3] [--width 640] [--height 480] [--kind range] [--no-profile]

The stream is the shape of the ImMesh paper's depth-image workload (AirSim 640 x 480 depth, Table VI): float32 images ray-cast from the
synth scene (tests/depth_reference.py) by a 70 degree pinhole camera moving 0.25 m per frame along synth.trajectory_pose, "range"
(AirSim DepthPerspective) by default; the mesher runs with the default MeshConfig (0.4 m voxels, 0.1 m xi, 10000 points appended per
frame).  Modes, alternated --rounds times in this one process on fresh handles:
  device_async   immesh_mesh_push_depth_async of the host image (staged through the pinned slots), one wait at the end
  device_sync    immesh_mesh_push_depth, blocking per frame
  host           the unprojection on the host (numpy, float64, the documented arithmetic) then immesh_mesh_push_frame of the points
  frames_per_s   host clock over --frames frames after a warm-up, ending with the handle drained
  depth_kernels_us  device time per frame of k_depth_count, k_rf_scan and k_depth_emit (torch.profiler, a run of its own)
  metrics        immesh_mesh_evaluate of the device_async mesh against the ground truth: the noise-free hits of a camera of twice the
                 resolution at every other pose (spacing 0.01 m, gt_leaf 0.01 m, threshold 0.05 m)
Prints one JSON line with the GPU's name, power limit and SM clock limit.  Writes nothing."""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

DEPTH_KERNELS = ("k_depth_count", "k_rf_scan", "k_depth_emit")
MODES = ("device_async", "device_sync", "host")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--kind", default="range", choices=["range", "planar"])
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    import depth_reference as dr
    from immesh_b200 import api
    w, h, n, W = args.width, args.height, args.frames, 4
    cam = dr.camera(w, h, kind=args.kind, z_min=0.2, z_max=60.0)
    poses = [dr.camera_pose(k) for k in range(W + n)]
    imgs = [dr.render(cam, w, h, R, t, kind=args.kind) for R, t in poses]
    cfg = api.MeshConfig(max_frame_points=w * h)

    def run(mode, profile=None):
        mesh = api.Mesh(cfg)

        def frame(k):
            R, t = poses[k]
            if mode == "device_async":
                mesh.push_depth_async(imgs[k], cam, R, t)
            elif mode == "device_sync":
                mesh.push_depth(imgs[k], cam, R, t)
            else:
                mesh.push_frame(dr.unproject(imgs[k], cam, R, t)[0], t)

        for k in range(W):
            frame(k)
        mesh.wait()
        torch.cuda.synchronize()
        if profile is not None:
            profile.start()
        t0 = time.perf_counter()
        for k in range(W, W + n):
            frame(k)
        mesh.wait()
        ms = (time.perf_counter() - t0) * 1e3
        if profile is not None:
            torch.cuda.synchronize()
            profile.stop()
        return mesh, n / ms * 1e3

    for m in MODES:   # warm-up: module loads, graph capture
        run(m)[0].close()
    rates = {m: [] for m in MODES}
    meshes = {}
    for _ in range(args.rounds):
        for m in MODES:
            mesh, r = run(m)
            rates[m].append(round(r, 2))
            if m in meshes:
                mesh.close()
            else:
                meshes[m] = mesh
    # the two paths build the same mesh
    va, ta, fa = meshes["device_async"].snapshot()
    vh, th, fh = meshes["host"].snapshot()
    same = va.tobytes() == vh.tobytes() and ta.tobytes() == th.tobytes() and fa.tobytes() == fh.tobytes()
    gcam = dataclasses.replace(cam, fx=2 * cam.fx, fy=2 * cam.fy, cx=2 * cam.cx + 0.5, cy=2 * cam.cy + 0.5)
    gt = np.concatenate([dr.unproject(dr.render(gcam, 2 * w, 2 * h, R, t, kind=args.kind), gcam, R, t)[0] for R, t in poses[::2]])
    ev = meshes["device_async"].evaluate(gt)
    out = {"frames": n, "image": [w, h], "kind": args.kind, "frames_per_s": rates, "same_mesh": bool(same),
           "points_per_frame": round(float(np.mean([dr.unproject(imgs[k], cam, *poses[k])[0].shape[0] for k in range(W, W + n)])), 1),
           "counts": meshes["device_async"].counts(), "metrics": {k: round(float(v), 5) for k, v in ev["metrics"].items()}}
    for m in meshes.values():
        m.close()
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        prof = profile(activities=[ProfilerActivity.CUDA])
        run("device_async", prof)[0].close()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0)
            for name in DEPTH_KERNELS:
                if e.key == name or e.key.startswith(name + "(") or f"::{name}(" in e.key:
                    per[name] = per.get(name, 0.0) + t
        out["depth_kernels_us"] = {k: round(v / n, 2) for k, v in per.items()}
        out["depth_kernels_us"]["total"] = round(sum(per.values()) / n, 2)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
