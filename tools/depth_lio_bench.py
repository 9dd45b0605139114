#!/usr/bin/env python
"""Localizing and meshing a depth-camera stream on the queued chain: immesh_lio_step_async_depth +
immesh_mesh_push_frame_from_lio_async_dev_n against the same LiDAR chain fed a host-filtered cloud, with the trajectory error and the
Experiment-3 metrics of the result.

  python tools/depth_lio_bench.py [--frames 60] [--rounds 3] [--point-filter-num 2] [--blind 0.5] [--leaf 0.2] [--no-profile]

The stream: 640 x 480 float32 range images (AirSim DepthPerspective) ray-cast from the synth scene (tests/depth_reference.py) by a
70 degree pinhole camera moving 0.25 m per frame along synth.trajectory_pose, mounted looking forward on an x-forward, z-up sensor
(tests/depth_lio_reference.py); the localization runs the default LioConfig with the sensor as the body, the mesher the default
MeshConfig.  Every run starts at frame 0's true pose and velocity (prepare_depth -> predict -> voxel_map_init).  Modes, alternated
--rounds times in this one process on fresh handles, each timed over --frames frames after a warm-up, ending with both handles drained:
  depth         VoxelGrid.step_async_depth of the host image + Mesh.push_frame_from_lio_async_dev_n: no host pass over the pixels
  host          the numpy unprojection + filter on the host (tests/depth_lio_reference.py), then step_async_raw + push_frame_from_lio_async
  device_cloud  the same with the restated cloud already on the device (uploaded before the timed window)
  kernel_us     device time per frame of the new front-end kernels (immesh_profile_report, a run of its own)
  rms_pos_err_m the depth chain's position error against the true poses, RMS over the frames (a run that waits after every frame)
  metrics       immesh_mesh_evaluate of the depth chain's mesh against the noise-free hits of a camera of twice the resolution at every
                fourth true pose (as the ground truth of tools/depth_mesh_bench.py, which takes every other pose)
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

FRONT_KERNELS = ("k_depth_count", "k_depth_keep", "k_depth_emit")
MODES = ("depth", "host", "device_cloud")
DT = 0.1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--point-filter-num", type=int, default=2)
    ap.add_argument("--blind", type=float, default=0.5)
    ap.add_argument("--leaf", type=float, default=0.2)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    import depth_lio_reference as dlr
    import depth_reference as dr
    from immesh_b200 import api
    w, h, n, WARM = args.width, args.height, args.frames, 4
    pfn, blind, leaf = args.point_filter_num, args.blind, args.leaf
    cam = dr.camera(w, h, kind="range", z_min=0.3, z_max=40.0)
    cam_poses = [dr.camera_pose(k) for k in range(WARM + n + 1)]
    poses = [dlr.sensor_pose(k) for k in range(WARM + n + 1)]
    imgs = [dr.render(cam, w, h, R, t, kind="range") for R, t in cam_poses]
    mount = (dlr.SENSOR_FROM_CAM, np.zeros(3))
    clouds = [dlr.sensor_cloud(img, cam, *mount, pfn, blind)[0] for img in imgs]
    lcfg, mcfg = api.LioConfig(ext_T=(0.0, 0.0, 0.0)), api.MeshConfig(max_frame_points=w * h)

    def handles():
        lio, vg, mesh = api.Lio(lcfg), api.VoxelGrid(w * h), api.Mesh(mcfg)
        lio.set_pose(*poses[0])
        lio.predict(DT)
        lio.voxel_map_init(vg.prepare_depth(imgs[0], cam, *mount, point_filter_num=pfn, blind=blind))
        s = lio.get_state()
        s[12:15] = (poses[1][1] - poses[0][1]) / DT
        lio.set_state(s)
        return lio, vg, mesh

    def run(mode, profile=False, per_frame_wait=False):
        lio, vg, mesh = handles()
        dev = [torch.from_numpy(clouds[k]).cuda() for k in range(WARM + n + 1)] if mode == "device_cloud" else None
        torch.cuda.synchronize()
        errs = []

        def frame(k):
            if mode == "depth":
                ns = vg.step_async_depth(lio, imgs[k], cam, leaf, *mount, point_filter_num=pfn, blind=blind, dt=DT)
                mesh.push_frame_from_lio_async_dev_n(lio, vg.input_points(), ns, vg.input_count())
            elif mode == "host":
                c = dlr.sensor_cloud(imgs[k], cam, *mount, pfn, blind)[0]
                vg.step_async_raw(lio, c, leaf, dt=DT)
                mesh.push_frame_from_lio_async(lio, c)
            else:
                d = dev[k]
                vg.step_async_raw(lio, d.data_ptr(), leaf, dt=DT, n=d.shape[0], on_device=True)
                mesh.push_frame_from_lio_async(lio, d.data_ptr(), n=d.shape[0], on_device=True)
            if per_frame_wait:
                lio.wait()
                errs.append(float(np.linalg.norm(lio.get_state()[9:12] - poses[k][1])))

        for k in range(1, WARM):
            frame(k)
        lio.wait()
        mesh.wait()
        torch.cuda.synchronize()
        if profile:
            api.profile_reset()
            api.profile_enable(True)
        t0 = time.perf_counter()
        for k in range(WARM, WARM + n):
            frame(k)
        lio.wait()
        mesh.wait()
        ms = (time.perf_counter() - t0) * 1e3
        if profile:
            torch.cuda.synchronize()
            rep = api.profile_report()
            api.profile_enable(False)
            return rep
        return (lio, vg, mesh), n / ms * 1e3, errs

    for m in MODES:   # warm-up: module loads, graph capture
        run(m)
    rates = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            rates[m].append(round(run(m)[1], 2))
    (lio, vg, mesh), _, errs = run("depth", per_frame_wait=True)
    gcam = dataclasses.replace(cam, fx=2 * cam.fx, fy=2 * cam.fy, cx=2 * cam.cx + 0.5, cy=2 * cam.cy + 0.5)
    gt = np.concatenate([dr.unproject(dr.render(gcam, 2 * w, 2 * h, R, t, kind="range"), gcam, R, t)[0] for R, t in cam_poses[::4]])
    ev = mesh.evaluate(gt)
    out = {"frames": n, "image": [w, h], "point_filter_num": pfn, "blind": blind, "leaf": leaf, "frames_per_s": rates,
           "points_per_frame": round(float(np.mean([clouds[k].shape[0] for k in range(WARM, WARM + n)])), 1),
           "rms_pos_err_m": round(float(np.sqrt(np.mean(np.square(errs[WARM - 1:])))), 5), "final_pos_err_m": round(errs[-1], 5),
           "counts": mesh.counts(), "metrics": {k: round(float(v), 5) for k, v in ev["metrics"].items()}}
    if not args.no_profile:
        rep = run("depth", profile=True)
        per = {k: round(rep[k][0] * 1e3 / n, 2) for k in FRONT_KERNELS if k in rep}
        per["total"] = round(sum(per.values()), 2)
        out["front_kernels_us"] = per
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
