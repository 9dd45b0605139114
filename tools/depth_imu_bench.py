#!/usr/bin/env python
"""The IMU-enabled loop on a depth-camera stream: immesh_lio_step_async_depth_imu (one queued call per frame, every branch decided on the
device) against the host round trip it replaces (immesh_frontend_prepare_depth -> host drop rule and t = 0 records ->
immesh_lio_step_async_imu), each followed by its mesh hand-off.

  python tools/depth_imu_bench.py [--frames 60] [--rounds 3] [--point-filter-num 2] [--blind 0.5] [--leaf 0.2]

The stream: 640 x 480 float32 range images ray-cast from the synth scene (tests/depth_reference.py) by the camera of
tests/depth_lio_reference.py, every 10th frame blanked (a cloud sync_packages drops), and a synthetic near-static 200 Hz IMU (20 samples
per frame, seeded noise).  Each run starts from fresh handles with immesh_imu_init_begin(3).  First the parity check: both paths over
the whole stream, state, VoxelMap and mesh snapshot compared after it; it is printed before any rate, and a mismatch ends the run.  Then the modes,
alternated --rounds times on fresh handles, each timed over --frames frames after a warm-up of 8 frames, ending with both handles drained:
  queued  VoxelGrid.step_async_depth_imu + Mesh.push_frame_from_lio_async_dev_n
  host    VoxelGrid.prepare_depth (blocking) + host drop / carry + step_async_imu + push_frame_from_lio_async in branch 3
Prints the parity line, then one JSON line with the GPU's name, power limit and SM clock limit.  Writes nothing."""
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

T0, DT, IMU_PER_FRAME, WARM = 500.0, 0.1, 20, 8


def imu_batch(k, m=IMU_PER_FRAME):
    rng = np.random.default_rng([11, k])
    t = T0 + DT * (k - 1) + (np.arange(m) + 1) * (DT / m)
    gyr = rng.normal(0.0, 0.002, (m, 3))
    acc = np.array([0.0, -9.81, 0.0]) + rng.normal(0.0, 0.02, (m, 3))
    return np.concatenate([t[:, None], gyr, acc], axis=1)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power, sm_clock_limit=clock)
    except Exception as e:   # the rates stand without it; say why it is missing
        return dict(gpu=f"unknown ({e})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--point-filter-num", type=int, default=2)
    ap.add_argument("--blind", type=float, default=0.5)
    ap.add_argument("--leaf", type=float, default=0.2)
    args = ap.parse_args()
    import torch
    import depth_lio_reference as dlr
    import depth_reference as dr
    from immesh_b200 import api
    if not torch.cuda.is_available():
        sys.exit("depth_imu_bench: no CUDA device (the rates are GPU measurements)")
    w, h, n = 640, 480, args.frames
    pfn, blind, leaf = args.point_filter_num, args.blind, args.leaf
    cam = dr.camera(w, h, kind="range", z_min=0.3, z_max=40.0)
    total = WARM + n
    imgs = []
    for k in range(total):
        R, t = dr.camera_pose(k)
        img = dr.render(cam, w, h, R, t, kind="range")
        imgs.append(np.full_like(img, np.nan) if k % 10 == 9 else img)
    batches = [imu_batch(k) for k in range(total)]
    icfg = dict(cov_gyr=[0.1] * 3, cov_acc=[0.1] * 3, cov_bias_gyr=[1e-4] * 3, cov_bias_acc=[1e-4] * 3, mean_acc_norm=9.81, lid_R=np.eye(3), lid_T=[0.0] * 3)

    def handles():
        lio = api.Lio(api.LioConfig(ext_T=(0.0, 0.0, 0.0)))
        vg = api.VoxelGrid(w * h)
        imu = api.Imu(icfg, max_points=w * h, max_imu=128)
        mesh = api.Mesh(api.MeshConfig(max_frame_points=w * h))
        imu.init_begin(3)
        return lio, vg, imu, mesh

    def queued(hd, k):
        lio, vg, imu, mesh = hd
        ns = vg.step_async_depth_imu(lio, imu, batches[k], imgs[k], cam, T0 + DT * k, leaf, point_filter_num=pfn, blind=blind, cam_R=dlr.SENSOR_FROM_CAM)
        mesh.push_frame_from_lio_async_dev_n(lio, vg.input_points(), ns, vg.input_count())

    def host(hd, k, carry):
        lio, vg, imu, mesh = hd
        cloud = vg.prepare_depth(imgs[k], cam, dlr.SENSOR_FROM_CAM, point_filter_num=pfn, blind=blind)
        if cloud.shape[0] <= 1:
            return np.concatenate([carry, batches[k]])
        pts = np.concatenate([cloud, np.zeros((cloud.shape[0], 1), np.float32)], axis=1)
        if vg.step_async_imu(lio, imu, np.concatenate([carry, batches[k]]), pts, T0 + DT * k, leaf) == 3:
            mesh.push_frame_from_lio_async(lio, vg.input_points(), cloud.shape[0], on_device=True)
        return np.zeros((0, 7))

    def run(mode, frames):
        hd = handles()
        carry = np.zeros((0, 7))
        for k in range(WARM):
            if mode == "queued":
                queued(hd, k)
            else:
                carry = host(hd, k, carry)
        hd[0].wait()
        hd[3].wait()
        t0 = time.perf_counter()
        for k in range(WARM, WARM + frames):
            if mode == "queued":
                queued(hd, k)
            else:
                carry = host(hd, k, carry)
        hd[0].wait()
        hd[3].wait()
        return frames / (time.perf_counter() - t0), hd

    _, a = run("queued", n)
    _, b = run("host", n)
    same = a[0].get_state().tobytes() == b[0].get_state().tobytes() and a[0].dump_map().tobytes() == b[0].dump_map().tobytes()
    same = same and all(x.tobytes() == y.tobytes() for x, y in zip(a[3].snapshot(), b[3].snapshot()))
    st = a[2].depth_chain_state()
    print(f"parity over {total} frames, queued without waits: state, VoxelMap and mesh {'bit-identical' if same else 'DIFFER'}; "
          f"queued chain counters {st}", flush=True)
    if not same:
        sys.exit(1)
    rates = {"queued": [], "host": []}
    for _ in range(args.rounds):
        for mode in ("queued", "host"):
            rates[mode].append(round(run(mode, n)[0], 1))
    out = dict(gpu_info(), frames=n, rounds=args.rounds, image=f"{w}x{h}", point_filter_num=pfn, blind=blind, leaf=leaf,
               queued_fps=rates["queued"], host_fps=rates["host"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
