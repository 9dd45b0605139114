#!/usr/bin/env python
"""Mesh quality in the terms of the ImMesh paper's Experiment-3 (section VIII-C, Tables V and VI): fairness (Max-Min angle, C2SE) and
correctness (completeness, accuracy, recall, precision, F-score) of the device mesh against the noise-free ground truth of the
synthetic streams (synth.make_gt_cloud), with immesh_mesh_evaluate.

Two streams: Avia-shaped (the C1 / C2 shape) and KITTI-shaped (HDL-64, the C3 shape).  Each is meshed two ways: through the
localization chain (estimated poses, drift included: Lio.step_async + push_frame_from_lio_async) and with push_frame at the true poses
(the mesher alone).  Each mesh is evaluated with its raw and its smoothed vertex positions (smooth_all(1.0, 20), what save_to_ply_file
writes).  Prints one table row per evaluation and the synchronised wall time of each evaluation call with the card's name and power
limit, read in the same run.  Asserts nothing.

  python tools/mesh_quality.py [--avia-scans 40] [--kitti-scans 30] [--spacing 0.01] [--gt-leaf 0.01] [--threshold 0.05] [--max-dist 1.0]
"""
from __future__ import annotations

import argparse
import dataclasses
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from immesh_b200 import api, synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown card ({e})"


def mesh_true_poses(kind, n, seed, ext_T):
    sensor, scans = synth.make_stream(kind, n, seed=seed, ext_T=ext_T)
    mesh = api.Mesh(api.MeshConfig())
    mesh.set_growth(24 << 30)
    for k, s in enumerate(scans):
        lidar_w = s["body_full"].astype(np.float64) @ s["R_true"].T + (s["R_true"] @ np.asarray(ext_T) + s["t_true"])
        mesh.push_frame(lidar_w.astype(np.float32), s["t_true"], k)
    return mesh


def mesh_lio(kind, n, seed, cfg):
    sensor, scans = synth.make_stream(kind, n, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg), api.Mesh(api.MeshConfig())
    mesh.set_growth(24 << 30)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    s = lio.get_state()
    s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
    lio.set_state(s)
    lio.voxel_map_init(scans[0]["body_full"])
    for k in range(1, n):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
    mesh.wait()
    return mesh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--avia-scans", type=int, default=40)
    ap.add_argument("--kitti-scans", type=int, default=30)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--spacing", type=float, default=0.01)
    ap.add_argument("--gt-leaf", type=float, default=0.01)
    ap.add_argument("--threshold", type=float, default=0.05)
    ap.add_argument("--max-dist", type=float, default=1.0)
    ap.add_argument("--only", choices=["avia", "kitti"], default=None)
    ap.add_argument("--only-path", choices=["lio", "true"], default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_quality: no CUDA device")
    streams = [("avia", "Avia (C1/C2 shape)", args.avia_scans, api.AVIA), ("kitti", "KITTI HDL-64 (C3 shape)", args.kitti_scans, api.VELODYNE)]
    print(f"card: {card()}")
    print(f"spacing {args.spacing} m, gt_leaf {args.gt_leaf} m, threshold {args.threshold} m, max_dist {args.max_dist} m, incorrect_ratio 0.8")
    hdr = f"{'stream':<24} {'poses':<5} {'pos':<8} {'tris':>9} {'Max-Min':>8} {'C2SE':>7} {'compl.':>8} {'acc.':>8} {'recall':>7} {'prec.':>7} {'F':>7} " \
          f"{'far S':>8} {'far GT':>8} {'wrong f':>8} {'samples':>11} {'GT pts':>10} {'eval s':>7} {'Msamp/s':>8} {'tiles':>5}"
    print(hdr)
    for key, name, n, cfg in streams:
        if args.only and args.only != key:
            continue
        kind = "avia" if key == "avia" else "hdl64"
        if key == "kitti":
            cfg = dataclasses.replace(cfg, calib_laser=0)   # step_async takes the already calibrated synthetic scans
        gt = synth.make_gt_cloud(kind, n, seed=args.seed, ext_T=cfg.ext_T)
        for path in ("lio", "true"):
            if args.only_path and args.only_path != path:
                continue
            mesh = mesh_lio(kind, n, args.seed, cfg) if path == "lio" else mesh_true_poses(kind, n, args.seed, cfg.ext_T)
            for smoothed in (False, True):
                if smoothed:
                    mesh.smooth_all(1.0, 20)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = mesh.evaluate(gt, spacing=args.spacing, gt_leaf=args.gt_leaf, threshold=args.threshold, max_dist=args.max_dist, smoothed=smoothed)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                c, m = r["counts"], r["metrics"]
                print(f"{name:<24} {path:<5} {'smoothed' if smoothed else 'raw':<8} {c['live_triangles']:>9} {m['maxmin_deg']:>8.3f} {m['c2se']:>7.4f} "
                      f"{m['completeness']:>8.5f} {m['accuracy']:>8.5f} {m['recall']:>7.4f} {m['precision']:>7.4f} {m['fscore']:>7.4f} "
                      f"{c['samples_far']:>8} {c['gt_far']:>8} {c['incorrect_facets']:>8} {c['samples']:>11} {c['gt_points']:>10} {dt:>7.2f} "
                      f"{c['samples'] / dt * 1e-6:>8.2f} {r['stats']['tiles']:>5}", flush=True)
            mesh.close()
    print("accuracy / completeness are lower bounds when the far counts are non-zero (a far query counts max_dist)")


if __name__ == "__main__":
    main()
