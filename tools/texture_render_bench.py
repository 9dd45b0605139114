#!/usr/bin/env python
"""Time the textured render (immesh_mesh_render_textured) and score the texture by leave-one-out, on bench.py's workloads with
tools/texture_bench.py's meshes and cameras.

  python tools/texture_render_bench.py [--configs C100k,C3] [--scans 30] [--reps 5]

Each workload's stream is localized and meshed through the queued chain; one camera per frame is posed from the frame's converged pose
and a fixed extrinsic (61-degree horizontal field of view), at 640 x 480, 1224 x 1024 and 1920 x 1080.  Every camera's image shows a
smooth seeded pattern painted on the world: render_view's depth at that camera, unprojected, coloured by the world point, so that the
held-out error measures the texturing and not the noise of random images.  texture_select picks each facet's camera among the even
cameras only; then every odd camera is a held-out view.  Per size:
  query_ms, call_host_ms, call_device_ms   medians of --reps calls at the first held-out view (after a warm-up, each ending in a device
                                           synchronise): the query (images = NULL), and the call with host (numpy) and device (torch)
                                           images and the truth image
  host_phases_ms, device_phases_ms         the library's CUDA-event phases of the last such call: pass A, pass B (host images: with the
                                           uploads it waits for), score
  needed, bytes_up                         the cameras that view samples and their image bytes
  psnr, mae, coverage                      means over the held-out views (device images)
Prints one JSON line per workload with the GPU's name, power limit and SM clock limit.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R_EXT = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])   # OpenCV camera axes in the sensor frame: z ahead, x right, y down
T_EXT = np.array([0.1, 0.0, 0.05])


def median_ms(fn, reps):
    import torch
    fn()   # warm-up
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return round(float(np.median(ts)) * 1e3, 3)


def painted(mesh, cam, seed=0):
    """the image of camera cam = (w, h, (fx, fy, cx, cy), R, t): a smooth seeded pattern of the world point under each pixel"""
    rng = np.random.default_rng(seed)
    f, ph = rng.uniform(0.5, 2.0, (3, 3)), rng.uniform(0, 2 * np.pi, 3)
    w, h, (fx, fy, cx, cy), R, t = cam
    Rr = np.asarray(R, np.float64).copy()
    Rr[:, 1:] = -Rr[:, 1:]   # the rasteriser's rotation of the OpenCV camera
    _, depth = mesh.render_view((fx, fy, cx, cy), w, h, 0.1, 1000.0, Rr, t)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    pc = np.stack([(xs - cx) / fx * depth, (ys - cy) / fy * depth, depth.astype(np.float64)], axis=-1)
    pw = pc @ np.asarray(R).T + t
    img = np.zeros((h, w, 3), np.uint8)
    for c in range(3):
        img[..., c] = np.clip(127.5 + 127.5 * np.sin(pw @ f[c] + ph[c]), 0, 255).astype(np.uint8)
    img[depth < 0] = 0
    return img


def run(config, n, reps):
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[config]
    scans = bench.get_stream(wl, 1 + n)
    d_ds = [torch.from_numpy(s["body_ds"]).cuda() for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).cuda() for s in scans]
    lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    poses = []
    for k in range(1, 1 + n):
        lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
        mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        s = lio.get_state()
        poses.append((s[0:9].reshape(3, 3).copy(), s[9:12].copy()))
    lio.wait()
    mesh.wait()
    out = {"config": config, "frames": n, "cameras": n, "triangles": mesh.counts()["n_triangles"]}
    for w, h in ((640, 480), (1224, 1024), (1920, 1080)):
        f = 0.85 * w
        cams = [(w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), R @ R_EXT, t + R @ T_EXT) for R, t in poses]
        imgs = [painted(mesh, c) for c in cams]
        even, odd = list(range(0, n, 2)), list(range(1, n, 2))
        train = [cams[k] for k in even]
        sel = mesh.texture_select(train, vertices=False)
        host = [imgs[k] for k in even]
        dev = [torch.from_numpy(im).cuda() for im in host]
        view, truth = cams[odd[0]], imgs[odd[0]]
        d_truth = torch.from_numpy(truth).cuda()
        q = mesh.render_textured(view, sel, train)
        need = [im if q["needed"][k] else None for k, im in enumerate(host)]
        r = dict(textured=sel["counts"]["textured"], needed=int(q["needed"].sum()), bytes_up=int(sum(im.nbytes for im in need if im is not None)))
        r["query_ms"] = median_ms(lambda: mesh.render_textured(view, sel, train), reps)
        r["call_host_ms"] = median_ms(lambda: mesh.render_textured(view, sel, train, need, truth=truth), reps)
        r["host_phases_ms"] = {k: round(v, 3) for k, v in mesh.render_textured_stats().items()}
        r["call_device_ms"] = median_ms(lambda: mesh.render_textured(view, sel, train, dev, truth=d_truth), reps)
        r["device_phases_ms"] = {k: round(v, 3) for k, v in mesh.render_textured_stats().items()}
        scores = [mesh.render_textured(cams[k], sel, train, dev, truth=torch.from_numpy(imgs[k]).cuda()) for k in odd]
        scores = [s for s in scores if s["counts"]["textured"] > 0]
        for key in ("psnr", "mae", "coverage"):
            r[key] = round(float(np.mean([s[key] for s in scores])), 3) if scores else None
        r["held_out_views"] = len(scores)
        out[f"{w}x{h}"] = r
        del dev, d_truth
    lio.close()
    mesh.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C100k,C3")
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for c in args.configs.split(","):
        out = run(c, args.scans, args.reps)
        out["gpu"] = gpu
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
