#!/usr/bin/env python
"""Time the colour equalisation (immesh_mesh_texture_gains) and score it by leave-one-out, on bench.py's workloads with
tools/texture_bench.py's meshes and cameras.

  python tools/texture_gains_bench.py [--configs C100k,C3] [--scans 30] [--reps 5]

Each workload's stream is localized and meshed through the queued chain; one camera per frame is posed from the frame's converged pose
and a fixed extrinsic (61-degree horizontal field of view), at 1224 x 1024 and 2448 x 2048.  Every camera's image shows a smooth seeded
pattern painted on the world (render_view's depth unprojected, coloured by the world point) multiplied per channel by a seeded gain in
[0.7, 1.3], rounded and clipped to 255: one exposure and white balance per camera.  Per size:
  call_host_ms, call_device_ms       medians of --reps calls with every camera's rows (texture_select over all cameras) and host (numpy)
                                     or device (torch) images, after a warm-up, each ending in a device synchronise
  host_phases_ms, device_phases_ms   the library's phases of the last such call: chosen samples, observer passes (CUDA events; host
                                     images: with the uploads they wait for), solve (host clock)
  pairs, samples, clipped, cg_iterations, observer_ms_per_camera
  loo                                texture_select with the even cameras, gains from their rows and images, apply_gains; every odd
                                     camera renders both textures against its unscaled painting: mean psnr_raw, psnr_equalised and
                                     coverage over the held-out views
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


def painted(mesh, cam, gain=(1.0, 1.0, 1.0), seed=0):
    """CUDA uint8 [h, w, 3]: the seeded world pattern under each pixel of cam = (w, h, (fx, fy, cx, cy), R, t), times gain per channel"""
    import torch
    rng = np.random.default_rng(seed)
    f, ph = rng.uniform(0.5, 2.0, (3, 3)), rng.uniform(0, 2 * np.pi, 3)
    w, h, (fx, fy, cx, cy), R, t = cam
    Rr = np.asarray(R, np.float64).copy()
    Rr[:, 1:] = -Rr[:, 1:]   # the rasteriser's rotation of the OpenCV camera
    _, depth = mesh.render_view((fx, fy, cx, cy), w, h, 0.1, 1000.0, Rr, t)
    d = torch.from_numpy(depth).cuda().double()
    ys, xs = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float64), torch.arange(w, device="cuda", dtype=torch.float64), indexing="ij")
    pc = torch.stack([(xs - cx) / fx * d, (ys - cy) / fy * d, d], dim=-1)
    pw = pc @ torch.from_numpy(np.asarray(R, np.float64).T.copy()).cuda() + torch.from_numpy(np.asarray(t, np.float64)).cuda()
    img = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
    for c in range(3):
        v = torch.clamp(127.5 + 127.5 * torch.sin(pw @ torch.from_numpy(f[c]).cuda() + ph[c]), 0, 255).floor()
        img[..., c] = torch.clamp(torch.floor(v * gain[c] + 0.5), 0, 255).to(torch.uint8)
    img[d < 0] = 0
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
    t_true = np.random.default_rng(17).uniform(0.7, 1.3, (n, 3))
    for w, h in ((1224, 1024), (2448, 2048)):
        f = 0.85 * w
        cams = [(w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), R @ R_EXT, t + R @ T_EXT) for R, t in poses]
        dev = [painted(mesh, c, t_true[k]) for k, c in enumerate(cams)]
        host = [im.cpu().numpy() for im in dev]
        sel = mesh.texture_select(cams, vertices=False)
        r = dict(textured=sel["counts"]["textured"])
        g = mesh.texture_gains(sel, cams, host)
        r.update({k: g["counts"][k] for k in ("pairs", "samples", "clipped", "cg_iterations")})
        r["call_host_ms"] = median_ms(lambda: mesh.texture_gains(sel, cams, host), reps)
        r["host_phases_ms"] = {k: round(v, 3) for k, v in mesh.texture_gains_stats().items()}
        r["call_device_ms"] = median_ms(lambda: mesh.texture_gains(sel, cams, dev), reps)
        r["device_phases_ms"] = {k: round(v, 3) for k, v in mesh.texture_gains_stats().items()}
        r["observer_ms_per_camera"] = round(r["device_phases_ms"]["observers"] / n, 3)
        r["apply_device_ms"] = median_ms(lambda: mesh.apply_gains(dev, g["gains"]), reps)
        # leave-one-out: even cameras texture, odd cameras score against the unscaled painting
        even, odd = list(range(0, n, 2)), list(range(1, n, 2))
        train = [cams[k] for k in even]
        tsel = mesh.texture_select(train, vertices=False)
        raw = [dev[k] for k in even]
        tg = mesh.texture_gains(tsel, train, raw)
        eq = mesh.apply_gains(raw, tg["gains"])
        loo = dict(raw=[], eq=[], coverage=[])
        for k in odd:
            truth = painted(mesh, cams[k])
            a = mesh.render_textured(cams[k], tsel, train, raw, truth=truth)
            if a["counts"]["textured"] == 0:
                continue
            b = mesh.render_textured(cams[k], tsel, train, eq, truth=truth)
            loo["raw"].append(a["psnr"]); loo["eq"].append(b["psnr"]); loo["coverage"].append(a["coverage"])
        r["loo"] = dict(views=len(loo["raw"]), psnr_raw=round(float(np.mean(loo["raw"])), 3), psnr_equalised=round(float(np.mean(loo["eq"])), 3),
                        coverage=round(float(np.mean(loo["coverage"])), 4))
        out[f"{w}x{h}"] = r
        del dev, host, raw, eq
        torch.cuda.empty_cache()
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
