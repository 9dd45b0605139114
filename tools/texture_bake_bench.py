#!/usr/bin/env python
"""Time the texture atlas (immesh_mesh_texture_bake) on bench.py's workloads, with tools/texture_bench.py's meshes and cameras.

  python tools/texture_bake_bench.py [--configs C100k,C3] [--scans 30] [--reps 3] [--page 4096] [--max-cell 64]

Each workload's stream is localized and meshed through the queued chain; one camera per frame is posed from the frame's converged pose
and a fixed extrinsic (61-degree horizontal field of view), at 1224 x 1024 and at 2448 x 2048.  On the final mesh, texture_select picks
each facet's camera; then the bake runs from seeded random images, host (numpy) and device (torch) ones.  Medians of --reps calls after
a warm-up, each ending in a device synchronise:
  layout_ms          the count query (pages = NULL): the rows' upload, class, sorts, placement and the rows' read-back
  call_host_ms       the whole call with host images;  call_device_ms  with device images
  bake_kernel_ms     k_bake_texels over the call (CUDA events of the library's profiler, host images)
  upload_ms          the used images' host-to-device copies alone, timed with torch (pageable source)
  readback_ms        the pages' device-to-host copy alone, timed with torch (pageable destination)
  texels, bytes_up, bytes_down   computed from the shapes: texels written, used image bytes, page bytes
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


def run(config, n, reps, page, max_cell):
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
    nt = mesh.counts()["n_triangles"]
    out = {"config": config, "frames": n, "cameras": n, "triangles": nt, "page_size": page, "max_cell": max_cell}
    rng = np.random.default_rng(0)
    for w, h in ((1224, 1024), (2448, 2048)):
        f = 0.85 * w
        cams = [(w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), R @ R_EXT, t + R @ T_EXT) for R, t in poses]
        sel = mesh.texture_select(cams, vertices=False)
        used = set(sel["cam"][sel["cam"] >= 0].tolist())
        host = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) if k in used else None for k in range(n)]
        dev = [None if im is None else torch.from_numpy(im).cuda() for im in host]
        kw = dict(page_size=page, max_cell=max_cell)
        layout_ms = median_ms(lambda: _layout(mesh, sel, cams, host, page, max_cell), reps)
        r = mesh.texture_bake(sel, cams, host, **kw)
        call_host = median_ms(lambda: mesh.texture_bake(sel, cams, host, **kw), reps)
        call_dev = median_ms(lambda: mesh.texture_bake(sel, cams, dev, **kw), reps)
        api.profile_reset()
        api.profile_enable(True)
        for _ in range(reps):
            mesh.texture_bake(sel, cams, host, **kw)
        mesh.wait()   # harvests the profiler's events
        prof = api.profile_report()
        api.profile_enable(False)
        kern = prof.get("k_bake_texels", (0.0, 0))
        up = [im for im in host if im is not None]
        d_up = [torch.empty(im.shape, dtype=torch.uint8, device="cuda") for im in up]

        def upload():
            for d, im in zip(d_up, up):
                d.copy_(torch.from_numpy(im))
        pages_dev = torch.empty(r["pages"].shape, dtype=torch.uint8, device="cuda")
        pages_host = np.empty(r["pages"].shape, np.uint8)

        def readback():
            torch.from_numpy(pages_host).copy_(pages_dev)
        out[f"{w}x{h}"] = dict(cameras_used=len(used), textured=r["counts"]["textured"], cells=r["counts"]["cells"], n_pages=int(r["pages"].shape[0]),
                               layout_ms=layout_ms, call_host_ms=call_host, call_device_ms=call_dev,
                               bake_kernel_ms=round(kern[0] / reps, 3), bake_kernel_launches_per_call=kern[1] // reps, upload_ms=median_ms(upload, reps), readback_ms=median_ms(readback, reps),
                               texels=r["counts"]["texels"], bytes_up=int(sum(im.nbytes for im in up)), bytes_down=int(r["pages"].nbytes))
        del dev, d_up, pages_dev
    lio.close()
    mesh.close()
    return out


def _layout(mesh, sel, cams, host, page, max_cell):
    """the count query alone, through the C ABI"""
    import ctypes as C
    from immesh_b200 import api
    arr, n_cams = api.texture_cameras(cams)
    imgs, on_dev, keep = api.texture_images(host)
    cam = np.ascontiguousarray(sel["cam"], np.int32)
    uv = np.ascontiguousarray(sel["uv"], np.float32)
    cfg = api._AtlasCfg(page, max_cell, 0)
    npg = C.c_int(0)
    rc = mesh.lib.immesh_mesh_texture_bake(mesh._h, arr, n_cams, imgs, on_dev, cam.ctypes.data_as(C.POINTER(C.c_int32)), uv.ctypes.data_as(C.POINTER(C.c_float)),
                                           len(cam), C.byref(cfg), None, 0, None, None, C.byref(npg), None)
    assert rc == 0
    return npg.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C100k,C3")
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--page", type=int, default=4096)
    ap.add_argument("--max-cell", type=int, default=64)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for c in args.configs.split(","):
        out = run(c, args.scans, args.reps, args.page, args.max_cell)
        out["gpu"] = gpu
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
