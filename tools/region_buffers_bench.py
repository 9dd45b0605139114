#!/usr/bin/env python
"""Time the viewer's region buffers, immesh_mesh_region_buffers (synchronize_triangle_list_for_disp -> unparse_triangle_set_to_vector +
get_axis_min_max), on the mesh one of bench.py's workloads ends with.

  python tools/region_buffers_bench.py --config C100k|C4|C5 [--scans 12] [--region-size 10] [--repeat 5]

The scans are localised and meshed through the blocking calls.  On the final mesh, three kinds of call are timed, each on a fresh copy
of the mesh state where it matters:
  first        every region, the first call after the frames (smooths every vertex the dilations left unsmoothed)
  repeat       every region again (smooths nothing)
  nbhd3x3      the 3 x 3 regions around the last sensor position (z = its region), on a mesh that has been through `first`
Median of the host clock around each blocking call, the row copy included (the count query that sizes the buffers is a call of its
own and is timed separately as `count_ms`).  Prints one JSON line with the GPU's name and power limit.  Writes nothing."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C100k", choices=["C100k", "C1", "C2", "C3", "C4", "C5"])
    ap.add_argument("--scans", type=int, default=12)
    ap.add_argument("--region-size", type=float, default=10.0)
    ap.add_argument("--repeat", type=int, default=5)
    args = ap.parse_args()
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[args.config]
    scans = bench.get_stream(wl, 1 + args.scans)
    rs = args.region_size

    def build_mesh():
        lio, mesh = api.Lio(wl["lio"]), api.Mesh(wl["mesh"])
        lio.set_state(bench.init_state_vec(scans))
        lio.voxel_map_init(scans[0]["body_full"])
        for k in range(1, 1 + args.scans):
            lio.step(scans[k]["body_ds"], scans[k]["dt"])
            mesh.push_frame_from_lio(lio, scans[k]["body_full"])
        return lio, mesh

    def call(mesh, keys):
        """(ms of the count query, ms of the call with rows, rows, vertices smoothed)"""
        lib = mesh.lib
        kp, nk = (None, 0) if keys is None else (keys.ctypes.data_as(C.POINTER(C.c_int32)), keys.shape[0])
        nr, nt, ns = C.c_int(0), C.c_int(0), C.c_int(0)
        t0 = time.perf_counter()
        lib.immesh_mesh_region_buffers(mesh._h, rs, kp, nk, 1.0, 20, None, None, 0, None, None, 0, None, C.byref(nr), C.byref(nt), C.byref(ns))
        t1 = time.perf_counter()
        xyz = np.empty((nt.value, 9), np.float32)
        ids = np.empty((nt.value, 3), np.int32)
        rk = np.empty((nr.value, 3), np.int32)
        ro = np.empty(nr.value + 1, np.int32)
        box = np.array([1e8] * 3 + [-1e8] * 3, np.float32)
        t2 = time.perf_counter()
        rc = lib.immesh_mesh_region_buffers(mesh._h, rs, kp, nk, 1.0, 20, xyz.ctypes.data_as(C.POINTER(C.c_float)), ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                            nt.value, rk.ctypes.data_as(C.POINTER(C.c_int32)), ro.ctypes.data_as(C.POINTER(C.c_int32)), nr.value,
                                            box.ctypes.data_as(C.POINTER(C.c_float)), C.byref(nr), C.byref(nt), C.byref(ns))
        t3 = time.perf_counter()
        assert rc == 0, rc
        return (t1 - t0) * 1e3, (t3 - t2) * 1e3, nt.value, ns.value

    res = {k: {"count_ms": [], "ms": [], "rows": [], "smoothed": []} for k in ("first", "repeat", "nbhd3x3")}
    for _ in range(args.repeat):
        lio, mesh = build_mesh()
        pos = lio.get_state()[9:12]
        c = np.round(pos / rs).astype(np.int32)
        nb = np.array([[c[0] + dx, c[1] + dy, c[2]] for dx in (-1, 0, 1) for dy in (-1, 0, 1)], np.int32)
        for name, keys in (("first", None), ("repeat", None), ("nbhd3x3", nb)):
            r = call(mesh, keys)
            for f, v in zip(("count_ms", "ms", "rows", "smoothed"), r):
                res[name][f].append(v)
        mesh.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"config": args.config, "gpu": gpu, "scans": args.scans, "region_size": rs, "repeat": args.repeat,
                      **{k: {"median_ms": round(float(np.median(v["ms"])), 4), "median_count_ms": round(float(np.median(v["count_ms"])), 4),
                             "rows_per_call": int(np.median(v["rows"])), "smoothed_per_call": int(np.median(v["smoothed"]))} for k, v in res.items()}}))


if __name__ == "__main__":
    main()
