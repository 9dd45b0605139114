"""Times the batched offline mesher: immesh_mesh_push_frame_batched and immesh_mesh_reconstruct_from_pointcloud_batched on synthetic
clouds of translated Avia tiles (10 M and 50 M points by default), wall clock around the blocking calls, plus the CPU oracle's single
frame on a 2 M-point cloud for comparison.  Prints one JSON line per run.

  python tools/offline_mesh_bench.py [--points 10000000 50000000] [--batch-voxels 65536] [--oracle-points 2000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests")]

from immesh_b200 import api  # noqa: E402
from offline_batched_common import avia_cloud  # noqa: E402


def tiled(n_points, tile):
    k = -(-n_points // len(tile))
    ext = np.ptp(tile, axis=0) + 10.0
    side = int(np.ceil(np.sqrt(k)))
    out = np.concatenate([tile + np.array([(i % side) * ext[0], (i // side) * ext[1], 0.0], np.float32) for i in range(k)])
    return out[:n_points]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[10_000_000, 50_000_000])
    ap.add_argument("--batch-voxels", type=int, default=1 << 16)
    ap.add_argument("--oracle-points", type=int, default=2_000_000)
    a = ap.parse_args()
    tile = avia_cloud(3)
    cfg = api.MeshConfig(points_minimum_scale=0.1, voxel_resolution=0.4, number_of_pts_append_to_map=50_000_000, max_vertices=1 << 25,
                         max_triangles=1 << 26, max_voxels=1 << 23)
    for n in a.points:
        cloud = tiled(n, tile)
        for call in ("push_frame_batched", "reconstruct_from_pointcloud_batched"):
            g = api.Mesh(cfg)
            t0 = time.perf_counter()
            if call == "push_frame_batched":
                st = g.push_frame_batched(cloud, np.zeros(3), 0, a.batch_voxels)
            else:
                st = {"meshed_points": g.reconstruct_from_pointcloud_batched(api.VoxelGrid(1 << 20), cloud, 0.01, 0, a.batch_voxels)}
            ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({"call": call, "points": n, "ms": round(ms, 1), "points_per_s": round(n / ms * 1e3), **st, **g.counts()}), flush=True)
            g.close()
    from oracle_api import OracleMesh
    o = OracleMesh(cfg)
    cloud = tiled(a.oracle_points, tile)
    t0 = time.perf_counter()
    o.push_frame(cloud, np.zeros(3))
    ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"call": "oracle push_frame (CPU)", "points": len(cloud), "ms": round(ms, 1), "points_per_s": round(len(cloud) / ms * 1e3)}), flush=True)


if __name__ == "__main__":
    main()
