"""Where the pipelined step idles between kernels: the idle time at every kernel boundary of the localization and the mesh-frame
chains, from a torch.profiler trace (CUDA activities only) of bench.py's `value` pattern -- a 256 MB L2-flush write, step_async and
push_frame_from_lio_async per scan, device-resident inputs, graph-replayed, after the same map warm-up and warm-up steps.

  python tools/chain_gaps.py [--config C100k C4] [--steps 30] [--out DIR]

Per configuration and chain: busy time per scan (union of the chain's kernel intervals), idle time per scan (sum of the gaps
between a kernel's start and the latest end of the chain's kernels before it), and a per-edge table (predecessor -> successor,
median gap in us).  The mesh chain's triangulation side branches (k_voxel_tri_warp, k_pull_vertices) count as busy time of the
chain but are not edges of it.  The card name, power limit and SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # as bench.py

LIO_FIRST, MESH_FIRST = "k_predict", "k_transform_full"
LIO = {"k_predict", "k_reset_scan", "k_prepare", "k_match", "k_terms", "k_grow_point", "k_grow_segment", "k_grow_scatter",
       "k_grow_simple", "k_grow_voxel", "k_grow_finish", "k_pose_publish"}
MESH_SIDE = {"k_voxel_tri_warp", "k_pull_vertices"}


def kernel_name(full: str) -> str:
    n = full.split("(")[0].strip()
    return n[5:] if n.startswith("void ") else n


def card_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout
        return dict(zip(q.split(","), [x.strip() for x in out.strip().split(",")]))
    except Exception as e:   # noqa: BLE001
        return {"error": str(e)[:200]}


def chain_stats(spans, first):
    """spans: [(t0, t1, name)] of one chain sorted by start; split into scans at every `first` kernel."""
    scans, cur = [], None
    for s in spans:
        if s[2] == first:
            cur = []
            scans.append(cur)
        if cur is not None:
            cur.append(s)
    busy, idle, edges = [], [], {}
    for sc in scans[:-1] if len(scans) > 1 else scans:   # the last scan may be cut by the end of the trace
        b = g = 0.0
        end, prev = sc[0][0], None
        for t0, t1, name in sc:
            if name in MESH_SIDE:    # side branch of the fork/join: busy, no edge
                b += max(0.0, t1 - max(t0, end))
                end = max(end, t1)
                continue
            gap = max(0.0, t0 - end)
            if prev is not None:
                g += gap
                edges.setdefault((prev, name), []).append(gap)
            b += max(0.0, t1 - max(t0, end))
            end = max(end, t1)
            prev = name
        busy.append(b)
        idle.append(g)
    table = [{"edge": f"{a} -> {b}", "median_us": round(float(np.median(v)), 2), "mean_us": round(float(np.mean(v)), 2),
              "p90_us": round(float(np.percentile(v, 90)), 2), "n": len(v)} for (a, b), v in edges.items()]
    return {"scans": len(busy), "busy_us_per_scan": round(float(np.mean(busy)), 1), "idle_us_per_scan": round(float(np.mean(idle)), 1),
            "idle_us_per_scan_median_edges": round(sum(e["median_us"] * e["n"] for e in table) / max(1, len(busy)), 1),
            "edges_per_scan": round(sum(len(v) for v in edges.values()) / max(1, len(busy)), 1), "edges": table}


def measure(config, K):
    import torch
    import bench
    from immesh_b200 import api
    wl = bench.workloads()[config]
    W, MW = 5, wl["map_warm"]
    scans = bench.get_stream(wl, 1 + MW + W + K + 1)
    lib = api.load_library()
    dev = torch.device("cuda", 0)
    d_ds = [torch.from_numpy(s["body_ds"]).to(dev) for s in scans]
    d_full = [torch.from_numpy(s["body_full"]).to(dev) for s in scans]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lio, mesh = api.Lio(wl["lio"], lib=lib), api.Mesh(wl["mesh"], lib=lib)
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    k = 1
    for _ in range(MW):
        lio.step_dev(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"])
        mesh.push_frame_from_lio(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
        k += 1

    def enqueue(n):
        nonlocal k
        for _ in range(n):
            lio.enqueue_memset(flush.data_ptr(), flush.numel())
            lio.step_async(d_ds[k].data_ptr(), d_ds[k].shape[0], scans[k]["dt"], on_device=True)
            mesh.push_frame_from_lio_async(lio, d_full[k].data_ptr(), d_full[k].shape[0], on_device=True)
            k += 1
        lio.wait()
        mesh.wait()
        torch.cuda.synchronize()

    enqueue(W)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        enqueue(K)
    clocks = card_info()
    stats = api.graph_stats(lio, mesh)
    lio.close()
    mesh.close()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    kern = sorted((float(e["ts"]), float(e["ts"]) + float(e["dur"]), kernel_name(e["name"])) for e in ev if e.get("cat") == "kernel")
    fills = sorted(float(e["ts"]) for e in ev if e.get("cat") in ("gpu_memset", "Memset"))
    lio_sp = [s for s in kern if s[2] in LIO]
    mesh_sp = [s for s in kern if s[2] not in LIO]
    out = {"config": config, "steps": K, "card": clocks, "cuda_graphs": stats,
           "lio": chain_stats(lio_sp, LIO_FIRST), "mesh": chain_stats(mesh_sp, MESH_FIRST)}
    if kern:
        t0 = fills[0] if fills else kern[0][0]
        out["traced_us_per_scan"] = round((kern[-1][1] - t0) / K, 1)
        out["idle_share_of_step"] = round((out["lio"]["idle_us_per_scan"] + out["mesh"]["idle_us_per_scan"]) / out["traced_us_per_scan"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["C100k", "C4"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the result as DIR/chain_gaps.json")
    args = ap.parse_args()
    from immesh_b200 import build
    build.build_oracle()
    res = [measure(c, args.steps) for c in args.config]
    for r in res:
        print(f"== {r['config']}  {r['card']}  traced {r.get('traced_us_per_scan')} us/scan, idle share (both chains) {r.get('idle_share_of_step')}")
        for ch in ("lio", "mesh"):
            c = r[ch]
            print(f"  {ch:4s} busy {c['busy_us_per_scan']:8.1f} us/scan  idle {c['idle_us_per_scan']:7.1f} us/scan "
                  f"(at every edge's median gap: {c['idle_us_per_scan_median_edges']:.1f})  edges/scan {c['edges_per_scan']}")
            print("      median     mean      p90  (us)")
            for e in sorted(c["edges"], key=lambda e: -e["mean_us"]):
                print(f"    {e['median_us']:8.2f} {e['mean_us']:8.2f} {e['p90_us']:8.2f}  {e['edge']}  (n={e['n']})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "chain_gaps.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
