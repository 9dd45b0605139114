"""CPU tier, world_size 2 over gloo: the scan publishers of a sharded handle (the split residual pass of tests/test_shard_gloo.py,
executed by the host emulation with the IESKF weights kept).  Each rank returns the effect rows of the matches it contributed; their
union ordered by scan index must be the single-process cloud, and the registered cloud must be the same on both ranks."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

N_SCANS = 5


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out_dir):
    import torch
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from immesh_b200 import api, synth
    from scan_pub_common import emu_scanpub_lib
    lib = emu_scanpub_lib()
    lib.emu_shard_bits.restype = C.POINTER(C.c_uint32)
    lib.emu_shard_acc.restype = C.POINTER(C.c_uint64)
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", N_SCANS, seed=0, ext_T=cfg.ext_T)
    g = api.Lio(cfg, lib=lib)
    lib.emu_lio_set_shard(g._h, rank, world)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    s = g.get_state()
    s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
    g.set_state(s)
    g.voxel_map_init(scans[0]["body_full"])
    out = {}
    for k in range(1, N_SCANS):
        body = np.ascontiguousarray(scans[k]["body_ds"], dtype=np.float32)
        g.predict(scans[k]["dt"])
        lib.emu_shard_begin(g._h, body.ctypes.data_as(C.POINTER(C.c_float)), body.shape[0])
        for it in range(cfg.max_iteration):
            lib.emu_shard_pass1(g._h)
            nw = C.c_int(0)
            bits = np.ctypeslib.as_array(lib.emu_shard_bits(g._h, C.byref(nw)), shape=(nw.value,))
            t = torch.from_numpy(bits.astype(np.int64))       # disjoint bits: SUM == OR
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
            bits[:] = t.numpy().astype(np.uint32)
            lib.emu_shard_pass2(g._h, it)
            acc = np.ctypeslib.as_array(lib.emu_shard_acc(g._h, it), shape=(60,))
            t = torch.from_numpy(acc.astype(np.int64))        # two's complement sums
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
            acc[:] = t.numpy().astype(np.uint64)
            if lib.emu_shard_solve(g._h, it):
                break
        g._last_n = body.shape[0]
        g.map_incremental_grow()
        rows, idx = g.effect_cloud()
        out[f"eff_{k}"], out[f"idx_{k}"] = rows, idx
        out[f"reg_{k}"] = g.registered_cloud(None, point_skip=2)
    np.savez(os.path.join(out_dir, f"scan_pub_{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_effect_rows_union_equals_single_process(tmp_path, built):
    from immesh_b200 import api, synth
    from scan_pub_common import ScanPubOracle
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", N_SCANS, seed=0, ext_T=cfg.ext_T)
    o = ScanPubOracle(cfg)
    o.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    s = o.get_state()
    s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
    o.set_state(s)
    o.voxel_map_init(scans[0]["body_full"])
    r0, r1 = np.load(tmp_path / "scan_pub_0.npz"), np.load(tmp_path / "scan_pub_1.npz")
    for k in range(1, N_SCANS):
        o.predict(scans[k]["dt"])
        o.lio_state_estimation(scans[k]["body_ds"])
        o.map_incremental_grow(scans[k]["body_ds"])
        ro, io = o.effect_cloud()
        idx = np.concatenate([r0[f"idx_{k}"], r1[f"idx_{k}"]])
        rows = np.concatenate([r0[f"eff_{k}"], r1[f"eff_{k}"]])
        order = np.argsort(idx, kind="stable")
        assert np.array_equal(idx[order], io), f"scan {k}: union of the ranks' effect indices"
        assert np.array_equal(rows[order].view(np.uint32), ro.view(np.uint32)), f"scan {k}: union of the ranks' effect rows"
        assert 0.2 < len(r0[f"idx_{k}"]) / len(io) < 0.8      # both ranks contributed
        reg = o.frame_world(scans[k]["body_ds"], 2)
        assert np.array_equal(r0[f"reg_{k}"], reg) and np.array_equal(r1[f"reg_{k}"], reg), f"scan {k}: registered rows"
