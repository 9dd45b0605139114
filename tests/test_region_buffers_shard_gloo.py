"""CPU tier, world_size 2 over gloo: the sharded mesher (per-voxel stage by voxel owner, the smoothed positions and the facet lists
exchanged between the stages, as tests/test_shard_gloo.py runs it) executed by the host emulation, with region-buffer calls between
frames.  Every replica holds the same triangle store, smoothed positions and m_smoothed flags, so every rank must return the
oracle's rows, and the later frames must stay equal to the oracle that made the same calls."""
import ctypes as C
import os

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from test_shard_gloo import _free_port, _gather_padded

N_FRAMES, CALLS, RS = 5, (1, 3), 2.0


def _keys():
    return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [-1, -1, 0], [2, 1, 0]], np.int32)


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from immesh_b200 import api
    from mesh_common import SMALL, world_scans
    from region_buffers_common import BOX0, emu_regionbuf_lib
    lib = emu_regionbuf_lib()
    u64p, i32p = C.POINTER(C.c_uint64), C.POINTER(C.c_int)
    g = api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lib.emu_mesh_set_shard(g._h, rank, world)
    out = {}
    for k, (w, t) in enumerate(world_scans("avia", N_FRAMES, 3, 20000)):
        w = np.ascontiguousarray(w, dtype=np.float32)
        t = np.ascontiguousarray(t, dtype=np.float64)
        assert lib.emu_mesh_phase_a(g._h, w.ctypes.data_as(C.POINTER(C.c_float)), w.shape[0], t.ctypes.data_as(C.POINTER(C.c_double))) == 0
        c = (C.c_int * 3)()
        lib.emu_mesh_xcounts(g._h, c)
        sm = np.zeros(c[0] * 32, dtype=np.uint8)
        lib.emu_mesh_xget(g._h, sm.ctypes.data_as(C.c_void_p), None, None, None)
        for r, buf in enumerate(_gather_padded(sm, world)):
            if r != rank and buf.size:
                lib.emu_mesh_xapply_smooth(g._h, buf.ctypes.data_as(C.c_void_p), buf.size // 32)
        lib.emu_mesh_phase_b(g._h)
        lib.emu_mesh_xcounts(g._h, c)
        face = np.zeros((c[1], 4), dtype=np.int32); word = np.zeros(c[1], dtype=np.uint64); rem = np.zeros((c[2], 4), dtype=np.int32)
        lib.emu_mesh_xget(g._h, None, face.ctypes.data_as(i32p), word.ctypes.data_as(u64p), rem.ctypes.data_as(i32p))
        faces, words, rems = _gather_padded(face, world), _gather_padded(word, world), _gather_padded(rem, world)
        for r in range(world):
            f = np.ascontiguousarray(faces[r].view(np.int32)); wd = np.ascontiguousarray(words[r].view(np.uint64)); rm = np.ascontiguousarray(rems[r].view(np.int32))
            lib.emu_mesh_xapply_lists(g._h, f.ctypes.data_as(i32p), wd.ctypes.data_as(u64p), wd.size, rm.ctypes.data_as(i32p), rm.size // 4)
        assert lib.emu_mesh_phase_c(g._h) == 0
        if k in CALLS:
            for name, keys in (("sub", _keys()), ("all", None)):
                box = BOX0.copy()
                xyz, ids, rk, ro, ns = g.region_buffers(RS, keys, 1.0, 20, box)
                out.update({f"{name}{k}_xyz": xyz, f"{name}{k}_ids": ids, f"{name}{k}_rk": rk, f"{name}{k}_ro": ro, f"{name}{k}_ns": np.array(ns), f"{name}{k}_box": box})
    v, tri, fl = g.snapshot()
    np.savez(os.path.join(out_dir, f"rb_{rank}.npz"), v=v, tri=tri, fl=fl, **out)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_replicas_return_the_oracle_rows(tmp_path, built):
    from immesh_b200 import api
    from mesh_common import SMALL, world_scans
    from region_buffers_common import BOX0, RegionOracle, same_bits
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    o = RegionOracle(api.MeshConfig(**SMALL))
    ref = {}
    for k, (w, t) in enumerate(world_scans("avia", N_FRAMES, 3, 20000)):
        o.push_frame(w, t, k)
        if k in CALLS:
            for name, keys in (("sub", _keys()), ("all", None)):
                box = BOX0.copy()
                ref[name + str(k)] = (*o.region_buffers(RS, keys, 1.0, 20, box), box)
    vo, to, fo = o.snapshot()
    for rank in (0, 1):
        r = np.load(tmp_path / f"rb_{rank}.npz")
        for key, (xyz, ids, rk, ro, ns, box) in ref.items():
            assert same_bits(r[key + "_xyz"], xyz) and np.array_equal(r[key + "_ids"], ids), (rank, key)
            assert np.array_equal(r[key + "_rk"], rk) and np.array_equal(r[key + "_ro"], ro) and int(r[key + "_ns"]) == ns, (rank, key)
            assert np.array_equal(r[key + "_box"].view(np.uint32), box.view(np.uint32)), (rank, key)
        assert np.array_equal(r["v"], vo) and np.array_equal(r["tri"], to) and np.array_equal(r["fl"], fo), rank
    assert len(ref["all3"][0]) > 1000 and ref["all1"][4] > 0
