"""CPU tier: growth of the VoxelMap pools (immesh_lio_reserve / immesh_lio_set_growth) on the host emulation of the device code
(tests/growth/emu_growth.cpp, which runs the migration bodies and the growth policy of immesh_b200/csrc/pool_growth.cuh):
the root-hash rebuild on adversarial key sets, and whole streams from tiny capacities against the oracle."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api
from pool_growth_common import doublings, run_growth_parity


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = api.load_library(build.build_growth())
    L.emu_hash_home.argtypes = [C.c_uint64, C.c_int]
    L.emu_growth_set_order.argtypes = [C.c_uint]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def rehash(lib, keys, marks, log2_old, log2_new):
    n = len(keys)
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    marks = np.ascontiguousarray(marks, dtype=np.int32)
    slot, root, mark, node_slot, lst, lkey = (np.zeros(max(n, 1), np.int32) for _ in range(6))
    m = lib.emu_rehash_check(_p(keys), _p(marks), n, log2_old, log2_new, _p(slot), _p(root), _p(mark), _p(node_slot), _p(lst), _p(lkey))
    assert m >= 0, f"table setup / rebuild failed ({m})"
    return slot[:n], root[:n], mark[:n], node_slot[:n], lst[:m], lkey[:m]


def pack(k):
    k = np.asarray(k, dtype=np.int64) + 1048576
    return ((k[:, 0].astype(np.uint64) << np.uint64(42)) | (k[:, 1].astype(np.uint64) << np.uint64(21)) | k[:, 2].astype(np.uint64))


def colliding_keys(lib, rng, log2, n, home):
    """n distinct packed keys whose home slot in a table of 2^log2 slots is in `home`"""
    out = set()
    while len(out) < n:
        cand = pack(rng.integers(-5000, 5000, size=(4096, 3)))
        for c in cand:
            if lib.emu_hash_home(int(c), log2) in home:
                out.add(int(c))
                if len(out) == n:
                    break
    return np.array(sorted(out), dtype=np.uint64)


@pytest.mark.parametrize("case", ["random", "one_home", "wrap_around"])
@pytest.mark.parametrize("order", [0, 7])
def test_root_rehash_keeps_every_key_and_back_pointer(lib, case, order):
    rng = np.random.default_rng(11)
    lib.emu_growth_set_order(order)
    log2_old = 8
    if case == "random":
        keys = np.unique(pack(rng.integers(-3000, 3000, size=(230, 3))))
    elif case == "one_home":      # one long probe chain: every key has the same home slot
        keys = colliding_keys(lib, rng, log2_old, 120, {37})
    else:                         # chains that run off the end of the old table and continue at slot 0
        keys = np.concatenate([colliding_keys(lib, rng, log2_old, 40, {254, 255}), colliding_keys(lib, rng, log2_old, 30, {0, 1})])
    marks = (rng.random(len(keys)) < 0.4).astype(np.int32)
    for log2_new in (log2_old + 1, log2_old + 3):
        slot, root, mark, node_slot, lst, lkey = rehash(lib, keys, marks, log2_old, log2_new)
        assert (slot >= 0).all(), "a key is not found after the rebuild"
        assert np.array_equal(root, np.arange(len(keys))), "root_node does not follow its key"
        assert np.array_equal(mark, marks), "pub_mark does not follow its key"
        assert np.array_equal(node_slot, slot), "NodeRec::root_slot does not point at the root's new slot"
        assert len(lst) == marks.sum() and np.array_equal(lst, slot[lkey]), "pub_list entries do not point at the new slots"
    lib.emu_growth_set_order(0)


def test_avia_stream_from_tiny_handle(lib):
    lib.emu_growth_set_order(5)
    r = run_growth_parity(lib, "avia", api.AVIA, n_scans=12, seed=0)
    lib.emu_growth_set_order(0)
    d = doublings(r["first"], r["last"])
    assert all(v >= 3 for v in d.values()), d
    r["handle"].close()


def test_hdl64_stream_from_tiny_handle(lib):
    lib.emu_growth_set_order(9)
    r = run_growth_parity(lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768)
    lib.emu_growth_set_order(0)
    d = doublings(r["first"], r["last"])
    assert all(v >= 3 for v in d.values()), d
    r["handle"].close()


def test_explicit_reserve_between_scans(lib):
    # growth off; reserve at every scan boundary: x4, a no-op request, +1 record, in turn
    def before(g, k):
        c = g.capacity()
        f = (4, 0, 1)[k % 3]
        if f == 0:
            g.reserve(c["root_slots"], c["nodes_cap"], c["chunks_cap"])
        elif f == 1:
            g.reserve(c["root_slots"] + 1, c["nodes_cap"] + 1, c["chunks_cap"] + 1)
        else:
            g.reserve(c["root_slots"] * 4, c["nodes_cap"] * 4, c["chunks_cap"] * 4)
    r = run_growth_parity(lib, "avia", api.AVIA, n_scans=8, seed=2, growth=0, before_scan=before)
    r["handle"].close()


@pytest.mark.parametrize("order", [0, 3])
def test_mesh_tables_rehash(lib, order):
    # the mesh-voxel hash (every per-voxel row -- chunk ids, count, meshing_times, new_added, frame -- follows its key) and the
    # triangle triple hash (every triple ever added, removed ones included, maps to its old index), on one long probe chain
    rng = np.random.default_rng(2)
    lib.emu_growth_set_order(order)
    log2_old = 9
    vkeys = np.concatenate([colliding_keys(lib, rng, log2_old, 60, {511, 0}), np.unique(pack(rng.integers(-900, 900, size=(150, 3))))])
    vkeys = np.unique(vkeys)
    tris = np.sort(rng.integers(0, 1 << 19, size=(200, 3)), axis=1)
    tris = np.unique(tris[(tris[:, 0] < tris[:, 1]) & (tris[:, 1] < tris[:, 2])], axis=0).astype(np.int32)
    for log2_new in (log2_old + 1, log2_old + 2):
        bad = lib.emu_mesh_rehash_check(_p(np.ascontiguousarray(vkeys, dtype=np.uint64)), len(vkeys), _p(np.ascontiguousarray(tris)), len(tris),
                                        log2_old, log2_new)
        assert bad == 0, f"{bad} keys / triples lost or moved without their rows"
    lib.emu_growth_set_order(0)


def _targets(lib, fn, c, steps, n, *rest, caps):
    cc = np.zeros(64, np.int32)
    for k, v in c.items():
        cc[k] = v
    out = np.array(caps, dtype=np.int64)
    getattr(lib, fn)(_p(cc), C.c_longlong(steps), C.c_longlong(n), *[C.c_int(r) for r in rest], _p(out))
    return [int(v) for v in out]


def test_growth_policy_with_steps_in_flight(lib):
    # localization, counters by slot (lio_core.cuh): 5 IM_LC_ROOTS, 0 IM_LC_NODES, 1 IM_LC_CHUNK_BUMP, 2 IM_LC_AVAIL_TOP (free-list
    # top); every result is the least doubling that satisfies the documented rule, for one step and for the five a full pipeline can hold
    c = {5: 3000, 0: 3100, 1: 4000, 2: 200}
    for steps in (1, 2, 5):
        cap, nodes, chunks = _targets(lib, "emu_growth_targets", c, steps, 1000, 700, 900, caps=[1024, 4096, 4096])
        assert (3000 + steps * 1000) * 2 <= cap and (cap == 1024 or (3000 + steps * 1000) * 2 > cap // 2)
        for capac, used, per in ((nodes, 3100, max(1400, 1000)), (chunks, 3800, max(1800, 1000))):
            assert capac - used >= max(capac // 4, steps * per)
            half = capac // 2
            assert capac == 4096 or half - used < max(half // 4, steps * per)
    # the mesh, counters by slot (mesh_core.cuh): 0 IM_MC_VERTICES, 27 IM_MC_VERT_CHUNKS, 4 IM_MC_VOXELS, 1 IM_MC_TRIS_ALLOC
    c = {0: 5000, 27: 2000, 4: 1500, 1: 20000}
    for steps in (1, 3):
        v, t, x = _targets(lib, "emu_mesh_growth_targets", c, steps, 800, 9000, caps=[6000, 21000, 2000])
        assert v - 5000 >= max(v // 4, steps * 800) and v // 4 + 1024 - 2000 >= max((v // 4 + 1024) // 4, steps * 800)
        assert x - 1500 >= max(x // 4, steps * 800)
        assert t - 20000 >= max(t // 4, steps * max(18000, 8 * 800))
