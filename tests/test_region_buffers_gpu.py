"""GPU tier: the viewer's region buffers (immesh_mesh_region_buffers: synchronize_triangle_list_for_disp -> unparse_triangle_set_to_vector
+ get_axis_min_max with the lazy smooth_pts) on the CUDA library against the oracle's literal walk, bit for bit, with the mesh of later
frames compared too; and the pipelined entry points against the blocking ones with the same calls between frames."""
import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL
from region_buffers_common import BOX0, RegionOracle, check_mesh, compare_call, run_region_parity, same_bits, subset_keys

pytestmark = pytest.mark.gpu


def test_avia_push_frame_bit_exact(cuda_lib):
    g, o, stats = run_region_parity(cuda_lib, "avia", 7, seed=0)
    assert min(s for _, s in stats[1:]) > 0 and stats[-1][0] > 10000


def test_hdl64_push_frame_bit_exact(cuda_lib):
    g, o, stats = run_region_parity(cuda_lib, "hdl64", 6, seed=2)
    assert stats[-1][0] > 5000


def test_knn_and_region_size_variants(cuda_lib):
    g, o, _ = run_region_parity(cuda_lib, "avia", 3, seed=6, call_after=())
    for knn, rs in ((1, 10.0), (8, 2.0), (32, 0.7)):
        compare_call(g, o, rs, subset_keys(o, rs, every=2), knn=knn, smooth_factor=0.5)
        compare_call(g, o, rs, None, knn=knn)
    assert g.region_buffers(2.0)[4] == 0


def _pipeline(lib, mode, calls, n_scans=7, seed=8):
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    out = []
    for k in range(1, n_scans):
        if mode == "sync":
            lio.step(scans[k]["body_ds"], scans[k]["dt"])
            mesh.push_frame_from_lio(lio, scans[k]["body_full"])
        else:
            lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
            mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if k in calls:   # the call itself waits for the queued frames; nothing else does in the async mode
            for keys in (np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0]], np.int32), None):
                box = BOX0.copy()
                out.append((mesh.region_buffers(2.0, keys, 1.0, 20, box), box))
    if mode == "async":
        lio.wait()
        mesh.wait()
    out.append(mesh.snapshot())
    return out


@pytest.mark.parametrize("graph", ["1", "0"])
def test_pipelined_calls_between_frames(cuda_lib, monkeypatch, graph):
    """graph-replayed push_frame_from_lio_async (IMMESH_GRAPH=1) and its direct launches (0), calls queued between frames, against the
    blocking push_frame_from_lio with the same calls"""
    monkeypatch.setenv("IMMESH_GRAPH", graph)
    calls = (2, 4, 6)
    a = _pipeline(cuda_lib, "sync", calls)
    b = _pipeline(cuda_lib, "async", calls)
    assert len(a) == len(b) == 2 * len(calls) + 1
    for (ra, ba), (rb, bb) in zip(a[:-1], b[:-1]):
        assert same_bits(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[3], rb[3]) and ra[4] == rb[4]
        assert np.array_equal(ba.view(np.uint32), bb.view(np.uint32))
    for x, y in zip(a[-1], b[-1]):
        assert np.array_equal(x, y)
    assert a[1][0][0].shape[0] > 1000 and a[1][0][4] > 0


def test_contract_on_device(cuda_lib):
    import ctypes as C
    g, o, _ = run_region_parity(cuda_lib, "avia", 3, seed=5, call_after=())
    i32, f32 = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    nr, nt, ns = C.c_int(0), C.c_int(0), C.c_int(0)
    before = g.snapshot()
    rows = np.zeros((4, 9), np.float32)
    assert cuda_lib.immesh_mesh_region_buffers(g._h, 2.0, None, 0, 1.0, 20, rows.ctypes.data_as(f32), None, 4, None, None, 1 << 20, None,
                                               C.byref(nr), C.byref(nt), C.byref(ns)) == -3
    assert nt.value == len(before[1]) and nr.value > 1 and ns.value == 0
    assert cuda_lib.immesh_mesh_region_buffers(g._h, 2.0, None, 0, 1.0, 20, None, None, 1 << 24, None, None, 1, None, C.byref(nr), C.byref(nt), C.byref(ns)) == -3
    rep = np.array([[0, 0, 0], [0, 0, 0]], np.int32)
    assert cuda_lib.immesh_mesh_region_buffers(g._h, 2.0, rep.ctypes.data_as(i32), 2, 1.0, 20, None, None, 0, None, None, 0, None, C.byref(nr), C.byref(nt), C.byref(ns)) == -1
    for bad in ((0.0, 20), (2.0, 0), (2.0, 33)):
        assert cuda_lib.immesh_mesh_region_buffers(g._h, bad[0], None, 0, 1.0, bad[1], None, None, 0, None, None, 0, None, C.byref(nr), C.byref(nt), C.byref(ns)) == -1
    compare_call(g, o, 2.0, None)       # nothing was smoothed by the refused calls: the oracle agrees on every smoothed count
    e = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    xyz, ids, keys, offs, n = e.region_buffers(2.0)
    assert xyz.shape == (0, 9) and keys.shape == (0, 3) and offs.tolist() == [0] and n == 0
    xyz, ids, keys, offs, n = e.region_buffers(2.0, np.array([[1, 2, 3]], np.int32))
    assert offs.tolist() == [0, 0] and keys.tolist() == [[1, 2, 3]]


def test_c100k_one_stream(cuda_lib):
    """one stream with bench.py's C100k settings (taken from bench.workloads(), so the two cannot drift), world frames from the
    true poses, calls after frames 1 and 3 against the oracle"""
    import bench
    w = bench.workloads()["C100k"]
    sensor, scans = synth.make_stream(w["kind"], 4, seed=21, leaf=w["lio"].filter_size_surf, ext_T=w["lio"].ext_T)
    g, o = api.Mesh(w["mesh"], lib=cuda_lib), RegionOracle(w["mesh"])
    for k, s in enumerate(scans):
        world = (s["body_full"].astype(np.float64) @ s["R_true"].T + s["t_true"]).astype(np.float32)
        g.push_frame(world, s["t_true"], k)
        o.push_frame(world, s["t_true"], k)
        if k in (1, 3):
            compare_call(g, o, 10.0, subset_keys(o, 10.0))
            rg, _ = compare_call(g, o, 10.0, None)
            check_mesh(g, o, f"frame {k}")
    assert rg[0].shape[0] > 10000
