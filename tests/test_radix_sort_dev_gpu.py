"""GPU tier: the device-count radix sort (radix_sort.cuh: k_rs_hist_dev, k_rs_scan_dev, k_rs_scatter_dev), whose blocks loop over the
count's tiles, against the host-count sort and numpy's stable argsort.  Counts across tile boundaries (0, 1, 2047, 2048, 2049 and
several tiles), grids of one to three blocks (more tiles than blocks: each block sorts several tiles in turn) and a grid that covers
the capacity (one tile per block, as the mesh's change feed runs it); keys with many repeats, so that stability is visible.
Harness: tests/radix_sort/rs_check.cu."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 2048
CAP = 12 * TILE + 5


@pytest.fixture(scope="module")
def rs():
    from immesh_b200 import build
    lib = C.CDLL(build.build_rs_check())
    lib.rs_check_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.rs_check_dev.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    k[::3] = rng.integers(0, 40, k[::3].shape[0]).astype(np.uint32)   # repeated keys
    return k


def _sort(rs, keys, passes, grid=None):
    n = keys.shape[0]
    ko, vo = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    k = np.ascontiguousarray(keys) if n else np.zeros(1, np.uint32)
    if grid is None:
        rc = rs.rs_check_host(k.ctypes.data, n, passes, ko.ctypes.data, vo.ctypes.data)
    else:
        rc = rs.rs_check_dev(k.ctypes.data, n, CAP, passes, grid, ko.ctypes.data, vo.ctypes.data)
    assert rc == 0, rc
    return ko[:n], vo[:n]


@pytest.mark.parametrize("n", [0, 1, 2047, 2048, 2049, 5 * TILE + 7, CAP])
@pytest.mark.parametrize("grid", [1, 2, 3, 0])
@pytest.mark.parametrize("passes", [4, 2])
def test_device_count_any_grid_equals_host_count(rs, n, grid, passes):
    keys = _keys(n, seed=n * 7 + grid)
    kd, vd = _sort(rs, keys, passes, grid)
    masked = keys & np.uint32((1 << (8 * passes)) - 1) if passes < 4 else keys
    order = np.argsort(masked, kind="stable").astype(np.uint32)
    assert np.array_equal(vd, order) and np.array_equal(kd, keys[order])
    if n > 0:
        kh, vh = _sort(rs, keys, passes)
        assert np.array_equal(vd, vh) and np.array_equal(kd, kh)
