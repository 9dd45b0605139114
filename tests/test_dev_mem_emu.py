"""CPU tier: the memory owner of the handles (immesh_b200/csrc/dev_mem.hpp), compiled for the host against allocation stubs
(tests/dev_mem/emu_dev_mem.cpp) that track every live block by kind and fail the k-th allocation on request.  For every k:
a growth-shaped transaction leaves the owning set as it was on failure and as expected on success, grow-only scratch frees
before it grows and is retryable after a failure, and no scenario leaves a block behind or frees one with the wrong call."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_dev_mem())
    for f in ("dm_transaction", "dm_regrow", "dm_allocs", "dm_live"):
        getattr(L, f).restype = C.c_longlong if f in ("dm_allocs", "dm_live") else C.c_int
    L.dm_transaction.argtypes = [C.c_longlong]
    L.dm_regrow.argtypes = [C.c_longlong, C.c_int]
    L.dm_live.argtypes = [C.c_int]
    return L


def _clean(lib):
    assert lib.dm_live(0) == 0 and lib.dm_live(1) == 0, "blocks left allocated"
    assert lib.dm_misuse() == 0, "a block was freed twice, unknown, or with the other kind's call"


def test_transaction_every_failure_point(lib):
    assert lib.dm_transaction(0) == 0
    n = lib.dm_allocs()
    assert n == 3
    for k in range(1, n + 2):   # each allocation of the transaction failing, then none (k = n + 1)
        line = lib.dm_transaction(k)
        assert line == 0, f"k={k}: check at emu_dev_mem.cpp:{line} failed"
        _clean(lib)


@pytest.mark.parametrize("pinned", [0, 1])
def test_regrow_every_failure_point(lib, pinned):
    for k in (0, 1, 2):
        line = lib.dm_regrow(k, pinned)
        assert line == 0, f"k={k}: check at emu_dev_mem.cpp:{line} failed"
        _clean(lib)


def test_memset_byte(lib):
    assert lib.dm_memset() == 0
    _clean(lib)


def test_kinds_and_moves(lib):
    assert lib.dm_kinds_and_moves() == 0
    _clean(lib)
