"""CPU tier: the scan feed's rings (immesh_b200/csrc/lio_feed.cuh: feed_append, feed_check_range, feed_read) in the host emulation
tests/lio_feed/emu_lio_feed.cpp, against a Python model of the rings -- rows that wrap the row ring, a lost scan in the middle of a
range, the conservative check against a scan still in flight, header ring wrap and resync from counts[2], capacity and count queries."""
import ctypes as C

import numpy as np
import pytest

HDR = 12
SCAN, ROW_BEGIN, ROW_EFFECT_END, ROW_END, ROWS_LOST = 0, 7, 8, 9, 11


@pytest.fixture(scope="module")
def emu():
    from immesh_b200 import build
    lib = C.CDLL(build.build_lio_feed())
    lib.emu_feed_enable.argtypes = [C.c_longlong, C.c_longlong, C.c_int]
    lib.emu_feed_head.argtypes = [C.c_longlong, C.c_longlong]
    lib.emu_feed_read.argtypes = [C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


class Model:
    """the rings as the documentation states them"""

    def __init__(self, lib, max_scans, max_rows, effect=1):
        self.lib, self.max_scans, self.max_rows = lib, max_scans, max_rows
        lib.emu_feed_enable(max_scans, max_rows, effect)
        self.scans = []          # (ne, nr, begin, lost)
        self.total = 0
        self.done = 0            # the newest finished scan

    def head(self, ne, nr):
        lost = ne + nr > self.max_rows
        self.scans.append((ne, nr, self.total, lost))
        if not lost:
            self.total += ne + nr
        self.lib.emu_feed_head(ne, nr)

    def finish(self):
        self.lib.emu_feed_finish()
        self.done = len(self.scans)

    def scan(self, ne, nr):
        self.head(ne, nr)
        self.finish()

    def expected_rows(self, k):
        ne, nr, _, lost = self.scans[k - 1]
        if lost:
            return np.zeros((0, 4), np.float32), np.zeros(0, np.int32)
        j = np.arange(ne + nr)
        rows = np.stack([np.full(j.shape, k), j, k + j, np.where(j < ne, 1, 2)], axis=1).astype(np.float32)
        return rows, np.where(j < ne, j * 3 + 1, -1).astype(np.int32)

    def read(self, since, cap_scans=None, cap_rows=None, with_rows=True):
        counts = np.zeros(4, np.int64)
        rc = self.lib.emu_feed_read(since, None, None, 0, None, None, 0, counts.ctypes.data)
        if rc or cap_scans == 0:
            return rc, counts, None
        ns, nr = int(counts[0]), int(counts[1])
        cs = ns if cap_scans is None else cap_scans
        cr = nr if cap_rows is None else cap_rows
        hdr = np.zeros((max(cs, 1), HDR), np.int64)
        st = np.zeros((max(cs, 1), 348))
        rows = np.zeros((max(cr, 1), 4), np.float32)
        idx = np.zeros(max(cr, 1), np.int32)
        rc = self.lib.emu_feed_read(since, hdr.ctypes.data, st.ctypes.data, cs, rows.ctypes.data if with_rows else None, idx.ctypes.data, cr,
                                    counts.ctypes.data)
        return rc, counts, (hdr[:ns], st[:ns], rows[:nr], idx[:nr])

    def check(self, since, out):
        hdr, st, rows, idx = out
        fin = self.done
        assert hdr[:, SCAN].tolist() == list(range(since + 1, fin + 1))
        r0 = hdr[0, ROW_BEGIN]
        for i, k in enumerate(range(since + 1, fin + 1)):
            ne, nr, begin, lost = self.scans[k - 1]
            h = hdr[i]
            assert h[ROW_BEGIN] == begin and h[ROWS_LOST] == int(lost)
            assert h[ROW_END] - h[ROW_BEGIN] == (0 if lost else ne + nr) and h[ROW_EFFECT_END] - h[ROW_BEGIN] == (0 if lost else ne)
            assert np.array_equal(st[i], k * 1000.0 + np.arange(348))
            er, ei = self.expected_rows(k)
            a, b = h[ROW_BEGIN] - r0, h[ROW_END] - r0
            assert np.array_equal(rows[a:b], er) and np.array_equal(idx[a:b], ei), k


def test_rows_wrap_the_ring(emu):
    m = Model(emu, 64, 100)
    rng = np.random.default_rng(1)
    straddled = 0
    for k in range(1, 40):
        ne, nr = int(rng.integers(0, 25)), int(rng.integers(1, 30))
        begin = m.total
        m.scan(ne, nr)
        straddled += begin % 100 + ne + nr > 100
        rc, counts, out = m.read(k - 1)
        assert rc == 0 and counts.tolist()[:1] == [1] and counts[2] == counts[3] == k
        m.check(k - 1, out)
        if k >= 3 and m.scans[k - 3][2] + 100 >= m.total:   # the last three scans' rows still in the ring: one read across the wrap
            rc, _, out = m.read(k - 3)
            assert rc == 0
            m.check(k - 3, out)
    assert straddled >= 5


def test_lost_scan_in_the_middle(emu):
    m = Model(emu, 16, 100)
    m.scan(20, 10)
    m.scan(70, 50)       # 120 rows > max_rows: header and state kept, no rows
    m.scan(10, 10)
    m.scan(0, 0)         # an empty scan
    rc, counts, out = m.read(0)
    assert rc == 0 and counts[0] == 4 and counts[1] == 50
    m.check(0, out)
    assert out[0][1, ROWS_LOST] == 1 and out[0][1, ROW_BEGIN] == out[0][1, ROW_END] == 30


def test_scan_in_flight_is_counted_against_the_range(emu):
    m = Model(emu, 16, 100)
    for _ in range(3):
        m.scan(10, 20)                       # rows 0..89
    rc, counts, out = m.read(0)
    assert rc == 0
    m.check(0, out)
    m.head(10, 20)                           # rows 90..119 placed but not written: scan 1's slots 0..19 are taken
    rc, counts, _ = m.read(0)
    assert rc == -5 and counts[2] == 3 and counts[3] == 4
    rc, counts, out = m.read(1)              # scans 2 and 3 (rows 30..89) are untouched
    assert rc == 0 and counts[0] == 2
    m.check(1, out)
    m.finish()
    rc, counts, out = m.read(3)
    assert rc == 0
    m.check(3, out)


def test_header_ring_wrap_and_resync(emu):
    m = Model(emu, 4, 1000)
    for _ in range(10):
        m.scan(3, 4)
    rc, counts, _ = m.read(0)
    assert rc == -5 and counts[2] == 10       # scans 1..6 left the header ring: resync from counts[2]
    rc, counts, out = m.read(int(counts[2]))
    assert rc == 0 and counts[0] == 0
    rc, counts, out = m.read(6)
    assert rc == 0 and counts[0] == 4
    m.check(6, out)
    m.head(3, 4)                               # scan 11 is rewriting scan 7's slot
    rc, counts, _ = m.read(6)
    assert rc == -5 and counts[2] == 10
    rc, counts, out = m.read(7)
    assert rc == 0 and counts[0] == 3
    m.check(7, out)


def test_capacity_and_count_query(emu):
    m = Model(emu, 16, 100, effect=0)
    for _ in range(3):
        m.scan(0, 15)
    rc, counts, _ = m.read(0, cap_scans=0)
    assert rc == 0 and counts.tolist() == [3, 45, 3, 3]
    rc, counts, out = m.read(0, cap_scans=2)
    assert rc == -3 and counts.tolist() == [3, 45, 3, 3] and not out[0].any()
    rc, counts, out = m.read(0, cap_rows=44)
    assert rc == -3 and not out[0].any()
    rc, counts, out = m.read(0, cap_rows=0, with_rows=False)   # no rows asked: the row cap does not apply
    assert rc == 0 and out[0][:, SCAN].tolist() == [1, 2, 3]
    rc, counts, out = m.read(0)
    assert rc == 0 and (out[3] == -1).all()    # effect off: every row is a registered row
    m.check(0, out)
