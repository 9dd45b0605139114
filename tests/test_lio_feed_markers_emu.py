"""CPU tier: the scan feed's plane-marker rings (immesh_b200/csrc/lio_feed.cuh: marker_append, marker_rings, feed_read;
voxelmap.cuh: plane_pub_at) in the host emulation tests/lio_feed/emu_lio_feed_markers.cpp, against a Python model -- marker rows that
wrap the ring, a lost scan in the middle that consumes nothing, a scan in flight counted against the range, header ring wrap and
resync from counts[2], capacity and count queries."""
import ctypes as C

import numpy as np
import pytest

HDR, COLS = 10, 16
SCAN, ROW_BEGIN, ROW_END, ROWS_NEEDED, LOST, ROOTS_WALKED, PLANES = 0, 1, 2, 3, 4, 5, 6


@pytest.fixture(scope="module")
def emu():
    from immesh_b200 import build
    lib = C.CDLL(build.build_lio_feed_markers())
    lib.emu_mark_enable.argtypes = [C.c_longlong, C.c_longlong]
    lib.emu_mark_head.argtypes = [C.c_longlong]
    lib.emu_mark_read.argtypes = [C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


class Model:
    """the marker rings as include/immesh_b200.h states them: a lost scan writes nothing and leaves its rows pending"""

    def __init__(self, lib, max_scans, max_rows):
        self.lib, self.max_scans, self.max_rows = lib, max_scans, max_rows
        lib.emu_mark_enable(max_scans, max_rows)
        self.scans = []          # (begin, ids published, need, lost)
        self.pending, self.created, self.total, self.done = [], 0, 0, 0

    def head(self, fresh):
        self.pending += list(range(self.created, self.created + fresh))
        self.created += fresh
        need = len(self.pending)
        lost = need > self.max_rows
        self.scans.append((self.total, [] if lost else list(self.pending), need, lost))
        if not lost:
            self.total += need
        self.lib.emu_mark_head(fresh)

    def finish(self):
        self.lib.emu_mark_finish()
        if not self.scans[-1][3]:
            self.pending = []
        self.done = len(self.scans)

    def scan(self, fresh):
        self.head(fresh)
        self.finish()

    def consume(self):
        self.lib.emu_mark_consume()
        self.pending = []

    def read(self, since, cap_scans=None, cap_rows=None, with_rows=True):
        counts = np.zeros(4, np.int64)
        rc = self.lib.emu_mark_read(since, None, 0, None, 0, counts.ctypes.data)
        if rc or cap_scans == 0:
            return rc, counts, None
        ns, nr = int(counts[0]), int(counts[1])
        cs = ns if cap_scans is None else cap_scans
        cr = nr if cap_rows is None else cap_rows
        hdr = np.zeros((max(cs, 1), HDR), np.int64)
        rows = np.zeros((max(cr, 1), COLS))
        rc = self.lib.emu_mark_read(since, hdr.ctypes.data, cs, rows.ctypes.data if with_rows else None, cr, counts.ctypes.data)
        return rc, counts, (hdr[:ns], rows[:nr])

    def check(self, since, out):
        hdr, rows = out
        assert hdr[:, SCAN].tolist() == list(range(since + 1, self.done + 1))
        r0 = hdr[0, ROW_BEGIN]
        for i, k in enumerate(range(since + 1, self.done + 1)):
            begin, ids, need, lost = self.scans[k - 1]
            h = hdr[i]
            assert h[ROW_BEGIN] == begin and h[LOST] == int(lost) and h[ROWS_NEEDED] == need and h[ROOTS_WALKED] == need
            assert h[PLANES:].tolist() == [0, 1, 2, 3]
            assert h[ROW_END] - h[ROW_BEGIN] == len(ids)
            a, b = h[ROW_BEGIN] - r0, h[ROW_END] - r0
            expect = np.asarray(ids, np.float64)[:, None] * 100 + np.arange(COLS)
            assert np.array_equal(rows[a:b], expect.reshape(-1, COLS)), k


def test_rows_wrap_the_ring(emu):
    m = Model(emu, 64, 100)
    rng = np.random.default_rng(2)
    straddled = 0
    for k in range(1, 40):
        begin = m.total
        m.scan(int(rng.integers(1, 40)))
        straddled += begin % 100 + len(m.scans[-1][1]) > 100
        rc, counts, out = m.read(k - 1)
        assert rc == 0 and counts[0] == 1 and counts[2] == counts[3] == k
        m.check(k - 1, out)
        if k >= 3 and m.scans[k - 3][0] + 100 >= m.total:   # the last three scans' rows are still in the ring: one read across the wrap
            rc, _, out = m.read(k - 3)
            assert rc == 0
            m.check(k - 3, out)
    assert straddled >= 5


def test_lost_scan_in_the_middle_consumes_nothing(emu):
    m = Model(emu, 16, 100)
    m.scan(30)
    m.scan(120)      # 120 rows > max_rows: lost, no rows written, all of them stay pending
    m.scan(0)        # nothing was consumed: the same 120 rows are needed again
    m.consume()      # a blocking call takes them out of the feed
    m.scan(10)
    rc, counts, out = m.read(0)
    assert rc == 0 and counts[0] == 4 and counts[1] == 40
    m.check(0, out)
    hdr, rows = out
    assert hdr[1:3, LOST].tolist() == [1, 1] and hdr[1:3, ROWS_NEEDED].tolist() == [120, 120]
    assert (hdr[1:3, ROW_BEGIN] == 30).all() and (hdr[1:3, ROW_END] == 30).all()
    assert hdr[3, ROW_BEGIN] == 30 and rows[30, 0] == 150 * 100   # the last scan's own rows follow scan 1's at once


def test_scan_in_flight_is_counted_against_the_range(emu):
    m = Model(emu, 16, 100)
    for _ in range(3):
        m.scan(30)                       # rows 0..89
    rc, counts, out = m.read(0)
    assert rc == 0
    m.check(0, out)
    m.head(30)                           # rows 90..119 placed but not written: scan 1's slots 0..19 are taken
    rc, counts, _ = m.read(0)
    assert rc == -5 and counts[2] == 3 and counts[3] == 4
    rc, counts, out = m.read(1)          # scans 2 and 3 (rows 30..89) are untouched
    assert rc == 0 and counts[0] == 2
    m.check(1, out)
    m.finish()
    rc, counts, out = m.read(3)
    assert rc == 0
    m.check(3, out)


def test_header_ring_wrap_and_resync(emu):
    m = Model(emu, 4, 1000)
    for _ in range(10):
        m.scan(7)
    rc, counts, _ = m.read(0)
    assert rc == -5 and counts[2] == 10       # scans 1..6 left the header ring: resync from counts[2]
    rc, counts, out = m.read(int(counts[2]))
    assert rc == 0 and counts[0] == 0
    rc, counts, out = m.read(6)
    assert rc == 0 and counts[0] == 4
    m.check(6, out)
    m.head(7)                                  # scan 11 is rewriting scan 7's slot
    rc, counts, _ = m.read(6)
    assert rc == -5 and counts[2] == 10
    rc, counts, out = m.read(7)
    assert rc == 0 and counts[0] == 3
    m.check(7, out)


def test_capacity_and_count_query(emu):
    m = Model(emu, 16, 100)
    for _ in range(3):
        m.scan(15)
    rc, counts, _ = m.read(0, cap_scans=0)
    assert rc == 0 and counts.tolist() == [3, 45, 3, 3]
    rc, counts, out = m.read(0, cap_scans=2)
    assert rc == -3 and counts.tolist() == [3, 45, 3, 3] and not out[0].any()
    rc, counts, out = m.read(0, cap_rows=44)
    assert rc == -3 and not out[0].any()
    rc, counts, out = m.read(0, cap_rows=0, with_rows=False)   # no rows asked: the row cap does not apply
    assert rc == 0 and out[0][:, SCAN].tolist() == [1, 2, 3]
    rc, counts, out = m.read(0)
    assert rc == 0
    m.check(0, out)
