"""CPU tier: the mesh frame feed's rings (immesh_b200/csrc/mesh_feed.cuh: mfeed_head, mfeed_row_slot, mfeed_slot; the shared read
feed_read of lio_feed.cuh on mfeed_point_rings / mfeed_image_rings) in the host emulation tests/mesh_feed/emu_mesh_feed.cpp, against a
Python model of the rings -- points that wrap the point ring, a lost frame inside a range, an image ring shorter than the header ring,
a frame still in flight, header-ring wrap and resync from counts[2], a range before the enable, batched frames inside a range, capacity
errors and count queries, and the index guard refusing a slot outside its ring."""
import ctypes as C

import numpy as np
import pytest

HDR, POSE = 22, 36
FRAME, KIND, N_POINTS, STEP, COUNTS, ERR, HAS_ROT, T_BEGIN, T_END = 0, 1, 2, 3, 4, 12, 13, 14, 15
ROW_BEGIN, ROW_END, ROWS_LOST, RF, IMG_BEGIN, IMG_END = 16, 17, 18, 19, 20, 21
PUSH, FROM_LIO_ASYNC, BATCHED = 0, 3, 5
OK, E_CAPACITY, E_RANGE = 0, -3, -5
MERR_FEED_INDEX = 256
NPX = 6


@pytest.fixture(scope="module")
def emu():
    from immesh_b200 import build
    lib = C.CDLL(build.build_mesh_feed())
    lib.emu_mfeed_enable.argtypes = [C.c_longlong] * 4 + [C.c_int, C.c_longlong]
    lib.emu_mfeed_head.argtypes = [C.c_int, C.c_int, C.c_longlong, C.c_int]
    lib.emu_mfeed_head.restype = C.c_longlong
    lib.emu_mfeed_restore.argtypes = [C.c_longlong, C.c_longlong]
    lib.emu_mfeed_read.argtypes = [C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.emu_mfeed_read_images.argtypes = [C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


class Model:
    """the rings as include/immesh_b200.h states them"""

    def __init__(self, lib, max_frames, max_rows, max_images=0, depth=1, start=0):
        self.lib, self.max_frames, self.max_rows, self.max_images = lib, max_frames, max_rows, max_images
        lib.emu_mfeed_enable(max_frames, max_rows, max_images, NPX, depth, start)
        self.start = start
        self.frames = {}       # frame -> (kind, rf, nrf, row_begin, lost, img index or None)
        self.rows = 0
        self.imgs = 0
        self.queued = self.done = start

    def head(self, kind=PUSH, rf=1, nrf=0, img=0):
        f = self.queued + 1
        need = nrf if (rf and self.max_rows > 0) else 0
        lost = need > self.max_rows
        im = None
        if img and self.max_images > 0:
            im = self.imgs
            self.imgs += 1
        self.frames[f] = (kind, rf, nrf, self.rows, lost, im)
        if not lost:
            self.rows += need
        self.queued = f
        assert self.lib.emu_mfeed_head(kind, rf, nrf, img) == (f - 1) % self.max_frames

    def finish(self):
        self.lib.emu_mfeed_finish()
        self.done = self.queued

    def frame(self, **kw):
        self.head(**kw)
        self.finish()

    def expected_points(self, f):
        kind, rf, nrf, begin, lost, _ = self.frames[f]
        n = 0 if (lost or not rf or self.max_rows == 0) else nrf
        i = np.arange(n)
        pts = np.stack([np.full(n, f), i, f + i], axis=1).astype(np.float32)
        return pts, (f * 1000 + i).astype(np.int32)

    def expected_image(self, f):
        p = np.arange(NPX)
        rgba = ((f * 7 + p[:, None] * 3 + np.arange(4)[None, :]) & 255).astype(np.uint8)
        return rgba, (f + 0.5 * p).astype(np.float32)

    def read(self, since, cap_frames=None, cap_rows=None):
        counts = np.zeros(4, np.int64)
        rc = self.lib.emu_mfeed_read(since, None, None, 0, None, None, 0, counts.ctypes.data)
        if rc or cap_frames == 0:
            return rc, counts, None
        nf, nr = int(counts[0]), int(counts[1])
        cf = nf if cap_frames is None else cap_frames
        cr = nr if cap_rows is None else cap_rows
        hdr = np.zeros((max(cf, 1), HDR), np.int64)
        poses = np.zeros((max(cf, 1), POSE))
        pts = np.zeros((max(cr, 1), 3), np.float32)
        pix = np.zeros(max(cr, 1), np.int32)
        rc = self.lib.emu_mfeed_read(since, hdr.ctypes.data, poses.ctypes.data, cf, pts.ctypes.data, pix.ctypes.data, cr, counts.ctypes.data)
        return rc, counts, (hdr[:nf], poses[:nf], pts[:nr], pix[:nr])

    def read_images(self, since, cap=None):
        counts = np.zeros(4, np.int64)
        rc = self.lib.emu_mfeed_read_images(since, None, 0, None, None, counts.ctypes.data)
        if rc or cap == 0:
            return rc, counts, None
        nf, ni = int(counts[0]), int(counts[1])
        c = nf if cap is None else cap
        hdr = np.zeros((max(c, 1), HDR), np.int64)
        rgba = np.zeros((max(c, 1), NPX, 4), np.uint8)
        dep = np.zeros((max(c, 1), NPX), np.float32)
        rc = self.lib.emu_mfeed_read_images(since, hdr.ctypes.data, c, rgba.ctypes.data, dep.ctypes.data, counts.ctypes.data)
        return rc, counts, (hdr[:nf], rgba[:ni], dep[:ni])

    def check(self, since, out):
        hdr, poses, pts, pix = out
        fin = self.done
        assert hdr[:, FRAME].tolist() == list(range(since + 1, fin + 1))
        r0 = hdr[0, ROW_BEGIN]
        for i, f in enumerate(range(since + 1, fin + 1)):
            kind, rf, nrf, begin, lost, im = self.frames[f]
            h = hdr[i]
            assert h[KIND] == kind and h[N_POINTS] == 100 * f and h[STEP] == 1 + f % 3
            assert h[COUNTS:COUNTS + 8].tolist() == [f + k for k in range(8)] and h[ERR] == 0
            assert h[HAS_ROT] == (1 if kind == FROM_LIO_ASYNC else 0) and h[RF] == rf
            assert h[T_BEGIN] == 1000 * f and h[T_END] == 1000 * f + 10
            assert h[ROW_BEGIN] == begin and h[ROWS_LOST] == int(lost)
            ep, ex = self.expected_points(f)
            assert h[ROW_END] - h[ROW_BEGIN] == len(ep)
            assert np.array_equal(pts[h[ROW_BEGIN] - r0:h[ROW_END] - r0], ep)
            assert np.array_equal(pix[h[ROW_BEGIN] - r0:h[ROW_END] - r0], ex)
            assert h[IMG_END] - h[IMG_BEGIN] == (0 if im is None else 1) and (im is None or h[IMG_BEGIN] == im)
            assert np.array_equal(poses[i], f * 100.0 + np.arange(POSE))
        assert len(pts) == hdr[-1, ROW_END] - r0

    def check_images(self, since, out):
        hdr, rgba, dep = out
        assert hdr[:, FRAME].tolist() == list(range(since + 1, self.done + 1))
        k = 0
        for i, f in enumerate(range(since + 1, self.done + 1)):
            if self.frames[f][5] is None:
                continue
            er, ed = self.expected_image(f)
            assert np.array_equal(rgba[k], er) and np.array_equal(dep[k], ed)
            k += 1
        assert k == len(rgba)


def test_points_wrap_the_ring(emu):
    m = Model(emu, 16, 10)
    for n in (4, 3, 5, 2, 6):
        m.frame(nrf=n)
    rc, counts, out = m.read(3)   # frames 4, 5: rows 12..19, slots 2..9 -- the first of them written after the wrap
    assert rc == OK and counts.tolist() == [2, 8, 5, 5]
    m.check(3, out)
    rc, _, _ = m.read(2)          # frame 3 (rows 7..11) was overwritten by frame 5's rows
    assert rc == E_RANGE


def test_lost_frame_in_the_middle(emu):
    m = Model(emu, 16, 8)
    m.frame(nrf=3)
    m.frame(nrf=9)                # more than the ring: header and poses kept, no row written, nothing consumed
    m.frame(nrf=2)
    m.frame(rf=0, nrf=5)          # the reinforcement did not run: no rows, RF = 0
    rc, counts, out = m.read(0)
    assert rc == OK and counts[0] == 4 and counts[1] == 5
    m.check(0, out)
    assert out[0][1, ROWS_LOST] == 1 and out[0][1, ROW_BEGIN] == out[0][1, ROW_END] == 3 and out[0][3, RF] == 0


def test_no_point_ring(emu):
    m = Model(emu, 8, 0)
    m.frame(nrf=5)
    rc, counts, out = m.read(0)
    assert rc == OK and counts[1] == 0 and out[0][0, ROWS_LOST] == 0 and out[0][0, RF] == 1
    m.check(0, out)


def test_image_ring_shorter_than_header_ring(emu):
    m = Model(emu, 32, 64, max_images=3)
    for f in range(1, 7):
        m.frame(nrf=2, img=1)
    rc, counts, out = m.read_images(3)   # images 3, 4, 5 are held
    assert rc == OK and counts.tolist() == [3, 3, 6, 6]
    m.check_images(3, out)
    rc, counts, out = m.read_images(2)   # image 2 (frame 3) left the ring
    assert rc == E_RANGE and counts[2] == 6
    rc, counts, out = m.read(0)          # while its header, poses and points are still held
    assert rc == OK and counts[0] == 6
    m.check(0, out)


def test_frame_in_flight(emu):
    m = Model(emu, 4, 12, max_images=2)
    for _ in range(4):
        m.frame(nrf=3, img=1)
    m.head(nrf=3, img=1)                 # frame 5 marks slot 0 (frame 1's) and places rows 12..14 over frame 1's
    assert m.done == 4
    rc, counts, out = m.read(1)          # frames 2..4: their slots are intact
    assert rc == OK and counts.tolist() == [3, 9, 4, 5]
    m.check(1, out)
    rc, counts, _ = m.read(0)            # frame 1's slot is being rewritten
    assert rc == E_RANGE and counts[2] == 4
    rc, counts, out = m.read_images(2)   # images 2, 3 (frames 3, 4) -- image 4 of frame 5 goes over image 2's slot
    assert rc == E_RANGE
    rc, counts, out = m.read_images(3)
    assert rc == OK and counts[1] == 1
    m.check_images(3, out)
    m.finish()
    rc, counts, out = m.read(1)
    assert rc == OK and counts.tolist() == [4, 12, 5, 5]
    m.check(1, out)


def test_header_wrap_and_resync(emu):
    m = Model(emu, 4, 1000)
    for f in range(1, 11):
        m.frame(nrf=f)
    rc, counts, _ = m.read(2)            # 8 frames > 4 slots
    assert rc == E_RANGE and counts[2] == 10
    rc, counts, out = m.read(int(counts[2]) - 4)
    assert rc == OK and counts[0] == 4
    m.check(6, out)
    rc, counts, out = m.read(10)
    assert rc == OK and counts[0] == 0 and counts[2] == 10


def test_range_before_the_enable(emu):
    m = Model(emu, 8, 32, start=5)       # the handle had queued 5 frames when the feed was enabled
    m.frame(nrf=2)
    m.frame(nrf=2)
    rc, counts, out = m.read(5)
    assert rc == OK and counts.tolist() == [2, 4, 7, 7]
    m.check(5, out)
    for since in (0, 4):
        rc, counts, _ = m.read(since)
        assert rc == E_RANGE and counts[2] == 7
    m2 = Model(emu, 8, 32, start=5)
    rc, counts, _ = m2.read(3)           # nothing recorded yet, and the range holds frames before the enable
    assert rc == E_RANGE and counts[2] == 5


def test_batched_frames_inside_a_range(emu):
    m = Model(emu, 16, 32, max_images=4)
    m.frame(kind=FROM_LIO_ASYNC, nrf=3, img=1)
    m.frame(kind=BATCHED, rf=0, nrf=0, img=0)
    m.frame(kind=BATCHED, rf=0, nrf=0, img=0)
    m.frame(kind=FROM_LIO_ASYNC, nrf=4, img=1)
    rc, counts, out = m.read(0)
    assert rc == OK and counts[0] == 4 and counts[1] == 7
    m.check(0, out)
    rc, counts, out = m.read_images(0)
    assert rc == OK and counts[0] == 4 and counts[1] == 2
    m.check_images(0, out)
    h = out[0]
    assert h[1, IMG_BEGIN] == h[1, IMG_END] == 1 and h[2, ROW_BEGIN] == h[2, ROW_END] == 3


def test_capacity_and_count_queries(emu):
    m = Model(emu, 16, 64, max_images=4)
    for n in (5, 6, 7):
        m.frame(nrf=n, img=1)
    rc, counts, _ = m.read(0, cap_frames=0)
    assert rc == OK and counts.tolist() == [3, 18, 3, 3]
    rc, counts, out = m.read(0, cap_frames=2)
    assert rc == E_CAPACITY and counts[0] == 3 and not out[0].any()
    rc, counts, out = m.read(0, cap_rows=17)
    assert rc == E_CAPACITY and counts[1] == 18 and not out[2].any()
    rc, counts, _ = m.read_images(0, cap=0)
    assert rc == OK and counts.tolist() == [3, 3, 3, 3]
    rc, counts, out = m.read_images(1, cap=1)
    assert rc == E_CAPACITY and counts[0] == 2 and not out[1].any()
    rc, counts, out = m.read(0)
    assert rc == OK
    m.check(0, out)


def test_index_guard_refuses_out_of_ring_slots(emu):
    m = Model(emu, 8, 16, max_images=2)
    m.frame(nrf=3, img=1)
    # the header ring reported empty: the head refuses the slot and writes nothing, and no cursor moves
    emu.emu_mfeed_corrupt(0)
    assert emu.emu_mfeed_head(PUSH, 1, 3, 1) == -1
    emu.emu_mfeed_finish()
    assert emu.emu_mfeed_err() & MERR_FEED_INDEX
    emu.emu_mfeed_restore(8, 2)
    counts = np.zeros(4, np.int64)
    assert emu.emu_mfeed_read(0, None, None, 0, None, None, 0, counts.ctypes.data) == E_RANGE   # frame 2 was never written
    # a negative point cursor: every row slot is refused, nothing written
    m2 = Model(emu, 8, 16, max_images=2)
    m2.frame(nrf=3, img=1)
    emu.emu_mfeed_corrupt(1)
    assert emu.emu_mfeed_head(PUSH, 1, 3, 0) == 1
    emu.emu_mfeed_finish()
    assert emu.emu_mfeed_err() & MERR_FEED_INDEX
    # an image slot beyond the image ring: the copy refuses it
    m3 = Model(emu, 8, 16, max_images=2)
    m3.head(nrf=1, img=1)
    emu.emu_mfeed_corrupt(2)
    emu.emu_mfeed_finish()
    assert emu.emu_mfeed_err() & MERR_FEED_INDEX
