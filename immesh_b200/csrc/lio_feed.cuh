// immesh_b200 -- the scan feed (immesh_lio_feed_enable / immesh_lio_feed): the device block its kernels share and the bookkeeping
// of its two rings, and those of its plane-map markers (immesh_lio_feed_markers_enable: a header ring beside the feed's, numbered
// like it, and a ring of marker rows).  Header and state ring: scan k (numbered 1, 2, ... from the enable) in slot (k - 1) % max_scans.  Row ring: the
// feed's rows are numbered in the order the scans append them, row r in slot r % max_rows; a scan's rows are its effect rows, then
// its registered rows.  The bookkeeping is __host__ __device__ and the read is host code, so that the host emulation
// (tests/lio_feed/emu_lio_feed.cpp) runs both as the product does.
// The read (feed_check_range, FeedRings, feed_read) is not specific to scans: it serves any ring of numbered headers with a fixed
// record of doubles beside each and a row ring of one or two per-row arrays -- the mesh frame feed (mesh_feed.cuh) reads its
// points and its images through it too.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "lio_core.cuh"

namespace immesh {

// per-scan inputs of the feed's kernels (one H2D copy per scan, like ScanDyn): the launch sequence stays the same for every scan
struct FeedDyn {
    long long scan;        // the scan's number
    const float* pts;      // registered source 2: the full scan, [n][3] (device)
    const float* inten;    // its intensity, [n] (device), or null (intensity 0)
    const int* n_dev;      // the count of pts when it is device resident (a depth image's filtered cloud), else null
    int n;                 // points of pts (the upper bound of *n_dev)
    int kind, branch;      // IMMESH_FEED_KIND_*, IMU branch (0: LiDAR-only)
    int src;               // registered source used: 0 none, 1 the down-sampled scan, 2 the full scan
    int lio;               // 1: the scan ran the IESKF (iterations, matches, rows); 0: an IMU branch 1 / 2 scan (header and state only)
    int pad_;
    const int* branch_dev; // the branch decided on the device (immesh_lio_step_async_depth_imu), or null: then `branch` is the branch, and
                           // a device branch other than 3 records the scan as lio = 0
};
// the points of the full scan (registered source 2)
IM_HD int feed_full_n(const FeedDyn& d) { return d.n_dev ? *d.n_dev : d.n; }
struct LioFeedDev {
    FeedDyn dyn;
    long long started;     // newest scan whose slot is being written (set before the slot's first byte changes)
    long long rows_total;  // rows placed since the enable: the cursor of the row ring
    long long eff_base, reg_base;   // the current scan's first effect / first registered row
    int lost, pad_;        // the current scan's rows are not written
};

// the plane-map markers' block (immesh_lio_feed_markers_enable).  started and rows_total lead, in the order of LioFeedDev's, so that
// the read takes both marks with one copy.
struct LioMarkDev {
    long long started;     // newest scan whose header slot is being written
    long long rows_total;  // rows placed since the enable: the cursor of the marker ring
    long long base;        // the current scan's first row
    int lost;              // the current scan's rows are not written (and nothing is consumed)
    int n;                 // roots the current scan walks: the pending count when its walk began
    int misc[5];           // the current walk's rows in all, then the reference's four counters
    int pad_[3];
};

// place a scan's ne effect and nr registered rows at the cursor, or lose them all when they exceed the ring; the header's row fields
IM_HD void feed_append(LioFeedDev& f, long long ne, long long nr, long long max_rows, long long* hdr) {
    const long long start = f.rows_total;
    const int lost = ne + nr > max_rows ? 1 : 0;
    f.lost = lost;
    f.eff_base = start;
    f.reg_base = start + (lost ? 0 : ne);
    if (!lost) f.rows_total = start + ne + nr;
    hdr[IMMESH_FEED_ROW_BEGIN] = start;
    hdr[IMMESH_FEED_ROW_EFFECT_END] = f.reg_base;
    hdr[IMMESH_FEED_ROW_END] = f.rows_total;
    hdr[IMMESH_FEED_ROWS_LOST] = lost;
}

// place a scan's `need` marker rows at the cursor, or lose them when they exceed the ring; the header's row fields
IM_HD void marker_append(LioMarkDev& m, long long need, long long max_rows, long long* hdr) {
    const int lost = need > max_rows ? 1 : 0;
    m.lost = lost;
    m.base = m.rows_total;
    hdr[IMMESH_MARKER_ROW_BEGIN] = m.rows_total;
    if (!lost) m.rows_total += need;
    hdr[IMMESH_MARKER_ROW_END] = m.rows_total;
    hdr[IMMESH_MARKER_ROWS_NEEDED] = need;
    hdr[IMMESH_MARKER_LOST] = lost;
}

// k_mark_head's work after it has marked the slot: the walk's rows placed (marker_append) or lost, the header written from the walk's
// totals in m (n, misc), and -- only when the rows fit -- the pending count *pub_n reset, so that k_pub_emit publishes and lists
// again just the roots that stay pending.  A lost scan leaves *pub_n and every flag as they are: nothing is consumed.  walk = 0: a
// record without a walk (no rows, nothing walked).  Returns 1 when k_pub_emit is to publish.
IM_HD int marker_header(LioMarkDev& m, long long scan, int walk, int* pub_n, long long max_rows, long long* h) {
    marker_append(m, walk ? m.misc[0] : 0, max_rows, h);
    h[IMMESH_MARKER_ROOTS_WALKED] = walk ? m.n : 0;
    for (int k = 0; k < 4; ++k) h[IMMESH_MARKER_PLANES + k] = walk ? m.misc[1 + k] : 0;
    h[IMMESH_MARKER_SCAN] = scan;
    const int commit = walk && !m.lost ? 1 : 0;
    if (commit) *pub_n = 0;
    return commit;
}

// What a read of the scans (since, fin] can return, from their copied headers `hdr` (oldest first) and the device marks read after
// the copy (`started`, `rows_total`): IMMESH_OK, or IMMESH_E_RANGE when a header slot or a row slot of the range may have been
// overwritten.  *rows: the rows the range holds.  hdr_len, row_begin, row_end: the header layout (the scan number is field 0).
IM_HD int feed_check_range(long long since, long long fin, long long max_scans, long long max_rows, const long long* hdr, long long started,
                              long long rows_total, long long* rows, int hdr_len = IMMESH_LIO_FEED_HDR, int row_begin = IMMESH_FEED_ROW_BEGIN,
                              int row_end = IMMESH_FEED_ROW_END) {
    static_assert(IMMESH_FEED_SCAN == 0 && IMMESH_MARKER_SCAN == 0, "the scan number leads every header");
    *rows = 0;
    const long long ns = fin - since;
    if (ns <= 0) return IMMESH_OK;
    if (ns > max_scans || started >= since + 1 + max_scans) return IMMESH_E_RANGE;
    for (long long i = 0; i < ns; ++i)
        if (hdr[i * hdr_len] != since + 1 + i) return IMMESH_E_RANGE;
    const long long r0 = hdr[row_begin], r1 = hdr[(ns - 1) * hdr_len + row_end];
    *rows = r1 - r0;
    if (r1 > r0 && rows_total - max_rows > r0) return IMMESH_E_RANGE;
    return IMMESH_OK;
}

// ---- the read of immesh_lio_feed, on the host.  The copies go through `copy(dst, src, bytes)`, which queues one contiguous copy and
// returns 0 or an IMMESH_E_* code; `marks(m)` finishes the copies queued before and reads the device marks m = (started, rows_total).
struct FeedRings {
    long long max_scans, max_rows;
    const long long* hdr;   // [max_scans][hdr_len]
    const double* states;   // [max_scans][state_doubles], or null (the marker records)
    const void* rows;       // [max_rows] rows of row_bytes
    const void* idx;        // [max_rows] second per-row array of idx_bytes per row, or null (effect off, the marker records)
    // the scan feed's header and rows unless set: the marker records' are IMMESH_LIO_FEED_MARKER_HDR and IMMESH_PLANE_MARKER_COLS doubles
    int hdr_len = IMMESH_LIO_FEED_HDR, row_begin = IMMESH_FEED_ROW_BEGIN, row_end = IMMESH_FEED_ROW_END;
    size_t row_bytes = 4 * sizeof(float);
    int state_doubles = IM_STATE_DOUBLES;
    size_t idx_bytes = sizeof(int);
    // the scan feed's row_index fix-up: the rows of each record from header field fill_col (idx set) or row_begin (idx null) to
    // row_end carry no index and read -1 (int32).  -1: no fix-up (the second array is copied as it is)
    int fill_col = IMMESH_FEED_ROW_EFFECT_END;
};
// the marker records' rings in the read's terms (immesh_lio_feed_markers)
inline FeedRings marker_rings(long long max_scans, long long max_rows, const long long* hdr, const double* ring) {
    FeedRings r{max_scans, max_rows, hdr, nullptr, ring, nullptr};
    r.hdr_len = IMMESH_LIO_FEED_MARKER_HDR;
    r.row_begin = IMMESH_MARKER_ROW_BEGIN;
    r.row_end = IMMESH_MARKER_ROW_END;
    r.row_bytes = IMMESH_PLANE_MARKER_COLS * sizeof(double);
    r.fill_col = -1;
    return r;
}
// entries [first, first + count) of a ring of `len` entries of `elem` bytes: the one or two contiguous copies
template <class Copy>
inline int feed_copy_ring(Copy& copy, void* dst, const void* ring, size_t elem, long long first, long long count, long long len) {
    const long long a = count < len - first ? count : len - first;
    int rc = copy(dst, (const char*)ring + (size_t)first * elem, (size_t)a * elem);
    if (rc == 0 && count > a) rc = copy((char*)dst + (size_t)a * elem, ring, (size_t)(count - a) * elem);
    return rc;
}
// The scans (since, fin] -- fin the newest finished scan -- into the caller's buffers, as immesh_lio_feed documents: counts[0..1] are
// set once the range is known; IMMESH_E_RANGE when a slot of the range may have been overwritten, before or during the copies;
// IMMESH_E_CAPACITY with the counts and nothing written; cap_scans = 0 a count query.
// The marker records (immesh_lio_feed_markers) are read by the same code with their layout in `r`, states and row_index null.
// The rings of any other layout are described by `r`: states the records of r.state_doubles, row_index the second per-row array.
template <class Copy, class Marks>
inline int feed_read(const FeedRings& r, long long since, long long fin, int64_t* scans, double* states, int cap_scans, void* rows, void* row_index,
                     int64_t cap_rows, int64_t* counts, Copy&& copy, Marks&& marks) {
    counts[0] = counts[1] = 0;
    if (since >= fin) return IMMESH_OK;
    const long long k0 = since + 1, ns = fin - since;
    if (ns > r.max_scans) return IMMESH_E_RANGE;
    std::vector<long long> hb((size_t)ns * r.hdr_len);
    long long m[2];
    int rc = feed_copy_ring(copy, hb.data(), r.hdr, r.hdr_len * sizeof(long long), (k0 - 1) % r.max_scans, ns, r.max_scans);
    if (rc == 0) rc = marks(m);
    if (rc) return rc;
    long long nrows = 0;
    auto check = [&] { return feed_check_range(since, fin, r.max_scans, r.max_rows, hb.data(), m[0], m[1], &nrows, r.hdr_len, r.row_begin, r.row_end); };
    if (check() != IMMESH_OK) return IMMESH_E_RANGE;
    counts[0] = ns;
    counts[1] = nrows;
    if (cap_scans == 0) return IMMESH_OK;   // a count query
    if (ns > cap_scans || (rows && nrows > cap_rows)) return IMMESH_E_CAPACITY;
    const long long r0 = hb[r.row_begin];
    if (states && r.states) rc = feed_copy_ring(copy, states, r.states, (size_t)r.state_doubles * sizeof(double), (k0 - 1) % r.max_scans, ns, r.max_scans);
    if (rc == 0 && rows && nrows > 0) {
        rc = feed_copy_ring(copy, rows, r.rows, r.row_bytes, r0 % r.max_rows, nrows, r.max_rows);
        if (rc == 0 && row_index && r.idx) rc = feed_copy_ring(copy, row_index, r.idx, r.idx_bytes, r0 % r.max_rows, nrows, r.max_rows);
    }
    if (rc == 0) rc = marks(m);   // the copies are done: nothing they read may have been overwritten meanwhile
    if (rc) return rc;
    if (check() != IMMESH_OK) return IMMESH_E_RANGE;
    std::memcpy(scans, hb.data(), hb.size() * sizeof(long long));
    if (rows && row_index && r.fill_col >= 0) {   // registered rows carry no scan index
        int32_t* ri = (int32_t*)row_index;
        for (long long i = 0; i < ns; ++i) {
            const long long* hd = hb.data() + (size_t)i * r.hdr_len;
            const long long a = r.idx ? hd[r.fill_col] : hd[r.row_begin];
            for (long long j = a; j < hd[r.row_end]; ++j) ri[j - r0] = -1;
        }
    }
    return IMMESH_OK;
}

}  // namespace immesh
