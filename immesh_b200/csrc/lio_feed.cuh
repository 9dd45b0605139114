// immesh_b200 -- the scan feed (immesh_lio_feed_enable / immesh_lio_feed): the device block its kernels share and the bookkeeping
// of its two rings.  Header and state ring: scan k (numbered 1, 2, ... from the enable) in slot (k - 1) % max_scans.  Row ring: the
// feed's rows are numbered in the order the scans append them, row r in slot r % max_rows; a scan's rows are its effect rows, then
// its registered rows.  The bookkeeping is __host__ __device__ and the read is host code, so that the host emulation
// (tests/lio_feed/emu_lio_feed.cpp) runs both as the product does.
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
    int n;                 // points of pts
    int kind, branch;      // IMMESH_FEED_KIND_*, IMU branch (0: LiDAR-only)
    int src;               // registered source used: 0 none, 1 the down-sampled scan, 2 the full scan
    int lio;               // 1: the scan ran the IESKF (iterations, matches, rows); 0: an IMU branch 1 / 2 scan (header and state only)
    int pad_;
};
struct LioFeedDev {
    FeedDyn dyn;
    long long started;     // newest scan whose slot is being written (set before the slot's first byte changes)
    long long rows_total;  // rows placed since the enable: the cursor of the row ring
    long long eff_base, reg_base;   // the current scan's first effect / first registered row
    int lost, pad_;        // the current scan's rows are not written
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

// What a read of the scans (since, fin] can return, from their copied headers `hdr` (oldest first) and the device marks read after
// the copy (`started`, `rows_total`): IMMESH_OK, or IMMESH_E_RANGE when a header slot or a row slot of the range may have been
// overwritten.  *rows: the rows the range holds.
IM_HD int feed_check_range(long long since, long long fin, long long max_scans, long long max_rows, const long long* hdr, long long started,
                              long long rows_total, long long* rows) {
    *rows = 0;
    const long long ns = fin - since;
    if (ns <= 0) return IMMESH_OK;
    if (ns > max_scans || started >= since + 1 + max_scans) return IMMESH_E_RANGE;
    for (long long i = 0; i < ns; ++i)
        if (hdr[i * IMMESH_LIO_FEED_HDR + IMMESH_FEED_SCAN] != since + 1 + i) return IMMESH_E_RANGE;
    const long long r0 = hdr[IMMESH_FEED_ROW_BEGIN], r1 = hdr[(ns - 1) * IMMESH_LIO_FEED_HDR + IMMESH_FEED_ROW_END];
    *rows = r1 - r0;
    if (r1 > r0 && rows_total - max_rows > r0) return IMMESH_E_RANGE;
    return IMMESH_OK;
}

// ---- the read of immesh_lio_feed, on the host.  The copies go through `copy(dst, src, bytes)`, which queues one contiguous copy and
// returns 0 or an IMMESH_E_* code; `marks(m)` finishes the copies queued before and reads the device marks m = (started, rows_total).
struct FeedRings {
    long long max_scans, max_rows;
    const long long* hdr;   // [max_scans][IMMESH_LIO_FEED_HDR]
    const double* states;   // [max_scans][IM_STATE_DOUBLES]
    const void* rows;       // [max_rows] float4
    const int* idx;         // [max_rows] or null (effect off)
};
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
template <class Copy, class Marks>
inline int feed_read(const FeedRings& r, long long since, long long fin, int64_t* scans, double* states, int cap_scans, float* rows, int32_t* row_index,
                     int64_t cap_rows, int64_t* counts, Copy&& copy, Marks&& marks) {
    counts[0] = counts[1] = 0;
    if (since >= fin) return IMMESH_OK;
    const long long k0 = since + 1, ns = fin - since;
    if (ns > r.max_scans) return IMMESH_E_RANGE;
    std::vector<long long> hb((size_t)ns * IMMESH_LIO_FEED_HDR);
    long long m[2];
    int rc = feed_copy_ring(copy, hb.data(), r.hdr, IMMESH_LIO_FEED_HDR * sizeof(long long), (k0 - 1) % r.max_scans, ns, r.max_scans);
    if (rc == 0) rc = marks(m);
    if (rc) return rc;
    long long nrows = 0;
    if (feed_check_range(since, fin, r.max_scans, r.max_rows, hb.data(), m[0], m[1], &nrows) != IMMESH_OK) return IMMESH_E_RANGE;
    counts[0] = ns;
    counts[1] = nrows;
    if (cap_scans == 0) return IMMESH_OK;   // a count query
    if (ns > cap_scans || (rows && nrows > cap_rows)) return IMMESH_E_CAPACITY;
    const long long r0 = hb[IMMESH_FEED_ROW_BEGIN];
    if (states) rc = feed_copy_ring(copy, states, r.states, IM_STATE_DOUBLES * sizeof(double), (k0 - 1) % r.max_scans, ns, r.max_scans);
    if (rc == 0 && rows && nrows > 0) {
        rc = feed_copy_ring(copy, rows, r.rows, 4 * sizeof(float), r0 % r.max_rows, nrows, r.max_rows);
        if (rc == 0 && row_index && r.idx) rc = feed_copy_ring(copy, row_index, r.idx, sizeof(int), r0 % r.max_rows, nrows, r.max_rows);
    }
    if (rc == 0) rc = marks(m);   // the copies are done: nothing they read may have been overwritten meanwhile
    if (rc) return rc;
    if (feed_check_range(since, fin, r.max_scans, r.max_rows, hb.data(), m[0], m[1], &nrows) != IMMESH_OK) return IMMESH_E_RANGE;
    std::memcpy(scans, hb.data(), hb.size() * sizeof(long long));
    if (rows && row_index) {   // registered rows carry no scan index
        for (long long i = 0; i < ns; ++i) {
            const long long* hd = hb.data() + (size_t)i * IMMESH_LIO_FEED_HDR;
            const long long a = r.idx ? hd[IMMESH_FEED_ROW_EFFECT_END] : hd[IMMESH_FEED_ROW_BEGIN];
            for (long long j = a; j < hd[IMMESH_FEED_ROW_END]; ++j) row_index[j - r0] = -1;
        }
    }
    return IMMESH_OK;
}

}  // namespace immesh
