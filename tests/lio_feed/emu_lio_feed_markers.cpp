// TEST INFRASTRUCTURE (not product code): the scan feed's plane-map marker rings on the host.  A scan's device work is run in the
// device's order (lio_capi.cu: k_mark_head, then k_pub_emit, then k_feed_done) in two halves, so that a scan can be left in flight:
// emu_mark_head marks the slot and runs marker_header (lio_feed.cuh), as k_mark_head does; emu_mark_finish writes the rows through
// plane_pub_at (voxelmap.cuh) at the ring cursor when marker_header let the emit run, keeps pending what its pub_n still counts, and
// publishes the scan as finished.  So whether a lost scan consumes anything is decided by the product's marker_header.  The read is
// feed_read itself on marker_rings, as in immesh_lio_feed_markers, with memcpy for the device copies.  Pending rows stand for the
// map's pending flags: each carries the number of the row it was created as, so that a test can follow a row held back by a lost
// scan to the scan that publishes it.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/lio_feed.cuh"

using namespace immesh;

namespace {
struct EmuMarkers {
    long long max_scans = 0, max_rows = 0, queued = 0, done = 0, created = 0;
    LioMarkDev dev = {};
    long long scan = 0;                  // the scan in flight
    int pub_n = 0, commit = 0;           // its pending count after marker_header, and whether the emit runs
    std::vector<long long> hdr;
    std::vector<double> ring;            // [max_rows][IMMESH_PLANE_MARKER_COLS]
    std::vector<long long> pending;      // the pending rows, by creation number
} g;
}  // namespace

extern "C" {

void emu_mark_enable(long long max_scans, long long max_rows) {
    g = EmuMarkers();
    g.max_scans = max_scans;
    g.max_rows = max_rows;
    g.hdr.assign((size_t)max_scans * IMMESH_LIO_FEED_MARKER_HDR, 0);
    g.ring.assign((size_t)max_rows * IMMESH_PLANE_MARKER_COLS, 0.0);
}

// the map update of the next scan leaves `fresh` more rows pending; k_mark_head of that scan: the slot marked, then marker_header
// with the walk's totals (rows = roots walked = the pending rows, counters 0 1 2 3) and the pending count standing for pub_n
void emu_mark_head(long long fresh) {
    for (long long i = 0; i < fresh; ++i) g.pending.push_back(g.created++);
    const long long k = ++g.queued;
    g.scan = k;
    g.dev.started = k;
    g.dev.n = (int)g.pending.size();
    g.dev.misc[0] = (int)g.pending.size();
    for (int c = 0; c < 4; ++c) g.dev.misc[1 + c] = c;
    g.pub_n = (int)g.pending.size();
    g.commit = marker_header(g.dev, k, 1, &g.pub_n, g.max_rows, g.hdr.data() + (k - 1) % g.max_scans * IMMESH_LIO_FEED_MARKER_HDR);
}

// k_pub_emit and k_feed_done of the scan in flight: the rows at the cursor when marker_header let the emit run; the pending rows
// are those pub_n still lists (all of them after a lost scan, none after a published one: no root is held back here)
void emu_mark_finish() {
    if (g.commit) {
        for (size_t j = 0; j < g.pending.size(); ++j) {
            double* r = plane_pub_at(g.ring.data(), g.dev.base, (int)j, g.max_rows);
            for (int c = 0; c < IMMESH_PLANE_MARKER_COLS; ++c) r[c] = (double)(g.pending[j] * 100 + c);
        }
    }
    g.pending.resize((size_t)g.pub_n);
    g.done = g.scan;
}

// a blocking immesh_voxelmap_plane_markers between scans: it consumes every pending row, outside the rings
void emu_mark_consume() { g.pending.clear(); }

int emu_mark_read(long long since, int64_t* scans, int cap_scans, double* rows, int64_t cap_rows, int64_t* counts) {
    counts[2] = g.done;
    counts[3] = g.queued;
    const FeedRings r = marker_rings(g.max_scans, g.max_rows, g.hdr.data(), g.ring.data());
    auto copy = [](void* dst, const void* src, size_t bytes) { std::memcpy(dst, src, bytes); return IMMESH_OK; };
    auto marks = [](long long* m) { m[0] = g.dev.started; m[1] = g.dev.rows_total; return IMMESH_OK; };
    return feed_read(r, since, g.done, scans, nullptr, cap_scans, rows, nullptr, cap_rows, counts, copy, marks);
}

}  // extern "C"
