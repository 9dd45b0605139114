// TEST INFRASTRUCTURE (not product code): the scan feed's rings on the host.  A scan's device work is run in the device's order
// (lio_capi.cu: k_feed_head, then k_eff_emit and k_reg_gather, then k_feed_done) in two halves, so that a scan can be left in flight:
// emu_feed_head marks the slot, copies the state and places the rows with feed_append (lio_feed.cuh), exactly as k_feed_head does;
// emu_feed_finish writes the rows at (base + j) % max_rows as the two emitters do, and publishes the scan as finished.  The read is
// feed_read itself (lio_feed.cuh), with memcpy for the device copies.  Row contents encode (scan, row of the scan) so that a test can
// tell every row apart.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/lio_feed.cuh"

using namespace immesh;

namespace {
struct EmuFeed {
    long long max_scans = 0, max_rows = 0, queued = 0, done = 0;
    int effect = 1;
    LioFeedDev dev = {};
    std::vector<long long> hdr;
    std::vector<double> states;
    std::vector<float> rows;   // [max_rows][4]
    std::vector<int> idx;
    long long ne = 0, nr = 0;  // the scan in flight
} g;
}  // namespace

extern "C" {

void emu_feed_enable(long long max_scans, long long max_rows, int effect) {
    g = EmuFeed();
    g.max_scans = max_scans;
    g.max_rows = max_rows;
    g.effect = effect;
    g.hdr.assign((size_t)max_scans * IMMESH_LIO_FEED_HDR, 0);
    g.states.assign((size_t)max_scans * IM_STATE_DOUBLES, 0.0);
    g.rows.assign((size_t)max_rows * 4, 0.f);
    g.idx.assign((size_t)max_rows, 0);
}

// k_feed_head of the next scan, with ne effect and nr registered rows
void emu_feed_head(long long ne, long long nr) {
    const long long k = ++g.queued;
    g.dev.dyn.scan = k;
    const long long slot = (k - 1) % g.max_scans;
    g.dev.started = k;
    for (int i = 0; i < IM_STATE_DOUBLES; ++i) g.states[(size_t)slot * IM_STATE_DOUBLES + i] = (double)k * 1000.0 + i;
    long long* h = g.hdr.data() + slot * IMMESH_LIO_FEED_HDR;
    feed_append(g.dev, ne, nr, g.max_rows, h);
    h[IMMESH_FEED_SCAN] = k;
    g.ne = ne;
    g.nr = nr;
}

// the emitters and k_feed_done of the scan in flight
void emu_feed_finish() {
    const long long k = g.dev.dyn.scan;
    if (!g.dev.lost) {
        for (long long j = 0; j < g.ne + g.nr; ++j) {
            const long long pos = ((j < g.ne ? g.dev.eff_base : g.dev.reg_base - g.ne) + j) % g.max_rows;
            float* r = g.rows.data() + pos * 4;
            r[0] = (float)k; r[1] = (float)j; r[2] = (float)(k + j); r[3] = j < g.ne ? 1.f : 2.f;
            if (j < g.ne) g.idx[(size_t)pos] = (int)(j * 3 + 1);
        }
    }
    g.done = k;
}

long long emu_feed_queued() { return g.queued; }

int emu_feed_read(long long since, int64_t* scans, double* states, int cap_scans, float* rows, int32_t* row_index, int64_t cap_rows, int64_t* counts) {
    counts[2] = g.done;
    counts[3] = g.queued;
    const FeedRings r{g.max_scans, g.max_rows, g.hdr.data(), g.states.data(), g.rows.data(), g.effect ? g.idx.data() : nullptr};
    auto copy = [](void* dst, const void* src, size_t bytes) { std::memcpy(dst, src, bytes); return IMMESH_OK; };
    auto marks = [](long long* m) { m[0] = g.dev.started; m[1] = g.dev.rows_total; return IMMESH_OK; };
    return feed_read(r, since, g.done, scans, states, cap_scans, rows, row_index, cap_rows, counts, copy, marks);
}

}  // extern "C"
