// TEST INFRASTRUCTURE (not product code): the mesh frame feed's rings on the host.  A frame's device work is run in the device's order
// (mesh_capi.cu: k_mfeed_begin, then k_mfeed_head, k_mfeed_points, k_mfeed_image and k_mfeed_done) in two halves, so that a frame can be
// left in flight: emu_mfeed_head marks the slot, writes the header and places the points and the image with mfeed_head (mesh_feed.cuh),
// exactly as k_mfeed_head does; emu_mfeed_finish copies the points at mfeed_row_slot and the image at the image slot, refusing a slot
// outside its ring as the kernels do, and publishes the frame as finished.  The reads are feed_read itself on mfeed_point_rings /
// mfeed_image_rings, with memcpy for the device copies.  Contents encode (frame, row) so that a test can tell every row apart.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/mesh_core.cuh"
#include "../../immesh_b200/csrc/mesh_feed.cuh"

using namespace immesh;

namespace {
struct EmuMeshFeed {
    long long max_frames = 0, max_rows = 0, max_images = 0, npx = 0, queued = 0, done = 0;
    int depth = 0, err = 0;
    MeshFeedDev dev = {};
    std::vector<long long> hdr;
    std::vector<double> poses;
    std::vector<float> pts;        // [max_rows][3]
    std::vector<int> pix;          // [max_rows]
    std::vector<uint8_t> rgba;     // [max_images][npx][4]
    std::vector<float> dep;        // [max_images][npx]
    long long nrf = 0;             // the frame in flight's reinforced points (what the reinforcement produced)
} g;
}  // namespace

extern "C" {

// the enable with the handle at frame `frame_counter`: rings zeroed, the done word at the newest frame before the enable
void emu_mfeed_enable(long long max_frames, long long max_rows, long long max_images, long long npx, int depth, long long frame_counter) {
    g = EmuMeshFeed();
    g.max_frames = max_frames;
    g.max_rows = max_rows;
    g.max_images = max_images;
    g.npx = npx;
    g.depth = depth;
    g.queued = g.done = frame_counter;
    g.hdr.assign((size_t)max_frames * IMMESH_MESH_FEED_HDR, 0);
    g.poses.assign((size_t)max_frames * IMMESH_MESH_FEED_POSE, 0.0);
    g.pts.assign((size_t)max_rows * 3, 0.f);
    g.pix.assign((size_t)max_rows, 0);
    g.rgba.assign((size_t)(max_images * npx * 4), 0);
    g.dep.assign((size_t)(depth ? max_images * npx : 0), 0.f);
}

// k_mfeed_begin and k_mfeed_head of the next frame: kind, rf (the reinforcement ran, with nrf points), img (the view's image recorded).
// Returns the header slot, or -1 when refused (the error flag is then set).
long long emu_mfeed_head(int kind, int rf, long long nrf, int img) {
    const long long f = ++g.queued;
    MeshFeedDyn& d = g.dev.dyn;
    d = MeshFeedDyn{};
    d.frame = f;
    d.n = 100 * f;
    d.step = 1 + (int)(f % 3);
    d.kind = kind;
    d.has_rot = kind == IMMESH_MFEED_KIND_FROM_LIO_ASYNC ? 1 : 0;
    d.rf = rf;
    d.img = img;
    g.dev.t_begin = 1000 * f;
    const long long c[8] = {f, f + 1, f + 2, f + 3, f + 4, f + 5, f + 6, f + 7};
    const long long slot = mfeed_head(g.dev, c, 0, nrf, g.max_frames, g.max_rows, g.max_images, g.hdr.data());
    if (slot < 0) { g.err |= IM_MERR_FEED_INDEX; return -1; }
    for (int i = 0; i < IMMESH_MESH_FEED_POSE; ++i) g.poses[(size_t)slot * IMMESH_MESH_FEED_POSE + i] = (double)f * 100.0 + i;
    g.nrf = nrf;
    return slot;
}

// k_mfeed_points, k_mfeed_image and k_mfeed_done of the frame in flight
void emu_mfeed_finish() {
    const long long f = g.dev.dyn.frame;
    if (g.dev.hdr_slot >= 0) {
        for (long long i = 0; i < g.dev.nrows; ++i) {
            const long long s = mfeed_row_slot(g.dev.row_base, i, g.max_rows);
            if (s < 0) { g.err |= IM_MERR_FEED_INDEX; continue; }
            g.pts[(size_t)s * 3 + 0] = (float)f; g.pts[(size_t)s * 3 + 1] = (float)i; g.pts[(size_t)s * 3 + 2] = (float)(f + i);
            g.pix[(size_t)s] = (int)(f * 1000 + i);
        }
        const long long is = g.dev.img_slot;
        if (is >= 0 && !mfeed_slot_ok(is, g.max_images)) g.err |= IM_MERR_FEED_INDEX;
        else if (is >= 0) {
            for (long long p = 0; p < g.npx; ++p) {
                for (int k = 0; k < 4; ++k) g.rgba[(size_t)((is * g.npx + p) * 4 + k)] = (uint8_t)((f * 7 + p * 3 + k) & 255);
                if (g.depth) g.dep[(size_t)(is * g.npx + p)] = (float)f + 0.5f * (float)p;
            }
        }
        g.hdr[(size_t)g.dev.hdr_slot * IMMESH_MESH_FEED_HDR + IMMESH_MFEED_T_END_NS] = 1000 * f + 10;
    }
    g.done = f;
}

// a bookkeeping fault injected for the index guard: 0 the header ring empty (max_frames 0), 1 the point cursor negative, 2 the image
// ring shrunk below the cursor's slot
void emu_mfeed_corrupt(int which) {
    if (which == 0) g.max_frames = 0;
    if (which == 1) g.dev.rows_total = -7;
    if (which == 2) g.max_images = 0;
}
void emu_mfeed_restore(long long max_frames, long long max_images) { g.max_frames = max_frames; g.max_images = max_images; }
int emu_mfeed_err() { return g.err; }
long long emu_mfeed_queued() { return g.queued; }

int emu_mfeed_read(long long since, int64_t* frames, double* poses, int cap_frames, float* points, int32_t* pixels, int64_t cap_rows, int64_t* counts) {
    counts[0] = counts[1] = 0;
    counts[2] = g.done;
    counts[3] = g.queued;
    const FeedRings r = mfeed_point_rings(g.max_frames, g.max_rows, g.hdr.data(), g.poses.data(), g.pts.data(), g.pix.data());
    auto copy = [](void* dst, const void* src, size_t bytes) { std::memcpy(dst, src, bytes); return IMMESH_OK; };
    auto marks = [](long long* m) { m[0] = g.dev.started; m[1] = g.dev.rows_total; return IMMESH_OK; };
    return feed_read(r, since, g.done, frames, poses, cap_frames, points, pixels, cap_rows, counts, copy, marks);
}

int emu_mfeed_read_images(long long since, int64_t* frames, int cap_images, uint8_t* rgba, float* depth, int64_t* counts) {
    counts[0] = counts[1] = 0;
    counts[2] = g.done;
    counts[3] = g.queued;
    const FeedRings r = mfeed_image_rings(g.max_frames, g.max_images, g.npx, g.hdr.data(), g.rgba.data(), g.depth ? g.dep.data() : nullptr);
    auto copy = [](void* dst, const void* src, size_t bytes) { std::memcpy(dst, src, bytes); return IMMESH_OK; };
    auto marks = [](long long* m) { m[0] = g.dev.started; m[1] = g.dev.imgs_total; return IMMESH_OK; };
    return feed_read(r, since, g.done, frames, nullptr, cap_images, rgba, depth, cap_images, counts, copy, marks);
}

}  // extern "C"
