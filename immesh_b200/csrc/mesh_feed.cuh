// immesh_b200 -- the mesh frame feed (immesh_mesh_feed_enable / immesh_mesh_feed / immesh_mesh_feed_images): the device block its
// kernels share and the bookkeeping of its rings.  Header and pose ring: frame f (the handle's frame number) in slot (f - 1) % max_frames.
// Point ring: the reinforced points are numbered in the order the frames append them, row r in slot r % max_rows.  Image ring: image
// i in slot i % max_images, at most one per frame.  The slot and cursor arithmetic is __host__ __device__ and the read is feed_read
// (lio_feed.cuh), so that the host emulation (tests/mesh_feed/emu_mesh_feed.cpp) runs both as the product does.
//
// What the record kernels may point at (all of it is captured in the frame's graph): the feed's own rings, block and pinned done word,
// freed only by immesh_mesh_feed_enable and immesh_mesh_destroy after the stream is drained and the graph dropped; the reinforcement's
// and the view's result buffers, whose enable calls drop the graph too.  The image ring is sized for one view configuration, so that
// every immesh_mesh_view_enable frees it and turns the image recording off.  Every slot is 64-bit and checked against its ring.
#pragma once
#include <cstdint>

#include "../../include/immesh_b200.h"
#include "hd_math.cuh"
#include "lio_feed.cuh"

#if defined(__CUDA_ARCH__)
#define IM_MFEED_FENCE() __threadfence()
#else
#define IM_MFEED_FENCE()
#endif

namespace immesh {

// per-frame inputs of the feed's kernels (one H2D copy per frame from a pinned slot): the launch sequence stays the same for every frame
struct MeshFeedDyn {
    long long frame;      // the handle's frame number
    long long n;          // N_POINTS (-1: the FrameDyn's, a depth frame's count set on the device; k_mfeed_head fills it in)
    int step;             // STEP
    int kind;             // IMMESH_MFEED_KIND_*
    int has_rot;          // 1: handed over by a localization handle (the pose is in the camera ring)
    int rf, img;          // the reinforcement ran for the frame / its view image is recorded
    int pad_;
    double pose_t[3];     // the world-frame push's pose_t (has_rot = 0)
};
struct MeshFeedDev {
    MeshFeedDyn dyn;
    long long started;      // newest frame whose header slot is being written (set before the slot's first byte changes)
    long long rows_total;   // point rows placed since the enable: the cursor of the point ring
    long long imgs_total;   // images placed since the enable: the cursor of the image ring
    long long row_base;     // the current frame's first row
    long long img_slot;     // the current frame's image slot, or -1 (none)
    long long hdr_slot;     // the current frame's header slot, or -1 (refused: nothing of the frame is written)
    long long t_begin;      // %globaltimer at the frame's begin stamp
    int nrows;              // the current frame's rows to copy (0 when lost)
    int pad_;
};

// slot of entry idx of a ring of len entries, or -1 when no slot holds it (idx < 0 or an empty ring): the kernels refuse a slot
// outside [0, len) as an internal error (IM_MERR_FEED_INDEX) and write nothing, so that a bookkeeping bug fails a call, not the device
IM_HD long long mfeed_slot(long long idx, long long len) { return (idx < 0 || len < 1) ? -1 : idx % len; }
IM_HD bool mfeed_slot_ok(long long slot, long long len) { return slot >= 0 && slot < len; }

// The head of frame f.dyn.frame (k_mfeed_head, one thread): marks the slot, places the frame's nrf reinforced points (lost when they
// exceed the ring; none recorded with max_rows = 0) and its image at the cursors, and writes the header with the frame's eight counts
// (immesh_mesh_counts' order) and error flags.  Returns the header slot, or -1 when the slot is refused (nothing written, no cursor moved).
IM_HD long long mfeed_head(MeshFeedDev& f, const long long counts[8], long long err, long long nrf, long long max_frames, long long max_rows,
                           long long max_images, long long* hdr_ring) {
    const MeshFeedDyn& d = f.dyn;
    const long long slot = mfeed_slot(d.frame - 1, max_frames);
    f.hdr_slot = mfeed_slot_ok(slot, max_frames) ? slot : -1;
    f.nrows = 0;
    f.img_slot = -1;
    if (f.hdr_slot < 0) return -1;
    f.started = d.frame;   // before any byte of the slot changes (a reader checks it after its copy)
    IM_MFEED_FENCE();
    long long* h = hdr_ring + slot * IMMESH_MESH_FEED_HDR;
    const long long need = (d.rf && max_rows > 0) ? nrf : 0;
    const int lost = need > max_rows ? 1 : 0;
    f.row_base = f.rows_total;
    h[IMMESH_MFEED_ROW_BEGIN] = f.rows_total;
    if (!lost) { f.rows_total += need; f.nrows = (int)need; }
    h[IMMESH_MFEED_ROW_END] = f.rows_total;
    h[IMMESH_MFEED_ROWS_LOST] = lost;
    h[IMMESH_MFEED_IMG_BEGIN] = f.imgs_total;
    if (d.img && max_images > 0) {
        const long long is = mfeed_slot(f.imgs_total, max_images);
        if (mfeed_slot_ok(is, max_images)) { f.img_slot = is; ++f.imgs_total; }
    }
    h[IMMESH_MFEED_IMG_END] = f.imgs_total;
    h[IMMESH_MFEED_KIND] = d.kind;
    h[IMMESH_MFEED_N_POINTS] = d.n;
    h[IMMESH_MFEED_STEP] = d.step;
    for (int k = 0; k < 8; ++k) h[IMMESH_MFEED_COUNTS + k] = counts[k];
    h[IMMESH_MFEED_ERR] = err;
    h[IMMESH_MFEED_HAS_ROTATION] = d.has_rot;
    h[IMMESH_MFEED_T_BEGIN_NS] = f.t_begin;
    h[IMMESH_MFEED_T_END_NS] = f.t_begin;   // the done kernel stamps the end
    h[IMMESH_MFEED_RF] = d.rf ? 1 : 0;
    h[IMMESH_MFEED_FRAME] = d.frame;
    return slot;
}
// the ring slot of row i of the frame whose first row is row_base, or -1 (refused)
IM_HD long long mfeed_row_slot(long long row_base, long long i, long long max_rows) {
    const long long s = mfeed_slot(row_base + i, max_rows);
    return mfeed_slot_ok(s, max_rows) ? s : -1;
}

// the frame feed's rings in feed_read's terms: the headers with their poses, and the points (x y z floats) with their pixels
inline FeedRings mfeed_point_rings(long long max_frames, long long max_rows, const long long* hdr, const double* poses, const float* pts, const int* pix) {
    FeedRings r{max_frames, max_rows, hdr, poses, pts, pix};
    r.hdr_len = IMMESH_MESH_FEED_HDR;
    r.row_begin = IMMESH_MFEED_ROW_BEGIN;
    r.row_end = IMMESH_MFEED_ROW_END;
    r.row_bytes = 3 * sizeof(float);
    r.state_doubles = IMMESH_MESH_FEED_POSE;
    r.idx_bytes = sizeof(int);
    r.fill_col = -1;
    return r;
}
// ... and the images: one "row" of npx rgba pixels per image, the depth image (or null) as the second per-row array
inline FeedRings mfeed_image_rings(long long max_frames, long long max_images, long long npx, const long long* hdr, const void* rgba, const float* depth) {
    FeedRings r{max_frames, max_images, hdr, nullptr, rgba, depth};
    r.hdr_len = IMMESH_MESH_FEED_HDR;
    r.row_begin = IMMESH_MFEED_IMG_BEGIN;
    r.row_end = IMMESH_MFEED_IMG_END;
    r.row_bytes = (size_t)npx * 4;
    r.idx_bytes = (size_t)npx * sizeof(float);
    r.fill_col = -1;
    return r;
}

}  // namespace immesh
