// immesh_b200 -- the mesher's two feeds: the change feed (immesh_mesh_changes_enable, mesh_changes.cuh) and the frame feed
// (immesh_mesh_feed_enable, mesh_feed.cuh).  CUDA kernels (sm_90a) queued behind each frame, and the C-ABI enables and reads.
#include <cstddef>

#include "block_scan.cuh"
#include "handles.hpp"
#include "pdl.cuh"

using namespace immesh;

// ---- the change feed (mesh_changes.cuh), queued after the push when enabled.  full: the frame lists its slots by the sweep (batched)
__global__ void __launch_bounds__(128) k_chg_gather(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = chg_gather_count(M, F);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) chg_gather(M, F, e);
}
__global__ void __launch_bounds__(128) k_chg_sweep(MeshDev M, FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    if (!chg_sweeping(F, full)) return;
    const int n = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) chg_sweep_slot(M, F, C, t);
}
__global__ void __launch_bounds__(128) k_chg_mark(MeshDev M, FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(chg_listed(F, full), F.chg_cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) chg_row_mark(M, F, C, i);
}
__global__ void __launch_bounds__(1024) k_chg_rows(FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(chg_listed(F, full), F.chg_cap);
    const int total = chunk_scan_1024(n, [&](int i) { return chg_row_count(C, i); }, [&](int i, int run) { return chg_row_emit(C, i, run); });
    if (threadIdx.x == 1023) F.chg_cnt[IM_CH_ROWS] = total;
}
__global__ void __launch_bounds__(128) k_chg_word(const int* cnt, ChgDev C, int w, const unsigned int* vin, unsigned int* kout, unsigned int* vout) {
    const int n = cnt[IM_CH_ROWS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vin ? vin[i] : (unsigned int)i;
        kout[i] = chg_word(C, w, (int)v);
        vout[i] = v;
    }
}
__global__ void __launch_bounds__(128) k_chg_emit(FrameBuf F_, ChgDev C, const unsigned int* order, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    if (chg_lost(F, C, full)) return;
    const int n = F.chg_cnt[IM_CH_ROWS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) chg_append(C, order, i);
}
__global__ void k_chg_end(MeshDev M, FrameBuf F_, ChgDev C, int full, int v_after) { chg_frame_end(M, frame_load_dyn(F_), C, full, v_after); }
// enable: the published bytes of the allocated slots from the store as it is
__global__ void __launch_bounds__(128) k_chg_init(MeshDev M, unsigned char* pub, int n_alloc) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) pub[t] = chg_state(M, t);
}

// ---- the frame feed (immesh_mesh_feed_enable, mesh_feed.cuh).  k_mfeed_begin stamps the start of the frame's launch sequence; behind
// the frame's last kernel (k_frame_end / k_chg_end, the reinforcement, the view) k_mfeed_head writes the header, the poses and the
// cursors (mfeed_head), k_mfeed_points and k_mfeed_image copy the reinforced points and the view image into their rings at the cursors,
// and k_mfeed_done stamps the end and publishes the frame's number to the host word the reader polls.  Fixed grids: every count is
// read on the device.  A slot outside its ring sets IM_MERR_FEED_INDEX and nothing is written.
extern "C" {   // profiles and tools name these kernels without a signature
__device__ __forceinline__ long long mfeed_clock() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__global__ void k_mfeed_begin(MeshFeedDev* fd) {
    pdl_wait();
    if (threadIdx.x == 0) fd->t_begin = mfeed_clock();
}
#define MFEED_THREADS 64
#define MFEED_COPY_THREADS 256
static_assert(IMMESH_MESH_FEED_POSE <= MFEED_THREADS, "one thread per pose value");
__global__ void __launch_bounds__(MFEED_THREADS) k_mfeed_head(MeshFeedDev* fd, int* cnt, long long* hdr, double* poses, long long max_frames, long long max_rows,
                                                              long long max_images, const double (*cam_ring)[12], RfOut rf0, RfOut rf1, const double* vw_pose0,
                                                              const double* vw_pose1, const FrameDyn* dyn) {
    pdl_wait();
    __shared__ long long s_slot, s_img;
    const long long frame = fd->dyn.frame;
    const int b = (int)(frame & 1);
    if (threadIdx.x == 0) {
        if (fd->dyn.n < 0) { fd->dyn.n = dyn->n; fd->dyn.step = dyn->step; }   // a depth frame: counted on the device
        const long long c[8] = {cnt[IM_MC_VERTICES], cnt[IM_MC_TRIS_LIVE], cnt[IM_MC_NEW_VERTICES], (long long)cnt[IM_MC_WORK_FRONT] + cnt[IM_MC_WORK_BACK],
                                cnt[IM_MC_ADD], cnt[IM_MC_REMOVE], cnt[IM_MC_VOXELS], cnt[IM_MC_ACT]};
        const int* nrf = b ? rf1.n : rf0.n;
        const long long slot = mfeed_head(*fd, c, cnt[IM_MC_ERR], (fd->dyn.rf && nrf) ? *nrf : 0, max_frames, max_rows, max_images, hdr);
        if (slot < 0) im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX);
        s_slot = slot;
        s_img = fd->img_slot;
    }
    __syncthreads();
    const long long slot = s_slot;
    if (slot < 0 || threadIdx.x >= IMMESH_MESH_FEED_POSE) return;
    // the frame pose, the reinforcement camera, the view camera: 12 doubles each (row-major R, then t)
    const int i = threadIdx.x, part = i / 12, k = i % 12;
    double v = 0.0;
    if (part == 0) {
        if (fd->dyn.has_rot) v = cam_ring[frame % IM_RF_RING][k];
        else if (k >= 9) v = fd->dyn.pose_t[k - 9];
    } else if (part == 1) {
        const double* p = b ? rf1.pose : rf0.pose;
        if (fd->dyn.rf && p) v = p[k];
    } else {
        const double* p = b ? vw_pose1 : vw_pose0;
        if (s_img >= 0 && p) v = p[k];
    }
    poses[slot * IMMESH_MESH_FEED_POSE + i] = v;
}
__global__ void __launch_bounds__(MFEED_COPY_THREADS) k_mfeed_points(const MeshFeedDev* fd, int* cnt, RfOut rf0, RfOut rf1, float* pts, int* pix, long long max_rows) {
    pdl_wait();
    const long long n = fd->nrows, base = fd->row_base;
    if (fd->hdr_slot < 0 || n <= 0) return;
    const RfOut o = (fd->dyn.frame & 1) ? rf1 : rf0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long s = mfeed_row_slot(base, i, max_rows);
        if (s < 0) { im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX); continue; }
        pts[s * 3 + 0] = o.pts[i * 3 + 0];
        pts[s * 3 + 1] = o.pts[i * 3 + 1];
        pts[s * 3 + 2] = o.pts[i * 3 + 2];
        pix[s] = o.pix[i];
    }
}
__global__ void __launch_bounds__(MFEED_COPY_THREADS) k_mfeed_image(const MeshFeedDev* fd, int* cnt, const uchar4* rgba0, const uchar4* rgba1, const float* depth0,
                                                                    const float* depth1, uchar4* ring, float* depth_ring, long long npx, long long max_images) {
    pdl_wait();
    const long long s = fd->img_slot;
    if (s < 0) return;   // no image for this frame
    if (!mfeed_slot_ok(s, max_images)) {
        if (blockIdx.x == 0 && threadIdx.x == 0) im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX);
        return;
    }
    const int b = (int)(fd->dyn.frame & 1);
    const uchar4* src = b ? rgba1 : rgba0;
    const float* dsrc = b ? depth1 : depth0;
    uchar4* dst = ring + s * npx;
    float* ddst = depth_ring ? depth_ring + s * npx : nullptr;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
        dst[i] = src[i];
        if (ddst) ddst[i] = dsrc[i];
    }
}
__global__ void k_mfeed_done(const MeshFeedDev* fd, long long* hdr, long long* done) {
    pdl_wait();
    if (threadIdx.x == 0) {
        const long long slot = fd->hdr_slot;   // checked by k_mfeed_head (-1: refused)
        if (slot >= 0) hdr[slot * IMMESH_MESH_FEED_HDR + IMMESH_MFEED_T_END_NS] = mfeed_clock();
        __threadfence_system();
        *(volatile long long*)done = fd->dyn.frame;
    }
}
}  // extern "C"
// the first kernel of a recorded frame's launch sequence
void mesh_feed_begin_launch(immesh_mesh* h, cudaStream_t st) { IM_LAUNCH(k_mfeed_begin, 1, 32, 0, st, h->feed.dev); }
// the frame's feed inputs, from pinned slot s (released with the frame that last used it), ahead of its kernels in stream order
int mesh_feed_stage(immesh_mesh* h, int s, long long frame, long long n, int step, int kind, const double* pose_t, bool rf, bool img) {
    auto& f = h->feed;
    MeshFeedDyn& d = f.h_dyn[s];
    d.frame = frame;
    d.n = n;
    d.step = step;
    d.kind = kind;
    d.has_rot = pose_t ? 0 : 1;
    d.rf = rf ? 1 : 0;
    d.img = img ? 1 : 0;
    d.pad_ = 0;
    for (int j = 0; j < 3; ++j) d.pose_t[j] = pose_t ? pose_t[j] : 0.0;
    IM_CUDA(cudaMemcpyAsync(&f.dev->dyn, &d, sizeof(MeshFeedDyn), cudaMemcpyHostToDevice, h->stream));
    return IMMESH_OK;
}
// the record behind the frame's last kernel; rf / img: the frame ran the reinforcement / its image is recorded (grids fixed)
void mesh_feed_launch(immesh_mesh* h, cudaStream_t st, bool rf, bool img) {
    auto& f = h->feed;
    const RfOut none = {};
    const RfOut r0 = rf ? h->rf.img.out[0] : none, r1 = rf ? h->rf.img.out[1] : none;
    IM_LAUNCH(k_mfeed_head, 1, MFEED_THREADS, 0, st, f.dev, h->M.cnt, f.hdr, f.poses, f.max_frames, f.max_rows, f.max_images, (const double (*)[12])h->cam_ring, r0, r1,
              img ? (const double*)h->vw.img.out[0].pose : (const double*)nullptr, img ? (const double*)h->vw.img.out[1].pose : (const double*)nullptr,
              (const FrameDyn*)h->d_dyn);
    if (rf && f.max_rows > 0)
        IM_LAUNCH(k_mfeed_points, h->n_sm * 2, MFEED_COPY_THREADS, 0, st, (const MeshFeedDev*)f.dev, h->M.cnt, r0, r1, f.pts, f.pix, f.max_rows);
    if (img)
        IM_LAUNCH(k_mfeed_image, h->n_sm * 4, MFEED_COPY_THREADS, 0, st, (const MeshFeedDev*)f.dev, h->M.cnt, (const uchar4*)h->vw.rgba[0], (const uchar4*)h->vw.rgba[1],
                  (const float*)h->vw.img.out[0].depth, (const float*)h->vw.img.out[1].depth, f.rgba, f.depth_ring, f.npx, f.max_images);
    IM_LAUNCH(k_mfeed_done, 1, 32, 0, st, (const MeshFeedDev*)f.dev, f.hdr, f.d_done);
}
cudaError_t mesh_feed_commit(immesh_mesh* h, long long frame) {
    h->feed.queued = frame;
    return cudaEventRecord(h->feed.ev, h->stream);
}
// drops the feed's buffers, stream and event; the caller has drained the stream and dropped the graph
void mesh_feed_free(immesh_mesh* h) {
    auto& f = h->feed;
    if (f.ev) cudaEventDestroy(f.ev);
    if (f.stream) cudaStreamDestroy(f.stream);
    h->feed = immesh_mesh::Feed();
}

// the change feed of the frame whose push was just queued (F: its FrameBuf; batched: a batched frame, after k_bat_frame_end): the
// touched set (the sweep when batched or overflowed), the rows against the published bytes (marked per slot, then compacted), their LSD sort by (a, b, c) over words
// of the bits of max_v - 1, the ring append and the header.  Fixed grids: every count is read on the device.
void mesh_changes_launch(immesh_mesh* h, const FrameBuf& F, cudaStream_t st, bool batched) {
    auto& c = h->chg;
    const int full = batched ? 1 : 0, cap = F.chg_cap;
    if (!batched) IM_LAUNCH(k_chg_gather, h->n_sm * 2, 128, 0, st, h->M, F);
    IM_LAUNCH(k_chg_sweep, h->n_sm * 8, 128, 0, st, h->M, F, c.C, full);
    unsigned int* ku[2] = {c.ku, c.ku + cap};
    unsigned int* vu[2] = {c.vu, c.vu + cap};
    const int g = mesh_grid_fixed(h, cap, 128), passes = rb_passes((unsigned long long)std::max(h->M.max_v - 1, 0));
    IM_LAUNCH(k_chg_mark, g, 128, 0, st, h->M, F, c.C, full);
    IM_LAUNCH(k_chg_rows, 1, 1024, 0, st, F, c.C, full);
    int cur = 0;
    for (int w = 0; w < 3; ++w) {
        IM_LAUNCH(k_chg_word, g, 128, 0, st, (const int*)F.chg_cnt, c.C, w, w == 0 ? (const unsigned int*)nullptr : (const unsigned int*)vu[cur], ku[cur ^ 1], vu[cur ^ 1]);
        cur = mesh_sort_passes(st, ku, vu, cur ^ 1, cap, passes, c.hist, F.chg_cnt + IM_CH_ROWS);
    }
    IM_LAUNCH(k_chg_emit, g, 128, 0, st, F, c.C, (const unsigned int*)vu[cur], full);
    IM_LAUNCH(k_chg_end, 1, 1, 0, st, h->M, F, c.C, full, full);
}

int immesh_mesh_changes_enable(immesh_mesh_t* h, int64_t max_rows, int max_frames) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (max_rows < 0 || max_rows > IM_MPOOL_LIMIT || (max_rows > 0 && (max_frames < 1 || max_frames > (1 << 20))))
        return im_fail(IMMESH_E_INVALID, "changes_enable: bad argument (0 <= max_rows <= 2^30; 1 <= max_frames <= 2^20 when max_rows > 0)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "changes_enable: a sharded mesh handle is not supported");
    IM_CUDA(im_stage_reset(h, [h] {
        h->chg = immesh_mesh::Changes();
        h->F.chg_stamp = nullptr; h->F.chg_list = nullptr; h->F.chg_cnt = nullptr; h->F.chg_cap = 0;
    }));
    if (max_rows == 0) return IMMESH_OK;
    immesh_mesh::Changes c;   // built in full before it replaces h->chg: after a failure the feed stays disabled
    ChgDev& C = c.C;
    C.max_rows = max_rows;
    C.max_frames = max_frames;
    const int cap = (int)std::min<int64_t>(max_rows, 1 << 21), max_t = h->M.max_t;   // a frame's touched slots: a bounded list
    int *stamp = nullptr, *list = nullptr, *cnt = nullptr;
    cudaError_t e = c.dev.alloc(&stamp, (size_t)max_t, 0xFF);
    auto add = [&e, &c](auto** p, size_t count, int fill = -1) { if (e == cudaSuccess) e = c.dev.alloc(p, std::max<size_t>(count, 1), fill); };
    add(&C.pub, (size_t)max_t, 0); add(&list, (size_t)cap); add(&cnt, IM_CH_SIZE, 0); add(&C.marked, (size_t)cap); add(&C.rowbuf, (size_t)cap);
    add(&c.ku, 2 * (size_t)cap); add(&c.vu, 2 * (size_t)cap); add(&c.hist, mesh_sort_hist_ints((size_t)cap));
    add(&C.hdr, (size_t)max_frames, 0xFF); add(&C.ring, (size_t)max_rows); add(&C.written, 1, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();   // the initialising memsets ran on the legacy stream
    int cnt_host[IM_MC_HOST];
    if (e == cudaSuccess) e = mesh_read_counters(h, cnt_host);
    if (e == cudaSuccess) {
        const int nalloc = std::min(cnt_host[IM_MC_TRIS_ALLOC], max_t);
        if (nalloc > 0) IM_LAUNCH(k_chg_init, mesh_grid(h, nalloc, 128), 128, 0, h->stream, h->M, C.pub, nalloc);
        if ((e = cudaGetLastError()) == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    }
    if (e != cudaSuccess) return im_fail_alloc(e, "changes_enable: allocation of the change feed's buffers failed");
    c.on = 1;
    c.enable_frame = c.last_frame = h->frame_counter;
    h->chg = std::move(c);
    h->F.chg_stamp = stamp; h->F.chg_list = list; h->F.chg_cnt = cnt; h->F.chg_cap = cap;
    return IMMESH_OK;
}
int immesh_mesh_changes(immesh_mesh_t* h, int64_t since_frame, int64_t* frames, int cap_frames, int32_t* rows, int64_t cap_rows, float* vertices,
                        int64_t cap_vertices, int64_t* counts) {
    if (!h || !counts || cap_frames < 0 || cap_rows < 0 || cap_vertices < 0 || (cap_frames > 0 && !frames) || (cap_rows > 0 && !rows) || (cap_vertices > 0 && !vertices))
        return im_fail(IMMESH_E_INVALID, "changes: bad argument");
    for (int i = 0; i < 4; ++i) counts[i] = 0;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "changes: a sharded mesh handle is not supported");
    const auto& c = h->chg;
    if (!c.on) return im_fail(IMMESH_E_INVALID, "changes: the change feed is not enabled (immesh_mesh_changes_enable)");
    const int64_t newest = c.last_frame, nf = newest - since_frame;
    counts[3] = newest;
    if (since_frame > newest) return im_fail(IMMESH_E_INVALID, "changes: since_frame is newer than the newest queued frame");
    if (since_frame < c.enable_frame) return im_fail(IMMESH_E_RANGE, "changes: since_frame is older than the enable (resync: snapshot, then read from the newest frame)");
    if (nf > c.C.max_frames) return im_fail(IMMESH_E_RANGE, "changes: the frames after since_frame are no longer held (max_frames; resync: snapshot, then read from the newest frame)");
    if (nf == 0) return IMMESH_OK;
    IM_CUDA(cudaEventSynchronize(h->ev_done[newest & (IM_SLOTS - 1)]));   // the newest frame only (a batched frame has finished already)
    std::vector<ChgHdr> hdr((size_t)c.C.max_frames);
    long long written = 0;
    IM_CUDA(cudaMemcpy(hdr.data(), c.C.hdr, hdr.size() * sizeof(ChgHdr), cudaMemcpyDeviceToHost));
    IM_CUDA(cudaMemcpy(&written, c.C.written, sizeof(written), cudaMemcpyDeviceToHost));
    for (int64_t f = since_frame + 1; f <= newest; ++f) {
        const ChgHdr& r = hdr[(size_t)(f % c.C.max_frames)];
        if (r.frame != f || r.lost || r.r_begin < written - c.C.max_rows)
            return im_fail(IMMESH_E_RANGE, ("changes: the rows of frame " + std::to_string(f) + " are not held (" + (r.frame != f ? "not recorded" : r.lost ? "lost to the feed's per-frame list or ring" : "ring wrapped") +
                                            "; resync: snapshot, then read from the newest frame)").c_str());
    }
    const ChgHdr& first = hdr[(size_t)((since_frame + 1) % c.C.max_frames)];
    const ChgHdr& last = hdr[(size_t)(newest % c.C.max_frames)];
    const int64_t nrows = last.r_end - first.r_begin, nverts = last.v_end - first.v_begin;
    counts[0] = nf; counts[1] = nrows; counts[2] = nverts;
    if (nf > cap_frames || nrows > cap_rows || nverts > cap_vertices)
        return im_fail(IMMESH_E_CAPACITY, "changes: a buffer is smaller than the counts (counts holds them; nothing was written)");
    for (int64_t f = since_frame + 1, k = 0; f <= newest; ++f, ++k) {
        const ChgHdr& r = hdr[(size_t)(f % c.C.max_frames)];
        frames[k * 4 + 0] = f; frames[k * 4 + 1] = r.v_begin; frames[k * 4 + 2] = r.v_end; frames[k * 4 + 3] = r.r_end - first.r_begin;
    }
    for (int64_t g = first.r_begin; g < last.r_end;) {   // the ring range, in at most two pieces
        const int64_t pos = g % c.C.max_rows, len = std::min(last.r_end - g, c.C.max_rows - pos);
        IM_CUDA(cudaMemcpy(rows + (g - first.r_begin) * 4, c.C.ring + pos, (size_t)len * sizeof(int4), cudaMemcpyDeviceToHost));
        g += len;
    }
    if (nverts > 0) {   // a vertex never moves after its append: the positions are read now
        std::vector<float4> v((size_t)nverts);
        IM_CUDA(cudaMemcpy(v.data(), h->M.vpos + first.v_begin, (size_t)nverts * sizeof(float4), cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < nverts; ++i) { vertices[i * 3] = v[i].x; vertices[i * 3 + 1] = v[i].y; vertices[i * 3 + 2] = v[i].z; }
    }
    return IMMESH_OK;
}

int immesh_mesh_feed_enable(immesh_mesh_t* h, const immesh_mesh_feed_config* c) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (c && (c->max_frames < 1 || c->max_frames > (1LL << 20) || c->max_rows < 0 || c->max_rows > (1LL << 32) || c->max_images < 0 || c->max_images > (1LL << 16) ||
              (c->depth != 0 && c->depth != 1) || (c->depth && c->max_images == 0)))
        return im_fail(IMMESH_E_INVALID, "feed_enable: bad argument (max_frames in [1, 2^20], max_rows in [0, 2^32], max_images in [0, 2^16], depth 0 or 1 and 1 only with images)");
    if (c && c->max_images > 0 && !h->vw.on) return im_fail(IMMESH_E_INVALID, "feed_enable: images need the queued view (immesh_mesh_view_enable first)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "feed_enable: a sharded mesh handle is not supported (the frame feed runs on a single GPU)");
    IM_CUDA(im_stage_reset(h, [h] { mesh_feed_free(h); }));   // frames in flight write the rings and the done word
    if (!c) return IMMESH_OK;
    auto& f = h->feed;
    f.max_frames = c->max_frames;
    f.max_rows = c->max_rows;
    f.max_images = c->max_images;
    f.depth = c->depth;
    f.npx = c->max_images > 0 ? (long long)h->vw.base.w * h->vw.base.h : 0;   // the view as it is configured now
    auto fail = [&](cudaError_t e) {
        mesh_feed_free(h);
        return im_fail_alloc(e, "feed_enable: allocation of the frame feed's buffers failed");
    };
    cudaError_t e;
    if ((e = f.dev_mem.alloc(&f.dev, 1, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.hdr, (size_t)f.max_frames * IMMESH_MESH_FEED_HDR, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.poses, (size_t)f.max_frames * IMMESH_MESH_FEED_POSE, 0)) != cudaSuccess) return fail(e);
    if (f.max_rows > 0) {
        if ((e = f.dev_mem.alloc(&f.pts, (size_t)f.max_rows * 3)) != cudaSuccess) return fail(e);
        if ((e = f.dev_mem.alloc(&f.pix, (size_t)f.max_rows)) != cudaSuccess) return fail(e);
    }
    if (f.max_images > 0) {
        if ((e = f.img_mem.alloc(&f.rgba, (size_t)f.max_images * (size_t)f.npx)) != cudaSuccess) return fail(e);
        if (f.depth && (e = f.img_mem.alloc(&f.depth_ring, (size_t)f.max_images * (size_t)f.npx)) != cudaSuccess) return fail(e);
    }
    if ((e = f.pinned.alloc(&f.h_dyn, IM_SLOTS, 0)) != cudaSuccess) return fail(e);
    if ((e = f.pinned.alloc(&f.h_done, 1)) != cudaSuccess) return fail(e);
    *f.h_done = h->frame_counter;
    if ((e = cudaHostGetDevicePointer((void**)&f.d_done, f.h_done, 0)) != cudaSuccess) return fail(e);
    if ((e = cudaStreamCreateWithFlags(&f.stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e);
    if ((e = cudaEventCreateWithFlags(&f.ev, cudaEventDisableTiming)) != cudaSuccess) return fail(e);
    if ((e = cudaEventRecord(f.ev, h->stream)) != cudaSuccess) return fail(e);
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return fail(e);   // the initialising memsets ran on the legacy stream
    f.enable_frame = f.queued = h->frame_counter;
    f.on = 1;
    return IMMESH_OK;
}
// the marks a read checks after its copies: the newest frame whose slot is being written and the cursor of the ring read (points or images)
static int mesh_feed_marks(immesh_mesh* h, bool images, long long* m) {
    auto& f = h->feed;
    long long b[3];
    IM_CUDA(cudaMemcpyAsync(b, &f.dev->started, sizeof(b), cudaMemcpyDeviceToHost, f.stream));
    IM_CUDA(cudaStreamSynchronize(f.stream));
    static_assert(offsetof(MeshFeedDev, rows_total) == offsetof(MeshFeedDev, started) + 8 && offsetof(MeshFeedDev, imgs_total) == offsetof(MeshFeedDev, started) + 16,
                  "the marks are read with one copy");
    m[0] = b[0];
    m[1] = images ? b[2] : b[1];
    return IMMESH_OK;
}
// the two reads: arguments, the wait, counts[2..3], then feed_read of `rings` with its copies on the feed's stream (never the handle's)
static int mesh_feed_read(immesh_mesh* h, const char* what, bool images, const FeedRings& rings, int64_t since, int wait, int64_t* frames, double* poses,
                          int cap_frames, void* rows, void* second, int64_t cap_rows, int64_t* counts) {
    auto& f = h->feed;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": a sharded mesh handle is not supported").c_str());
    if (!f.on) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": the frame feed is not enabled (immesh_mesh_feed_enable)").c_str());
    if (since > f.queued) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": since_frame is newer than the newest queued frame").c_str());
    if (wait) IM_CUDA(cudaEventSynchronize(f.ev));   // the newest queued frame's record, nothing else
    const long long fin = *(volatile long long*)f.h_done;
    counts[2] = fin;
    counts[3] = f.queued;
    auto copy = [&f](void* dst, const void* src, size_t bytes) {
        IM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, f.stream));
        return IMMESH_OK;
    };
    auto marks = [&](long long* m) { return mesh_feed_marks(h, images, m); };
    const int rc = feed_read(rings, since, fin, frames, poses, cap_frames, rows, second, cap_rows, counts, copy, marks);
    if (rc == IMMESH_E_RANGE)
        return im_fail(rc, (std::string(what) + ": frames of the range predate the enable, left the rings or were overwritten while they were read; read on from counts[2]").c_str());
    if (rc == IMMESH_E_CAPACITY) return im_fail(rc, (std::string(what) + ": more frames or rows than the caps (counts holds them; nothing was written)").c_str());
    return rc;
}
int immesh_mesh_feed(immesh_mesh_t* h, int64_t since, int wait, int64_t* frames, double* poses, int cap_frames, float* points, int32_t* pixels, int64_t cap_rows,
                     int64_t* counts) {
    if (counts) for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (!h || !counts || since < 0 || cap_frames < 0 || cap_rows < 0 || (cap_frames > 0 && !frames)) return im_fail(IMMESH_E_INVALID, "feed: bad argument");
    auto& f = h->feed;
    const FeedRings rings = mfeed_point_rings(f.max_frames, f.max_rows, f.hdr, f.poses, f.pts, f.pix);
    return mesh_feed_read(h, "feed", false, rings, since, wait, frames, poses, cap_frames, points, pixels, cap_rows, counts);
}
int immesh_mesh_feed_images(immesh_mesh_t* h, int64_t since, int wait, int64_t* frames, int cap_images, uint8_t* rgba, float* depth, int64_t* counts) {
    if (counts) for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (!h || !counts || since < 0 || cap_images < 0 || (cap_images > 0 && !frames)) return im_fail(IMMESH_E_INVALID, "feed_images: bad argument");
    auto& f = h->feed;
    if (f.on && f.max_images == 0)
        return im_fail(IMMESH_E_INVALID, "feed_images: image recording is off (max_images = 0, or immesh_mesh_view_enable was called after the enable)");
    if (f.on && depth && !f.depth) return im_fail(IMMESH_E_INVALID, "feed_images: depth requested but the feed was enabled without depth");
    FeedRings rings = mfeed_image_rings(f.max_frames, f.max_images, f.npx, f.hdr, f.rgba, f.depth_ring);
    void* rows = rgba;
    void* second = depth;
    if (!rgba && depth) {   // the depth images alone: they are the rows
        rings.rows = f.depth_ring;
        rings.idx = nullptr;
        rows = depth;
        second = nullptr;
    }
    return mesh_feed_read(h, "feed_images", true, rings, since, wait, frames, nullptr, cap_images, rows, second, cap_images, counts);
}

