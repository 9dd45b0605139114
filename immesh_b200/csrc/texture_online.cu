// immesh_b200 -- the texturing queued behind every frame (immesh_mesh_texture_enable, _pose, _rows; the rule is stated in
// include/immesh_b200.h).  CUDA kernels (sm_90a, bodies in texture_core.cuh) and their C-ABI host orchestration.
//   Per frame, on the mesh stream inside the frame's captured launch sequence, after the view: one thread derives the frame's texture
// camera (k_txo_cam: the caller's, the rig on the handed-over pose from the camera ring, the rig on the depth frame's camera, or none)
// and clears the tile counters; immesh_mesh_texture_select's binning passes (rf_bin_launch) and tile kernel (k_tex_tile, counting per
// triangle slot); then one thread per slot (k_txo_update) applies the "seen" test to the slots that have counts, keeps the nearer
// frame with a strict <, and clears the counts.  A frame without a camera runs the same launches at an empty z range: nothing is
// counted and no state changes.
//   Rows (blocking): the live triangles in snapshot order (mesh_tri_order) read out (k_txo_rows); the records' frames keyed with their
// liveness, sorted (mesh_sort_passes) and made unique (k_txo_unique) for the frames list and the frames used by live rows.
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "block_scan.cuh"
#include "handles.hpp"
#include "texture_core.cuh"

using namespace immesh;

namespace {

enum TxoSrc { TXO_SRC_NONE = 0, TXO_SRC_RING = 1, TXO_SRC_DEPTH = 2 };   // where a frame's sensor pose comes from (static per graph)

// k_tex_tile counts a slot's pixels at the slot itself
struct TexSlot {
    __device__ __forceinline__ int operator()(int slot) const { return slot; }
};

// one block: the frame's texture camera into *cam (rd->mode 1: the caller's camera; else the rig on the frame's sensor pose), the
// tile counters cleared, and w * h added to *pixels when the frame has a camera.  Without one, an empty z range (z_near = z_far = 0)
// lets no triangle through the set-up.
__global__ void __launch_bounds__(256) k_txo_cam(int src, const double (*ring)[12], const int* ring_frame, const DepthFrame* df, const FrameDyn* dyn,
                                                 const RfDyn* rd, immesh_texture_camera rig, double z_near, double z_far, DepthCam* cam, int* tile_cnt,
                                                 int ntiles, long long* pixels) {
    for (int i = threadIdx.x; i < ntiles; i += blockDim.x) tile_cnt[i] = 0;
    if (threadIdx.x != 0) return;
    const int frame = dyn->frame, s = frame % IM_RF_RING;
    immesh_texture_camera c = rig;
    bool has = true;
    if (rd->mode == 1) c = txo_fixed_camera(rig, rd->R, rd->t);
    else if (src == TXO_SRC_RING && ring_frame[s] == frame) c = txo_camera(rig, ring[s], ring[s] + 9);
    else if (src == TXO_SRC_DEPTH) c = txo_camera(rig, df->R, df->t);
    else has = false;
    DepthCam C = tex_camera(c, z_near, z_far);
    if (!has) C.z_near = C.z_far = 0.0;
    *cam = C;
    if (has) *pixels += (long long)rig.width * rig.height;
}

// one thread per allocated slot: the slots k_tex_tile counted (live at this frame) get the "seen" test at the frame's camera with their
// current flip, the nearer frame kept (txo_observe); the counts cleared for the next frame
__global__ void __launch_bounds__(128) k_txo_update(MeshDev M, const DepthCam* cam, TexRule rule, const FrameDyn* dyn, TxoRecord* rec, int* won, int* cov) {
    const int n_alloc = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int wn = won[t], cv = cov[t];
        if (wn == 0 && cv == 0) continue;
        won[t] = 0; cov[t] = 0;
        if (wn < 1) continue;
        const int4 r = M.tri[t];
        const float4 p[3] = {M.vpos[r.x], M.vpos[r.y], M.vpos[r.z]};
        const int frame = dyn->frame;
        TxoRecord s = rec[t];
        txo_observe(*cam, p, (int)(M.tri_flip[t] & 1ull), wn, cv, rule, frame, &s);
        if (s.frame == frame) rec[t] = s;
    }
}

// a fresh state: every record unobserved, the counts zero
__global__ void __launch_bounds__(128) k_txo_init(TxoRecord* rec, int* won, int* cov, int n) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        TxoRecord s;
        s.frame = -1; s.e2 = INFINITY; s.won = 0; s.cov = 0;
        for (int k = 0; k < 6; ++k) s.uv[k] = 0.f;
        rec[t] = s;
        won[t] = 0; cov[t] = 0;
    }
}

// the rows in snapshot order: frame, texture coordinates in the current face order (textured rows only), won / covered; counts
// [textured, untextured]
__global__ void __launch_bounds__(128) k_txo_rows(MeshDev M, const int4* orec, const unsigned int* order, int n, const TxoRecord* rec, int* cam_out, float* uv_out,
                                                  int* px_out, int* cnt) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int t = orec[order[i]].w;
        const TxoRecord& s = rec[t];
        cam_out[i] = s.frame;
        px_out[2 * (size_t)i] = s.frame >= 0 ? s.won : 0;
        px_out[2 * (size_t)i + 1] = s.frame >= 0 ? s.cov : 0;
        if (s.frame < 0) { atomicAdd(&cnt[1], 1); continue; }
        txo_face_uv(s.uv, (int)(M.tri_flip[t] & 1ull), uv_out + 6 * (size_t)i);
        atomicAdd(&cnt[0], 1);
    }
}

// every observed record's key (frame << 1) | (not live), in any order, their count in *nk
__global__ void __launch_bounds__(128) k_txo_keys(MeshDev M, int n_alloc, const TxoRecord* rec, unsigned int* key, unsigned int* val, int* nk) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int f = rec[t].frame;
        if (f < 0) continue;
        const int e = atomicAdd(nk, 1);
        key[e] = ((unsigned int)f << 1) | (M.tri[t].w ? 0u : 1u);
        val[e] = (unsigned int)t;
    }
}

// one block over the sorted keys: the first key of each frame appends the frame to frames (ascending); it is even when a live record
// has that frame.  cnt[2]: frames of live records, cnt[3]: frames
__global__ void __launch_bounds__(1024) k_txo_unique(const unsigned int* key, int n, int* frames, int* cnt) {
    auto first = [&](int c) { return c == 0 || (key[c] >> 1) != (key[c - 1] >> 1); };
    const int total = chunk_scan_1024(n, [&](int c) { return first(c) ? 1 : 0; }, [&](int c, int run) {
        if (!first(c)) return 0;
        frames[run] = (int)(key[c] >> 1);
        if (!(key[c] & 1u)) atomicAdd(&cnt[2], 1);
        return 1;
    });
    if (threadIdx.x == 1023) cnt[3] = total;
}

}  // namespace

// ---- the state's growth along the triangle pool (mesh_grow, mesh_capi.cu)
cudaError_t txo_state_alloc(immesh::MemSet& mem, size_t tris, TxoRecord** rec, int** won, int** cov) {
    cudaError_t e = mem.alloc(rec, std::max<size_t>(tris, 1));
    if (e == cudaSuccess) e = mem.alloc(won, std::max<size_t>(tris, 1));
    if (e == cudaSuccess) e = mem.alloc(cov, std::max<size_t>(tris, 1));
    return e;
}
// the new state: fresh for all `tris` slots, then the first nt records of the old one (the counts are zero between frames)
cudaError_t txo_state_migrate(const immesh_mesh* h, cudaStream_t st, TxoRecord* rec, int* won, int* cov, int tris, const TxoRecord* old_rec, int nt) {
    IM_LAUNCH(k_txo_init, mesh_grid(h, tris, 128), 128, 0, st, rec, won, cov, tris);
    if (nt > 0) return cudaMemcpyAsync(rec, old_rec, (size_t)nt * sizeof(TxoRecord), cudaMemcpyDeviceToDevice, st);
    return cudaGetLastError();
}

// ---- the frame's stage (mesh_enqueue's launch sequence): source 0 a world-frame push, 1 a localization hand-off, 2 a depth frame
void mesh_texture_launch(immesh_mesh* h, int src, cudaStream_t st) {
    auto& x = h->tx;
    const RfImage& im = x.img;
    IM_LAUNCH(k_txo_cam, 1, 256, 0, st, src, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame, (const DepthFrame*)h->dep.d_df,
              (const FrameDyn*)h->d_dyn, (const RfDyn*)x.rd, x.rig, x.cfg.z_near, x.cfg.z_far, im.cam, im.tile_cnt, im.ntiles, x.pixels);
    rf_bin_launch(h, im, 0, st);
    IM_LAUNCH(k_tex_tile<TexSlot>, im.ntiles, IM_RT_THREADS, 0, st, h->M, 0, (const DepthCam*)im.cam, (const int*)im.tile_off, (const int*)im.bin, (const int*)im.misc,
              TexSlot{}, x.won, x.cov);
    IM_LAUNCH(k_txo_update, h->n_sm * 8, 128, 0, st, h->M, (const DepthCam*)im.cam, tex_rule(x.cfg), (const FrameDyn*)h->d_dyn, x.rec, x.won, x.cov);
}

int immesh_mesh_texture_enable(immesh_mesh_t* h, const immesh_texture_camera* rig, const immesh_texture_config* cfg) {
    if (!h) return im_fail(IMMESH_E_INVALID, "texture_enable: null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "texture_enable: a sharded mesh handle is not supported (the texturing runs on a single GPU)");
    if (rig) {
        if (!cfg || !tex_config_ok(*cfg) || cfg->positions != 0)
            return im_fail(IMMESH_E_INVALID, "texture_enable: bad config (0 < z_near < z_far < inf; min_cos in [0, 1]; min_visible_permille in [0, 1000]; two_sided 0 or 1; positions 0)");
        if (!tex_camera_ok(*rig))
            return im_fail(IMMESH_E_INVALID, "texture_enable: bad rig (1 <= width * height <= 2^26; finite intrinsics and pose; fx, fy != 0)");
    }
    IM_CUDA(im_stage_reset(h, [h] { h->tx = immesh_mesh::Texture(); }));
    if (!rig) return IMMESH_OK;
    immesh_mesh::Texture x;   // built in full before it replaces h->tx: after a failure the texturing stays off
    x.rig = *rig;
    x.cfg = *cfg;
    RfImage& im = x.img;
    im.ntiles = ((rig->width + IM_RT_TILE - 1) / IM_RT_TILE) * ((rig->height + IM_RT_TILE - 1) / IM_RT_TILE);
    im.bin_cap = std::max(1 << 22, 16 * im.ntiles);   // beyond it a frame's tiles walk every triangle slot (same counts, slower)
    const int tris = h->M.max_t;
    cudaError_t e = cudaSuccess;
    auto add = [&e, &x](auto** p, size_t count) { if (e == cudaSuccess) e = x.dev.alloc(p, std::max<size_t>(count, 1)); };
    add(&im.cam, 1); add(&im.tile_cnt, (size_t)im.ntiles); add(&im.tile_off, (size_t)im.ntiles + 1); add(&im.bin, (size_t)im.bin_cap); add(&im.misc, 4);
    add(&x.pixels, 1);
    if (e == cudaSuccess) e = txo_state_alloc(x.dev, (size_t)tris, &x.rec, &x.won, &x.cov);
    if (e == cudaSuccess) e = queued_cam_alloc(x);
    if (e == cudaSuccess) e = cudaMemsetAsync(x.pixels, 0, sizeof(long long), h->stream);
    if (e == cudaSuccess) {
        IM_LAUNCH(k_txo_init, mesh_grid(h, tris, 128), 128, 0, h->stream, x.rec, x.won, x.cov, tris);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return im_fail_alloc(e, "texture_enable: allocation of the texturing state failed");
    x.on = 1;
    h->tx = std::move(x);
    return IMMESH_OK;
}

int immesh_mesh_texture_pose(immesh_mesh_t* h, const double* cam_R, const double* cam_t) {
    if (!h || (!cam_R) != (!cam_t)) return im_fail(IMMESH_E_INVALID, "texture_pose: bad argument (cam_R and cam_t both given or both NULL)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "texture_pose: a sharded mesh handle is not supported");
    if (!h->tx.on) return im_fail(IMMESH_E_INVALID, "texture_pose: the texturing is not enabled (immesh_mesh_texture_enable)");
    for (int i = 0; cam_R && i < 9; ++i)
        if (!std::isfinite(cam_R[i])) return im_fail(IMMESH_E_INVALID, "texture_pose: a non-finite cam_R");
    for (int i = 0; cam_t && i < 3; ++i)
        if (!std::isfinite(cam_t[i])) return im_fail(IMMESH_E_INVALID, "texture_pose: a non-finite cam_t");
    h->tx.mode = cam_R ? 1 : 0;
    for (int i = 0; i < 9; ++i) h->tx.R[i] = cam_R ? cam_R[i] : 0.0;
    for (int i = 0; i < 3; ++i) h->tx.t[i] = cam_t ? cam_t[i] : 0.0;
    return IMMESH_OK;
}

int immesh_mesh_texture_rows(immesh_mesh_t* h, int32_t* facet_cam, float* facet_uv, int32_t* facet_px, int64_t cap, int64_t* n_facets, int64_t* counts,
                             int32_t* frames, int64_t cap_frames, int64_t* n_frames) {
    if (!h || !n_facets || cap < 0 || cap_frames < 0 || (frames && !n_frames))
        return im_fail(IMMESH_E_INVALID, "texture_rows: bad argument (NULL h or n_facets; cap or cap_frames < 0; frames without n_frames)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "texture_rows: a sharded mesh handle is not supported");
    if (!h->tx.on) return im_fail(IMMESH_E_INVALID, "texture_rows: the texturing is not enabled (immesh_mesh_texture_enable)");
    const auto& x = h->tx;
    cudaStream_t st = h->stream;
    IM_CUDA(cudaStreamSynchronize(st));   // the frames already queued, the pipelined ones included
    int mc[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, mc));
    const int n = mc[IM_MC_TRIS_LIVE], nalloc = std::min(mc[IM_MC_TRIS_ALLOC], h->M.max_t);
    const size_t n1 = (size_t)std::max(n, 1), na1 = (size_t)std::max(nalloc, 1);
    MemSet mem;   // every buffer of the call, released on every return
    TriOrder o = {};
    unsigned int *fk[2] = {}, *fv[2] = {};
    int *fhist = nullptr, *nk = nullptr, *fr_out = nullptr, *cam_out = nullptr, *px_out = nullptr, *cnt = nullptr;
    float* uv_out = nullptr;
    {
        cudaError_t e = cudaSuccess;
        auto add = [&e, &mem](auto** p, size_t count) { if (e == cudaSuccess) e = mem.alloc(p, std::max<size_t>(count, 1)); };
        o.cap = n;
        add(&o.rec, n1);
        for (int b = 0; b < 2; ++b) { add(&o.k[b], n1); add(&o.v[b], n1); add(&fk[b], na1); add(&fv[b], na1); }
        add(&o.hist, mesh_sort_hist_ints(n1)); add(&o.misc, 8);
        add(&fhist, mesh_sort_hist_ints(na1)); add(&nk, 1); add(&fr_out, na1);
        add(&cam_out, n1); add(&uv_out, n1 * 6); add(&px_out, n1 * 2); add(&cnt, 4);
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_rows: allocation of the call's buffers failed");
    }
    IM_CUDA(cudaMemsetAsync(cnt, 0, 4 * sizeof(int), st));
    IM_CUDA(cudaMemsetAsync(nk, 0, sizeof(int), st));
    if (n > 0) {
        if (const int rc = mesh_tri_order(h, mc, 0.0, o)) return rc;
        IM_LAUNCH(k_txo_rows, mesh_grid(h, n, 128), 128, 0, st, h->M, (const int4*)o.rec, o.order, n, (const TxoRecord*)x.rec, cam_out, uv_out, px_out, cnt);
    }
    int hk = 0;
    if (nalloc > 0) IM_LAUNCH(k_txo_keys, mesh_grid(h, nalloc, 128), 128, 0, st, h->M, nalloc, (const TxoRecord*)x.rec, fk[0], fv[0], nk);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(&hk, nk, sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (hk > 0) {
        const int cur = mesh_sort_passes(st, fk, fv, 0, hk, rb_passes(((unsigned long long)h->frame_counter << 1) | 1ull), fhist);
        IM_LAUNCH(k_txo_unique, 1, 1024, 0, st, (const unsigned int*)fk[cur], hk, fr_out, cnt);
    }
    IM_CUDA(cudaGetLastError());
    int hcnt[4] = {0, 0, 0, 0};
    long long pixels = 0;
    IM_CUDA(cudaMemcpyAsync(hcnt, cnt, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaMemcpyAsync(&pixels, x.pixels, sizeof(pixels), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int nfr = hcnt[3];
    *n_facets = n;
    if (n_frames) *n_frames = nfr;
    if (counts) {
        counts[0] = hcnt[0]; counts[1] = hcnt[1]; counts[2] = hcnt[2]; counts[3] = pixels;
    }
    if (n > cap || (frames && nfr > cap_frames))
        return im_fail(IMMESH_E_CAPACITY, "texture_rows: more live triangles than cap or more frames than cap_frames (*n_facets and *n_frames hold the numbers needed; nothing was written)");
    std::vector<int32_t> hcam(n1);
    std::vector<float> huv;
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(hcam.data(), cam_out, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (facet_uv) {
            huv.resize((size_t)n * 6);
            IM_CUDA(cudaMemcpyAsync(huv.data(), uv_out, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
        if (facet_px) IM_CUDA(cudaMemcpyAsync(facet_px, px_out, (size_t)n * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    if (frames && nfr > 0) IM_CUDA(cudaMemcpyAsync(frames, fr_out, (size_t)nfr * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (facet_cam && n > 0) std::memcpy(facet_cam, hcam.data(), (size_t)n * sizeof(int32_t));
    for (int i = 0; facet_uv && i < n; ++i)   // the rows of untextured facets are left as the caller had them
        if (hcam[i] >= 0) std::memcpy(facet_uv + 6 * (size_t)i, huv.data() + 6 * (size_t)i, 6 * sizeof(float));
    return IMMESH_OK;
}
