// immesh_b200 -- the textured mesh rendered at a camera and scored against a photo (immesh_mesh_render_textured; the pixel rule is stated
// in include/immesh_b200.h).  CUDA kernels (sm_90a, bodies in texture_render_core.cuh) and their C-ABI host orchestration.
//   Once: the live triangles in snapshot order (mesh_tri_order) and each live slot's snapshot row (k_trv_rows).
//   Pass A: the depth image's binning passes at the rows' positions (rf_bin_launch), then one block per tile (k_trv_tile, k_view_tile's
// shape and visibility) that writes every pixel's depth and row, the source point of a textured winner in its image (float64) and its
// camera's needed flag, the colour of an untextured or empty pixel, and the three pixel counts (a block count, one atomic per block).
//   Pass B: one thread per pixel (k_trv_sample) samples its image bilinearly.  Device images: one launch.  Host images: the needed flags
// are read back and only the needed images are uploaded, in camera order, through the bake's two alternating arenas
// (tex_upload_batches); each batch's launch samples the pixels whose camera is in that batch.
//   Score: with a truth image, one pass (k_trv_score) sums exact int64 squared and absolute differences over the textured pixels, a warp
// reduction and one atomic per warp and value.
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "handles.hpp"
#include "texture_render_core.cuh"

using namespace immesh;

namespace {

// the per-pixel outputs of pass A
struct TrvOut {
    float* depth;                 // render_view's depth
    int* row;                     // the winner's snapshot row, -1: no sample
    double2* src;                 // a textured winner's source point in its image
    unsigned char* needed;        // [n_cams]
    unsigned char* rgb;           // [npx][3] or null: the colour of untextured and empty pixels
    uchar4 untex, bg;
    unsigned long long* cnt;      // [0] textured, [1] untextured, [2] empty pixels
};

// each live slot's snapshot row
__global__ void __launch_bounds__(128) k_trv_rows(const int4* rec, const unsigned int* order, int n, int* row_of) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) row_of[rec[order[i]].w] = i;
}

// pass A: one block per tile, one thread per pixel (k_view_tile's shape and visibility): the bin's set-ups and (a, b, c, slot) staged
// IM_RT_THREADS at a time in shared memory, each thread keeps its pixel's best (depth bits, triple, slot) in registers.  Bins over
// capacity (misc[0]): every triangle slot instead.  k_view_tile shades its winner and k_tex_tile counts covered samples inside the
// loop; here the winner's row, weights and source point are resolved once after it.
__global__ void __launch_bounds__(IM_RT_THREADS) k_trv_tile(MeshDev M, int pos_mode, const DepthCam* cam, const int* tile_off, const int* bin, const int* misc,
                                                            const int* row_of, const int* fcam, const float* fuv, const int4* wh, TrvOut o) {
    __shared__ DepthTri S[IM_RT_THREADS];
    __shared__ int4 Q[IM_RT_THREADS];
    const DepthCam C = *cam;
    const int ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    const int x = (blockIdx.x % ntx) * IM_RT_TILE + (int)(threadIdx.x % IM_RT_TILE), y = (blockIdx.x / ntx) * IM_RT_TILE + (int)(threadIdx.x / IM_RT_TILE);
    const bool all = misc[0] != 0;
    const int lo = all ? 0 : tile_off[blockIdx.x], hi = all ? min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t) : tile_off[blockIdx.x + 1];
    unsigned int best = 0x7f800000u;   // +inf: nothing drawn
    int ba = INT_MAX, bb = INT_MAX, bc = INT_MAX, bs = -1;
    for (int b = lo; b < hi; b += IM_RT_THREADS) {
        const int i = b + (int)threadIdx.x;
        bool ok = false;
        if (i < hi) {
            const int slot = all ? i : bin[i];
            const int4 r = M.tri[slot];
            ok = r.w && depth_tri_setup(C, tex_vertex(M, pos_mode, r.x), tex_vertex(M, pos_mode, r.y), tex_vertex(M, pos_mode, r.z), &S[threadIdx.x]);
            Q[threadIdx.x] = make_int4(r.x, r.y, r.z, slot);
        }
        if (!ok) { S[threadIdx.x].x_lo = 1; S[threadIdx.x].x_hi = 0; }   // an empty box
        __syncthreads();
        const int n = min(IM_RT_THREADS, hi - b);
        for (int j = 0; j < n; ++j) {
            const DepthTri& T = S[j];
            if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
            float zf;
            if (!depth_sample(T, x, y, &zf)) continue;
            const unsigned int bits = __float_as_uint(zf);
            const int4 q = Q[j];
            if (bits < 0x7f800000u && view_better(bits, q.x, q.y, q.z, best, ba, bb, bc)) { best = bits; ba = q.x; bb = q.y; bc = q.z; bs = q.w; }
        }
        __syncthreads();
    }
    const bool in = x < C.w && y < C.h;
    const int row = in && bs >= 0 ? row_of[bs] : -1, k = row >= 0 ? fcam[row] : -1;
    const int n_tex = __syncthreads_count(k >= 0), n_untex = __syncthreads_count(row >= 0 && k < 0), n_empty = __syncthreads_count(in && row < 0);
    if (threadIdx.x == 0) {
        if (n_tex) atomicAdd(&o.cnt[0], (unsigned long long)n_tex);
        if (n_untex) atomicAdd(&o.cnt[1], (unsigned long long)n_untex);
        if (n_empty) atomicAdd(&o.cnt[2], (unsigned long long)n_empty);
    }
    if (!in) return;
    const size_t px = (size_t)y * C.w + x;
    const float val = __uint_as_float(best);
    o.depth[px] = depth_valid(C, val) ? val : -1.0f;
    o.row[px] = row;
    if (k >= 0) {
        const int4 r = M.tri[bs];
        DepthTri T;
        depth_tri_setup(C, tex_vertex(M, pos_mode, r.x), tex_vertex(M, pos_mode, r.y), tex_vertex(M, pos_mode, r.z), &T);
        double w[3], p[6], sx, sy;
        trv_weights(T, x, y, (int)(M.tri_flip[bs] & 1ull), w);
        const int4 d = wh[k];
        bake_scaled(fuv + 6 * (size_t)row, d.x, d.y, d.z, d.w, p);
        trv_source(w, p, &sx, &sy);
        o.src[px] = make_double2(sx, sy);
        o.needed[k] = 1;
    } else if (o.rgb) {
        const uchar4 c = row >= 0 ? o.untex : o.bg;
        o.rgb[3 * px] = c.x; o.rgb[3 * px + 1] = c.y; o.rgb[3 * px + 2] = c.z;
    }
}

// pass B: one thread per pixel; the pixels whose camera is in [k_lo, k_hi] sample their image
__global__ void __launch_bounds__(256) k_trv_sample(const int* prow, const int* fcam, const double2* src, int npx, int k_lo, int k_hi, const BakeImg* imgs,
                                                    unsigned char* rgb) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += gridDim.x * blockDim.x) {
        const int r = prow[i];
        if (r < 0) continue;
        const int k = fcam[r];
        if (k < k_lo || k > k_hi) continue;
        const double2 s = src[i];
        bake_bilinear(imgs[k], s.x, s.y, rgb + 3 * (size_t)i);
    }
}

// the score: per thread the sums over its textured pixels, a warp reduction, one atomic per warp and value into cnt[4, 8)
__global__ void __launch_bounds__(256) k_trv_score(const int* prow, const int* fcam, const unsigned char* rgb, BakeImg truth, int npx, unsigned long long* cnt) {
    long long e[4] = {0, 0, 0, 0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += gridDim.x * blockDim.x) {
        const int r = prow[i];
        if (r < 0 || fcam[r] < 0) continue;
        trv_error(rgb + 3 * (size_t)i, truth.data + (size_t)(i / truth.w) * truth.pitch + 3 * (size_t)(i % truth.w), e, e + 3);
    }
    for (int v = 0; v < 4; ++v) {
        long long s = e[v];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(&cnt[4 + v], (unsigned long long)s);
    }
}

int trv_tiles(int w, int h) { return ((w + IM_RT_TILE - 1) / IM_RT_TILE) * ((h + IM_RT_TILE - 1) / IM_RT_TILE); }

// the phases of the last call on this thread (immesh_mesh_render_textured_stats)
thread_local double trv_ms[3] = {0, 0, 0};

// the call's timing events, released on every return
struct TrvEvents {
    cudaEvent_t e[4] = {};
    cudaError_t create() {
        cudaError_t r = cudaSuccess;
        for (int i = 0; i < 4 && r == cudaSuccess; ++i) r = cudaEventCreate(&e[i]);
        return r;
    }
    ~TrvEvents() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
};

}  // namespace

int immesh_mesh_render_textured(immesh_mesh_t* h, const immesh_texture_camera* view, const immesh_texture_view_config* cfg, const immesh_texture_camera* cams,
                                int n_cams, const immesh_texture_image* images, int on_device, const int32_t* facet_cam, const float* facet_uv, int64_t n_facets,
                                const immesh_texture_image* truth, uint8_t* rgb, float* depth, int32_t* facet, uint8_t* needed, int64_t* counts) {
    if (!h) return im_fail(IMMESH_E_INVALID, "render_textured: bad argument (NULL h)");
    cudaStream_t st = h->stream;
    IM_CUDA(cudaStreamSynchronize(st));   // the frames already queued, the pipelined ones included
    int mc[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, mc));
    const int n = mc[IM_MC_TRIS_LIVE], nalloc = std::min(mc[IM_MC_TRIS_ALLOC], h->M.max_t);
    std::vector<unsigned char> used;
    {
        const std::string why = trv_check(view, cfg, cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, truth, rgb, n, h->F.shard_n, used);
        if (!why.empty()) return im_fail(IMMESH_E_INVALID, ("render_textured: " + why).c_str());
    }
    const DepthCam C = tex_camera(*view, cfg->z_near, cfg->z_far);
    const int W = view->width, H = view->height, npx = W * H, ntiles = trv_tiles(W, H), pos = cfg->positions;
    const bool colour = images && (rgb || truth);
    std::vector<int4> hwh(n_cams);
    trv_sizes(cams, images, n_cams, &hwh[0].x);
    const size_t n1 = (size_t)std::max(n, 1);
    MemSet mem;   // every buffer of the call, released on every return
    DepthCam* d_cam = nullptr;
    RfImage im;
    TriOrder o = {};
    int *row_of = nullptr, *d_fcam = nullptr, *prow = nullptr;
    float *d_fuv = nullptr, *d_depth = nullptr;
    int4* d_wh = nullptr;
    BakeImg* d_img = nullptr;
    double2* src = nullptr;
    unsigned char *d_needed = nullptr, *d_rgb = nullptr, *d_truth = nullptr;
    unsigned long long* cnt = nullptr;
    {
        cudaError_t e = cudaSuccess;
        auto add = [&e, &mem](auto** p, size_t count) { if (e == cudaSuccess) e = mem.alloc(p, std::max<size_t>(count, 1)); };
        add(&d_cam, 1);
        im.ntiles = ntiles;
        im.bin_cap = (int)std::min<long long>(INT_MAX, std::max<long long>({1LL << 22, 16LL * ntiles, 8LL * nalloc}));
        add(&im.tile_cnt, (size_t)ntiles); add(&im.tile_off, (size_t)ntiles + 1); add(&im.bin, (size_t)im.bin_cap); add(&im.misc, 4);
        if (n > 0) {
            o.cap = n;
            add(&o.rec, n1);
            for (int b = 0; b < 2; ++b) { add(&o.k[b], n1); add(&o.v[b], n1); }
            add(&o.hist, mesh_sort_hist_ints(n1)); add(&o.misc, 8);
        }
        add(&row_of, (size_t)nalloc); add(&d_fcam, n1); add(&d_fuv, 6 * n1); add(&d_wh, (size_t)n_cams); add(&d_img, (size_t)n_cams);
        add(&prow, (size_t)npx); add(&src, (size_t)npx); add(&d_depth, (size_t)npx); add(&d_needed, (size_t)n_cams); add(&cnt, 8);
        if (colour) add(&d_rgb, 3 * (size_t)npx);
        if (truth && !on_device) add(&d_truth, 3 * (size_t)npx);
        if (e != cudaSuccess) return im_fail_alloc(e, "render_textured: allocation of the call's buffers failed");
    }
    TrvEvents ev;
    IM_CUDA(ev.create());
    im.cam = d_cam;
    IM_CUDA(cudaEventRecord(ev.e[0], st));
    IM_CUDA(cudaMemcpyAsync(d_cam, &C, sizeof(C), cudaMemcpyHostToDevice, st));
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(d_fcam, facet_cam, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaMemcpyAsync(d_fuv, facet_uv, (size_t)n * 6 * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    IM_CUDA(cudaMemcpyAsync(d_wh, hwh.data(), (size_t)n_cams * sizeof(int4), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(d_needed, 0, (size_t)n_cams, st));
    IM_CUDA(cudaMemsetAsync(cnt, 0, 8 * sizeof(unsigned long long), st));
    IM_CUDA(cudaMemsetAsync(im.tile_cnt, 0, (size_t)ntiles * sizeof(int), st));
    // pass A
    if (n > 0) {
        if (const int rc = mesh_tri_order(h, mc, 0.0, o)) return rc;
        IM_LAUNCH(k_trv_rows, mesh_grid(h, n, 128), 128, 0, st, (const int4*)o.rec, o.order, n, row_of);
    }
    rf_bin_launch(h, im, pos, st);
    const TrvOut out{d_depth, prow, src, d_needed, d_rgb, make_uchar4(cfg->untextured[0], cfg->untextured[1], cfg->untextured[2], 0),
                     make_uchar4(cfg->background[0], cfg->background[1], cfg->background[2], 0), cnt};
    IM_LAUNCH(k_trv_tile, ntiles, IM_RT_THREADS, 0, st, h->M, pos, (const DepthCam*)d_cam, (const int*)im.tile_off, (const int*)im.bin, (const int*)im.misc,
              (const int*)row_of, (const int*)d_fcam, (const float*)d_fuv, (const int4*)d_wh, out);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaEventRecord(ev.e[1], st));
    std::vector<unsigned char> hneed(n_cams);
    IM_CUDA(cudaMemcpyAsync(hneed.data(), d_needed, (size_t)n_cams, cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    {
        const std::string why = trv_check_needed(images, hneed.data(), n_cams);
        if (!why.empty()) return im_fail(IMMESH_E_INVALID, ("render_textured: " + why).c_str());
    }
    // pass B
    if (colour) {
        std::vector<BakeImg> himg(n_cams);
        for (int k = 0; k < n_cams; ++k) himg[k] = BakeImg{hneed[k] ? images[k].data : nullptr, images[k].width, images[k].height, (long long)images[k].pitch};
        auto sample = [&](int k_lo, int k_hi) {
            IM_LAUNCH(k_trv_sample, mesh_grid(h, npx, 256), 256, 0, st, (const int*)prow, (const int*)d_fcam, (const double2*)src, npx, k_lo, k_hi,
                      (const BakeImg*)d_img, d_rgb);
        };
        if (on_device) {
            IM_CUDA(cudaMemcpyAsync(d_img, himg.data(), (size_t)n_cams * sizeof(BakeImg), cudaMemcpyHostToDevice, st));
            sample(0, n_cams - 1);
        } else {
            long long arena_bytes = 0;
            const std::vector<int> batch_start = bake_batches(images, hneed.data(), n_cams, bake_arena_bytes(cfg->max_image_bytes), &arena_bytes);
            unsigned char* arena[2] = {nullptr, nullptr};
            cudaError_t e = cudaSuccess;
            for (int a = 0; a < 2 && e == cudaSuccess && arena_bytes > 0 && (a == 0 || batch_start.size() > 2); ++a) e = mem.alloc(&arena[a], (size_t)arena_bytes);
            if (e != cudaSuccess) return im_fail_alloc(e, "render_textured: allocation of the image arenas failed");
            if (const int rc = tex_upload_batches(st, images, hneed.data(), batch_start, arena, himg, d_img, sample)) return rc;
        }
    }
    IM_CUDA(cudaEventRecord(ev.e[2], st));
    // score
    if (truth) {
        BakeImg T{truth->data, W, H, (long long)truth->pitch};
        if (!on_device) {
            IM_CUDA(cudaMemcpy2DAsync(d_truth, (size_t)W * 3, truth->data, (size_t)truth->pitch, (size_t)W * 3, (size_t)H, cudaMemcpyHostToDevice, st));
            T = BakeImg{d_truth, W, H, 3LL * W};
        }
        IM_LAUNCH(k_trv_score, mesh_grid(h, npx, 256), 256, 0, st, (const int*)prow, (const int*)d_fcam, (const unsigned char*)d_rgb, T, npx, cnt);
    }
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaEventRecord(ev.e[3], st));
    unsigned long long hcnt[8];
    IM_CUDA(cudaMemcpyAsync(hcnt, cnt, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
    if (rgb) IM_CUDA(cudaMemcpyAsync(rgb, d_rgb, 3 * (size_t)npx, cudaMemcpyDeviceToHost, st));
    if (depth) IM_CUDA(cudaMemcpyAsync(depth, d_depth, (size_t)npx * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (facet) IM_CUDA(cudaMemcpyAsync(facet, prow, (size_t)npx * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < 3; ++i) {
        float ms = 0.f;
        IM_CUDA(cudaEventElapsedTime(&ms, ev.e[i], ev.e[i + 1]));
        trv_ms[i] = ms;
    }
    if (needed) std::memcpy(needed, hneed.data(), (size_t)n_cams);
    if (counts) {
        long long sampled = 0;
        for (int k = 0; k < n_cams; ++k) sampled += hneed[k];
        counts[0] = (int64_t)hcnt[0]; counts[1] = (int64_t)hcnt[1]; counts[2] = (int64_t)hcnt[2]; counts[3] = sampled;
        for (int i = 4; i < 8; ++i) counts[i] = (int64_t)hcnt[i];
    }
    return IMMESH_OK;
}

int immesh_mesh_render_textured_stats(double* ms) {
    if (!ms) return im_fail(IMMESH_E_INVALID, "render_textured_stats: null ms");
    for (int i = 0; i < 3; ++i) ms[i] = trv_ms[i];
    return IMMESH_OK;
}
