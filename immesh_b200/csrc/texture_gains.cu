// immesh_b200 -- colour equalisation between cameras (immesh_mesh_texture_gains, immesh_texture_apply_gains; the rule is stated in
// include/immesh_b200.h).  CUDA kernels (sm_90a, bodies in texture_gains_core.cuh) and their C-ABI host orchestration.
//   Once: the live triangles in snapshot order (mesh_tri_order) and each live slot's snapshot row (k_tg_rows).
//   Chosen side: one thread per textured row whose camera is in the batch (k_tg_chosen) stores its 10 RGB samples (30 B per row).
//   Observer pass, per camera k with an image in index order: texture_select's binning passes and tile kernel (rf_bin_launch,
// k_tex_tile counting at the snapshot row), then one thread per row (k_tg_observe) applies the "seen" test, samples image k and adds
// the kept sample pairs into a dense int64 row [n_cams][7] keyed by the row's camera c, aggregated per warp (__match_any_sync on c,
// one atomic per group and value); then one block (k_tg_compact) appends the non-zero entries in ascending c to the pair list
// (chunk_scan_1024) and clears the row.  No host round trip per camera.
//   Device images: one chosen launch, then every pass.  Host images: whole images in camera order through the bake's two alternating
// arenas (tex_upload_batches); with one batch its launch samples the chosen side then runs its passes; with more, a first sweep samples
// the chosen side of every batch and a second sweep runs the passes, since a pass pairs with rows of every camera.
//   Solve: the pair list is read back and the normal equations are solved on the host (tg_solve: K x K, sparse, tiny next to the passes).
#include <chrono>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "block_scan.cuh"
#include "handles.hpp"
#include "texture_gains_core.cuh"

using namespace immesh;

namespace {

// each live slot's snapshot row and record; the rows' counts cleared
__global__ void __launch_bounds__(128) k_tg_rows(const int4* rec, const unsigned int* order, int n, int* row_of, int4* row_rec, int* won, int* cov) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 r = rec[order[i]];
        row_of[r.w] = i;
        row_rec[i] = r;
        won[i] = 0; cov[i] = 0;
    }
}

// the chosen side: rows whose camera is in [k_lo, k_hi] store their 10 samples of that camera's image
__global__ void __launch_bounds__(128) k_tg_chosen(const int* fcam, const float* fuv, int n, int k_lo, int k_hi, const int4* wh, const BakeImg* imgs,
                                                   unsigned char* chosen) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = fcam[i];
        if (c < k_lo || c > k_hi) continue;
        const int4 d = wh[c];
        double p[6];
        bake_scaled(fuv + 6 * (size_t)i, d.x, d.y, d.z, d.w, p);
        tg_sample(imgs[c], p, chosen + (size_t)(3 * IM_TG_POINTS) * i);
    }
}

// observer k: per row the "seen" test on k_tex_tile's counts (cleared here for the next pass), the observer's samples against the
// chosen side's, the kept sums added into prow [n_cams][7] at the row's camera; per warp one atomic per camera group and value, and
// one per warp for the used / clipped totals (cnt [0], [1])
__global__ void __launch_bounds__(128) k_tg_observe(MeshDev M, int pos_mode, const DepthCam* cam, int k, TexRule rule, const int4* row_rec, const int* fcam,
                                                    int n, int* won, int* cov, const int4* wh, const BakeImg* imgs, const unsigned char* chosen,
                                                    unsigned long long* prow, unsigned long long* cnt) {
    const DepthCam C = *cam;
    const int lane = threadIdx.x & 31;
    int used = 0, clipped = 0;
    for (int base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {   // warp-uniform trip count
        const int i = base + (int)threadIdx.x;
        int c = -1, sum[IM_TG_SUMS] = {0, 0, 0, 0, 0, 0, 0};
        if (i < n) {
            const int wn = won[i], cv = cov[i];
            if (wn || cv) { won[i] = 0; cov[i] = 0; }
            const int fc = fcam[i];
            if (wn >= 1 && fc >= 0 && fc != k) {
                const int4 r = row_rec[i];
                float4 q[3];
                tex_corners(tex_vertex(M, pos_mode, r.x), tex_vertex(M, pos_mode, r.y), tex_vertex(M, pos_mode, r.z), (int)(M.tri_flip[r.w] & 1ull), q);
                double e2;
                if (tex_seen(C, q, wn, cv, rule, &e2)) {
                    float uv[6];
                    tex_uv(C, q, uv);
                    const int4 d = wh[k];
                    double p[6];
                    bake_scaled(uv, d.x, d.y, d.z, d.w, p);
                    unsigned char ok[3 * IM_TG_POINTS];
                    tg_sample(imgs[k], p, ok);
                    tg_accumulate(ok, chosen + (size_t)(3 * IM_TG_POINTS) * i, sum, &clipped);
                    if (sum[0] > 0) c = fc;
                }
            }
        }
        used += sum[0];
        const unsigned int grp = __match_any_sync(0xffffffffu, c);
        unsigned int leads = __ballot_sync(0xffffffffu, c >= 0 && lane == __ffs(grp) - 1);
        while (leads) {   // uniform over the warp
            const int src = __ffs(leads) - 1;
            leads &= leads - 1;
            const bool mine = (__shfl_sync(0xffffffffu, grp, src) >> lane) & 1u;
            const int cc = __shfl_sync(0xffffffffu, c, src);
#pragma unroll
            for (int v = 0; v < IM_TG_SUMS; ++v) {
                const int s = __reduce_add_sync(0xffffffffu, mine ? sum[v] : 0);
                if (lane == src && s) atomicAdd(&prow[(size_t)IM_TG_SUMS * cc + v], (unsigned long long)s);
            }
        }
    }
    const int u = __reduce_add_sync(0xffffffffu, used), cl = __reduce_add_sync(0xffffffffu, clipped);
    if (lane == 0) {
        if (u) atomicAdd(&cnt[0], (unsigned long long)u);
        if (cl) atomicAdd(&cnt[1], (unsigned long long)cl);
    }
}

// one block of 1024: observer k's non-zero entries of prow in ascending c appended to the pair list at *n_pairs (kept below cap,
// counted beyond it), and the row cleared
__global__ void __launch_bounds__(1024) k_tg_compact(unsigned long long* prow, int n_cams, int k, long long* n_pairs, long long cap, int* pair_cam,
                                                     long long* pair_sums) {
    const long long base = *n_pairs;
    const int total = chunk_scan_1024(
        n_cams, [&](int c) { return prow[(size_t)IM_TG_SUMS * c] ? 1 : 0; },
        [&](int c, int run) {
            unsigned long long* e = prow + (size_t)IM_TG_SUMS * c;
            if (!e[0]) return 0;
            const long long at = base + run;
            if (at < cap) {
                pair_cam[2 * at] = k;
                pair_cam[2 * at + 1] = c;
                for (int v = 0; v < IM_TG_SUMS; ++v) pair_sums[IM_TG_SUMS * at + v] = (long long)e[v];
            }
            for (int v = 0; v < IM_TG_SUMS; ++v) e[v] = 0;
            return 1;
        });
    if (threadIdx.x == 1023) *n_pairs = base + total;
}

// one image of immesh_texture_apply_gains
struct TgImg { const unsigned char* in; unsigned char* out; int w, h; long long pin, pout; double g[3]; };

// blockIdx.y strides over the images, the x threads over each image's pixels
__global__ void __launch_bounds__(256) k_tg_apply(const TgImg* imgs, int n) {
    for (int k = blockIdx.y; k < n; k += gridDim.y) {
        const TgImg I = imgs[k];
        if (!I.in) continue;
        const long long npx = (long long)I.w * I.h;
        for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npx; p += (long long)gridDim.x * blockDim.x) {
            const long long y = p / I.w, x = p % I.w;
            const unsigned char* a = I.in + y * I.pin + 3 * x;
            unsigned char* b = I.out + y * I.pout + 3 * x;
            const unsigned char v0 = a[0], v1 = a[1], v2 = a[2];
            b[0] = tg_apply(v0, I.g[0]); b[1] = tg_apply(v1, I.g[1]); b[2] = tg_apply(v2, I.g[2]);
        }
    }
}

int tg_tiles(int w, int h) { return ((w + IM_RT_TILE - 1) / IM_RT_TILE) * ((h + IM_RT_TILE - 1) / IM_RT_TILE); }

// the phases of the last call on this thread that reached the solve (immesh_mesh_texture_gains_stats)
thread_local double tg_ms[3] = {0, 0, 0};

// the call's timing events, released on every return
struct TgEvents {
    cudaEvent_t e[3] = {};
    cudaError_t create() {
        cudaError_t r = cudaSuccess;
        for (int i = 0; i < 3 && r == cudaSuccess; ++i) r = cudaEventCreate(&e[i]);
        return r;
    }
    ~TgEvents() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
};

}  // namespace

int immesh_mesh_texture_gains(immesh_mesh_t* h, const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device,
                              const int32_t* facet_cam, const float* facet_uv, int64_t n_facets, const immesh_texture_gains_config* cfg, double* gains,
                              int32_t* pair_cam, int64_t* pair_sums, int64_t* n_pairs, int64_t* counts) {
    if (!h) return im_fail(IMMESH_E_INVALID, "texture_gains: bad argument (NULL h)");
    cudaStream_t st = h->stream;
    IM_CUDA(cudaStreamSynchronize(st));   // the frames already queued, the pipelined ones included
    int mc[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, mc));
    const int n = mc[IM_MC_TRIS_LIVE], nalloc = std::min(mc[IM_MC_TRIS_ALLOC], h->M.max_t);
    std::vector<unsigned char> have;
    {
        const std::string why = tg_check(cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, cfg, gains, n, h->F.shard_n, have);
        if (!why.empty()) return im_fail(IMMESH_E_INVALID, ("texture_gains: " + why).c_str());
    }
    const immesh_texture_config& sel = cfg->sel;
    const int pos = sel.positions;
    std::vector<DepthCam> hc(n_cams);
    std::vector<int4> hwh(n_cams);
    std::vector<BakeImg> himg(n_cams);
    int n_obs = 0, max_tiles = 1;
    long long pixels = 0;
    for (int k = 0; k < n_cams; ++k) {
        hwh[k] = make_int4(1, 1, 1, 1);
        himg[k] = BakeImg{nullptr, 1, 1, 3};
        if (!have[k]) continue;
        hc[k] = tex_camera(cams[k], sel.z_near, sel.z_far);
        hwh[k] = make_int4(images[k].width, images[k].height, cams[k].width, cams[k].height);
        himg[k] = BakeImg{images[k].data, images[k].width, images[k].height, (long long)images[k].pitch};
        ++n_obs;
        pixels += (long long)cams[k].width * cams[k].height;
        max_tiles = std::max(max_tiles, tg_tiles(cams[k].width, cams[k].height));
    }
    if (n == 0) { n_obs = 0; pixels = 0; }   // nothing to see: no pass runs
    // each pass adds at most n_cams - 1 pairs
    const long long cap = std::max(1LL, std::min<long long>(cfg->max_pairs, (long long)n_obs * n_cams));
    const size_t n1 = (size_t)std::max(n, 1);
    MemSet mem;   // every buffer of the call, released on every return
    DepthCam* d_cams = nullptr;
    RfImage im;
    TriOrder o = {};
    int *row_of = nullptr, *won = nullptr, *cov = nullptr, *d_fcam = nullptr, *d_pcam = nullptr;
    int4 *row_rec = nullptr, *d_wh = nullptr;
    float* d_fuv = nullptr;
    BakeImg* d_img = nullptr;
    unsigned char* chosen = nullptr;
    unsigned long long *prow = nullptr, *cnt = nullptr;
    long long *d_npairs = nullptr, *d_psums = nullptr;
    {
        cudaError_t e = cudaSuccess;
        auto add = [&e, &mem](auto** p, size_t count) { if (e == cudaSuccess) e = mem.alloc(p, std::max<size_t>(count, 1)); };
        add(&d_cams, (size_t)n_cams); add(&d_wh, (size_t)n_cams); add(&d_img, (size_t)n_cams);
        add(&prow, (size_t)IM_TG_SUMS * n_cams); add(&cnt, 2); add(&d_npairs, 1);
        add(&d_pcam, 2 * (size_t)cap); add(&d_psums, (size_t)IM_TG_SUMS * cap);
        if (n > 0) {
            im.ntiles = max_tiles;
            im.bin_cap = (int)std::min<long long>(INT_MAX, std::max<long long>({1LL << 22, 16LL * max_tiles, 8LL * nalloc}));
            add(&im.tile_cnt, (size_t)max_tiles); add(&im.tile_off, (size_t)max_tiles + 1); add(&im.bin, (size_t)im.bin_cap); add(&im.misc, 4);
            o.cap = n;
            add(&o.rec, n1);
            for (int b = 0; b < 2; ++b) { add(&o.k[b], n1); add(&o.v[b], n1); }
            add(&o.hist, mesh_sort_hist_ints(n1)); add(&o.misc, 8);
            add(&row_of, (size_t)nalloc); add(&row_rec, n1); add(&won, n1); add(&cov, n1);
            add(&d_fcam, n1); add(&d_fuv, 6 * n1); add(&chosen, (size_t)(3 * IM_TG_POINTS) * n1);
        }
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_gains: allocation of the call's buffers failed");
    }
    TgEvents ev;
    IM_CUDA(ev.create());
    IM_CUDA(cudaEventRecord(ev.e[0], st));
    IM_CUDA(cudaMemcpyAsync(d_cams, hc.data(), (size_t)n_cams * sizeof(DepthCam), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemcpyAsync(d_wh, hwh.data(), (size_t)n_cams * sizeof(int4), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(prow, 0, (size_t)IM_TG_SUMS * n_cams * sizeof(unsigned long long), st));
    IM_CUDA(cudaMemsetAsync(cnt, 0, 2 * sizeof(unsigned long long), st));
    IM_CUDA(cudaMemsetAsync(d_npairs, 0, sizeof(long long), st));
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(d_fcam, facet_cam, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaMemcpyAsync(d_fuv, facet_uv, (size_t)n * 6 * sizeof(float), cudaMemcpyHostToDevice, st));
        if (const int rc = mesh_tri_order(h, mc, 0.0, o)) return rc;
        IM_LAUNCH(k_tg_rows, mesh_grid(h, n, 128), 128, 0, st, (const int4*)o.rec, o.order, n, row_of, row_rec, won, cov);
    }
    const TexRule rule = tex_rule(sel);
    auto chosen_side = [&](int k_lo, int k_hi) {
        if (n > 0)
            IM_LAUNCH(k_tg_chosen, mesh_grid(h, n, 128), 128, 0, st, (const int*)d_fcam, (const float*)d_fuv, n, k_lo, k_hi, (const int4*)d_wh,
                      (const BakeImg*)d_img, chosen);
    };
    auto observe = [&](int k_lo, int k_hi) {
        for (int k = k_lo; n > 0 && k <= k_hi; ++k) {
            if (!have[k]) continue;
            RfImage ik = im;
            ik.cam = d_cams + k;
            ik.ntiles = tg_tiles(cams[k].width, cams[k].height);
            cudaMemsetAsync(im.tile_cnt, 0, (size_t)ik.ntiles * sizeof(int), st);
            rf_bin_launch(h, ik, pos, st);
            IM_LAUNCH(k_tex_tile<TexRowOf>, ik.ntiles, IM_RT_THREADS, 0, st, h->M, pos, (const DepthCam*)ik.cam, (const int*)im.tile_off, (const int*)im.bin,
                      (const int*)im.misc, TexRowOf{row_of}, won, cov);
            IM_LAUNCH(k_tg_observe, mesh_grid(h, n, 128), 128, 0, st, h->M, pos, (const DepthCam*)ik.cam, k, rule, (const int4*)row_rec, (const int*)d_fcam, n,
                      won, cov, (const int4*)d_wh, (const BakeImg*)d_img, (const unsigned char*)chosen, prow, cnt);
            IM_LAUNCH(k_tg_compact, 1, 1024, 0, st, prow, n_cams, k, d_npairs, cap, d_pcam, d_psums);
        }
    };
    if (on_device) {
        IM_CUDA(cudaMemcpyAsync(d_img, himg.data(), (size_t)n_cams * sizeof(BakeImg), cudaMemcpyHostToDevice, st));
        chosen_side(0, n_cams - 1);
        IM_CUDA(cudaEventRecord(ev.e[1], st));
        observe(0, n_cams - 1);
    } else {
        long long arena_bytes = 0;
        const std::vector<unsigned char>& want = n > 0 ? have : std::vector<unsigned char>(n_cams, 0);
        const std::vector<int> batch_start = bake_batches(images, want.data(), n_cams, bake_arena_bytes(cfg->max_image_bytes), &arena_bytes);
        unsigned char* arena[2] = {nullptr, nullptr};
        cudaError_t e = cudaSuccess;
        for (int a = 0; a < 2 && e == cudaSuccess && arena_bytes > 0 && (a == 0 || batch_start.size() > 2); ++a) e = mem.alloc(&arena[a], (size_t)arena_bytes);
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_gains: allocation of the image arenas failed");
        if (batch_start.size() == 2) {   // one batch: its images stay resident for both phases
            if (const int rc = tex_upload_batches(st, images, want.data(), batch_start, arena, himg, d_img, [&](int first, int last) {
                    chosen_side(first, last);
                    cudaEventRecord(ev.e[1], st);
                    observe(first, last);
                }))
                return rc;
        } else {
            if (const int rc = tex_upload_batches(st, images, want.data(), batch_start, arena, himg, d_img, chosen_side)) return rc;
            IM_CUDA(cudaEventRecord(ev.e[1], st));
            IM_CUDA(cudaStreamSynchronize(st));   // the second sweep's copies reuse the arenas the first sweep's launches read
            if (const int rc = tex_upload_batches(st, images, want.data(), batch_start, arena, himg, d_img, observe)) return rc;
        }
    }
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaEventRecord(ev.e[2], st));
    long long np = 0;
    unsigned long long hcnt[2] = {0, 0};
    IM_CUDA(cudaMemcpyAsync(&np, d_npairs, sizeof(np), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaMemcpyAsync(hcnt, cnt, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const auto t0 = std::chrono::steady_clock::now();
    int iters = 0, left = 0;
    auto fill_counts = [&]() {
        if (n_pairs) *n_pairs = np;
        if (counts) {
            counts[0] = np; counts[1] = (int64_t)hcnt[0]; counts[2] = (int64_t)hcnt[1]; counts[3] = n_obs;
            counts[4] = left; counts[5] = iters; counts[6] = pixels; counts[7] = 0;
        }
    };
    if (np > cfg->max_pairs) {
        fill_counts();
        return im_fail(IMMESH_E_CAPACITY, "texture_gains: more pairs than max_pairs (*n_pairs holds the number; no gain was written)");
    }
    std::vector<int> hpc(2 * (size_t)std::max(np, 1LL));
    std::vector<long long> hps((size_t)IM_TG_SUMS * std::max(np, 1LL));
    if (np > 0) {
        IM_CUDA(cudaMemcpy(hpc.data(), d_pcam, 2 * (size_t)np * sizeof(int), cudaMemcpyDeviceToHost));
        IM_CUDA(cudaMemcpy(hps.data(), d_psums, (size_t)IM_TG_SUMS * np * sizeof(long long), cudaMemcpyDeviceToHost));
    }
    tg_solve(n_cams, hpc.data(), hps.data(), np, cfg->sigma_n, cfg->sigma_g, gains, &iters, &left);
    const auto t1 = std::chrono::steady_clock::now();
    if (pair_cam && np > 0) std::memcpy(pair_cam, hpc.data(), 2 * (size_t)np * sizeof(int32_t));
    if (pair_sums && np > 0) std::memcpy(pair_sums, hps.data(), (size_t)IM_TG_SUMS * np * sizeof(int64_t));
    fill_counts();
    float ms0 = 0.f, ms1 = 0.f;
    IM_CUDA(cudaEventElapsedTime(&ms0, ev.e[0], ev.e[1]));
    IM_CUDA(cudaEventElapsedTime(&ms1, ev.e[1], ev.e[2]));
    tg_ms[0] = ms0; tg_ms[1] = ms1;
    tg_ms[2] = std::chrono::duration<double, std::milli>(t1 - t0).count();
    return IMMESH_OK;
}

int immesh_mesh_texture_gains_stats(double* ms) {
    if (!ms) return im_fail(IMMESH_E_INVALID, "texture_gains_stats: null ms");
    for (int i = 0; i < 3; ++i) ms[i] = tg_ms[i];
    return IMMESH_OK;
}

int immesh_texture_apply_gains(immesh_mesh_t* h, const immesh_texture_image* in, const immesh_texture_image* out, int n, int on_device, const double* gains) {
    if (!h) return im_fail(IMMESH_E_INVALID, "texture_apply_gains: bad argument (NULL h)");
    {
        const std::string why = tg_apply_check(in, out, n, on_device, gains);
        if (!why.empty()) return im_fail(IMMESH_E_INVALID, ("texture_apply_gains: " + why).c_str());
    }
    std::vector<TgImg> hi(std::max(n, 1));
    long long max_px = 1;
    for (int k = 0; k < n; ++k) {
        hi[k] = TgImg{in[k].data, const_cast<unsigned char*>(out[k].data), in[k].width, in[k].height, (long long)in[k].pitch, (long long)out[k].pitch,
                      {gains[3 * k], gains[3 * k + 1], gains[3 * k + 2]}};
        if (in[k].data) max_px = std::max(max_px, (long long)in[k].width * in[k].height);
    }
    if (!on_device) {
        for (int k = 0; k < n; ++k) {
            const TgImg& I = hi[k];
            if (!I.in) continue;
            for (int y = 0; y < I.h; ++y)
                for (int x = 0; x < 3 * I.w; ++x) I.out[y * I.pout + x] = tg_apply(I.in[y * I.pin + x], I.g[x % 3]);
        }
        return IMMESH_OK;
    }
    if (n == 0) return IMMESH_OK;
    cudaStream_t st = h->stream;
    MemSet mem;
    TgImg* d = nullptr;
    {
        const cudaError_t e = mem.alloc(&d, (size_t)n);
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_apply_gains: allocation failed");
    }
    IM_CUDA(cudaMemcpyAsync(d, hi.data(), (size_t)n * sizeof(TgImg), cudaMemcpyHostToDevice, st));
    const dim3 grid((unsigned)mesh_grid_fixed(h, max_px, 256, 4), (unsigned)std::min(n, 65535));
    IM_LAUNCH(k_tg_apply, grid, 256, 0, st, (const TgImg*)d, n);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaStreamSynchronize(st));
    return IMMESH_OK;
}
