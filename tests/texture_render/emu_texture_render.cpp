// TEST INFRASTRUCTURE (not product code): immesh_mesh_render_textured's __host__ __device__ bodies (immesh_b200/csrc/texture_render_core.cuh,
// texture_bake_core.cuh, texture_core.cuh, reinforce.cuh) and its argument check run on the CPU with the device call's orchestration:
// the binning passes at the rows' positions (count, exclusive scan, fill in reverse slot order, or every slot when the bins overflow),
// every tile's pixels over its bin in batches of IM_RT_THREADS set-ups with the view's tie-break (k_trv_tile: depth, row, the source
// point and the needed flag of a textured winner, the colour of the others, the pixel counts), the needed check, then pass B
// (k_trv_sample) over device images in one pass or over host images batch by batch (bake_batches), each batch's images packed into an
// arena at pitch 3 width as tex_upload_batches lays them out, and the score (k_trv_score).  The shipped library never links or calls this.
#include <cstring>
#include <string>
#include <vector>

#include "../../immesh_b200/csrc/texture_render_core.cuh"

using namespace immesh;

static std::string g_err;

extern "C" {
const char* emu_texture_render_error() { return g_err.c_str(); }

// verts [nv][3] float; smooth [nv][3] / flags [nv] (or NULL); tris [nt][3] ascending triples and flips [nt], every one live, in the rows'
// (snapshot) order; bin_cap: bin entries beyond it walk every slot; shard_n: the handle's shards.  The other arguments and outputs as
// immesh_mesh_render_textured's; *n_batches: the host-image batches pass B ran (0 for device images or without colour).
int emu_texture_render(const immesh_texture_camera* view, const immesh_texture_view_config* cfg, const immesh_texture_camera* cams, int n_cams,
                       const immesh_texture_image* images, int on_device, const int32_t* facet_cam, const float* facet_uv, int64_t n_facets,
                       const immesh_texture_image* truth, const float* verts, const double* smooth, const unsigned char* flags, int nv, const int* tris,
                       const int* flips, int nt, long long bin_cap, int shard_n, uint8_t* rgb, float* depth, int32_t* facet, uint8_t* needed,
                       int64_t* counts, int* n_batches) {
    std::vector<unsigned char> used;
    g_err = trv_check(view, cfg, cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, truth, rgb, nt, shard_n, used);
    if (!g_err.empty()) return IMMESH_E_INVALID;
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    auto vtx = [&](int i) { return view_vertex(vpos.data(), smooth, flags, cfg->positions, i); };
    const DepthCam C = tex_camera(*view, cfg->z_near, cfg->z_far);
    const int w = C.w, h = C.h, npx = w * h;
    auto setup = [&](int t, DepthTri* T) { return depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), T); };
    std::vector<int> wh(4 * (size_t)n_cams);
    trv_sizes(cams, images, n_cams, wh.data());
    const bool colour = images && (rgb || truth);
    // k_rf_count / k_rf_scan / k_rf_fill
    const int ntx = (w + IM_RT_TILE - 1) / IM_RT_TILE, nty = (h + IM_RT_TILE - 1) / IM_RT_TILE, ntiles = ntx * nty;
    std::vector<long long> cnt(ntiles, 0), off(ntiles + 1, 0);
    for (int t = 0; t < nt; ++t) {
        DepthTri T;
        if (!setup(t, &T)) continue;
        for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
            for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) ++cnt[ty * ntx + tx];
    }
    for (int i = 0; i < ntiles; ++i) off[i + 1] = off[i] + cnt[i];
    const bool all = off[ntiles] > bin_cap;
    std::vector<int> bin(all || off[ntiles] == 0 ? 1 : (size_t)off[ntiles]);
    if (!all) {
        std::vector<long long> cur(off.begin(), off.end() - 1);
        for (int t = nt - 1; t >= 0; --t) {
            DepthTri T;
            if (!setup(t, &T)) continue;
            for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
                for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) bin[cur[ty * ntx + tx]++] = t;
        }
    }
    // k_trv_tile
    std::vector<float> d_depth(npx);
    std::vector<int> prow(npx, -1);
    std::vector<double> src(2 * (size_t)npx, 0.0);
    std::vector<unsigned char> d_rgb(colour ? 3 * (size_t)npx : 1, 0), need(n_cams, 0);
    long long pc[3] = {0, 0, 0};
    std::vector<DepthTri> S(IM_RT_THREADS);
    std::vector<int> Q(IM_RT_THREADS * 4);
    for (int tile = 0; tile < ntiles; ++tile) {
        const long long lo = all ? 0 : off[tile], hi = all ? nt : off[tile + 1];
        unsigned int best[IM_RT_THREADS];
        int ba[IM_RT_THREADS], bb[IM_RT_THREADS], bc[IM_RT_THREADS], bs[IM_RT_THREADS];
        for (int p = 0; p < IM_RT_THREADS; ++p) { best[p] = 0x7f800000u; ba[p] = bb[p] = bc[p] = 0x7fffffff; bs[p] = -1; }
        for (long long b = lo; b < hi; b += IM_RT_THREADS) {
            for (int p = 0; p < IM_RT_THREADS; ++p) {
                const long long i = b + p;
                bool ok = false;
                if (i < hi) {
                    const int t = all ? (int)i : bin[i];
                    ok = setup(t, &S[p]);
                    Q[p * 4] = tris[t * 3]; Q[p * 4 + 1] = tris[t * 3 + 1]; Q[p * 4 + 2] = tris[t * 3 + 2]; Q[p * 4 + 3] = t;
                }
                if (!ok) { S[p].x_lo = 1; S[p].x_hi = 0; }
            }
            const int n = hi - b < IM_RT_THREADS ? (int)(hi - b) : IM_RT_THREADS;
            for (int p = 0; p < IM_RT_THREADS; ++p) {
                const int x = (tile % ntx) * IM_RT_TILE + p % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + p / IM_RT_TILE;
                for (int j = 0; j < n; ++j) {
                    const DepthTri& T = S[j];
                    if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
                    float zf;
                    if (!depth_sample(T, x, y, &zf)) continue;
                    unsigned int bits;
                    std::memcpy(&bits, &zf, 4);
                    const int* q = &Q[j * 4];
                    if (bits < 0x7f800000u && view_better(bits, q[0], q[1], q[2], best[p], ba[p], bb[p], bc[p])) {
                        best[p] = bits; ba[p] = q[0]; bb[p] = q[1]; bc[p] = q[2]; bs[p] = q[3];
                    }
                }
            }
        }
        for (int p = 0; p < IM_RT_THREADS; ++p) {
            const int x = (tile % ntx) * IM_RT_TILE + p % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + p / IM_RT_TILE;
            if (x >= w || y >= h) continue;
            const size_t px = (size_t)y * w + x;
            const int row = bs[p], k = row >= 0 ? facet_cam[row] : -1;
            ++pc[k >= 0 ? 0 : (row >= 0 ? 1 : 2)];
            float val;
            std::memcpy(&val, &best[p], 4);
            d_depth[px] = depth_valid(C, val) ? val : -1.0f;
            prow[px] = row;
            if (k >= 0) {
                DepthTri T;
                setup(row, &T);
                double o[3], sp[6];
                trv_weights(T, x, y, flips[row] != 0, o);
                bake_scaled(facet_uv + 6 * (size_t)row, wh[4 * k], wh[4 * k + 1], wh[4 * k + 2], wh[4 * k + 3], sp);
                trv_source(o, sp, &src[2 * px], &src[2 * px + 1]);
                need[k] = 1;
            } else if (colour) {
                const uint8_t* c = row >= 0 ? cfg->untextured : cfg->background;
                std::memcpy(&d_rgb[3 * px], c, 3);
            }
        }
    }
    g_err = trv_check_needed(images, need.data(), n_cams);
    if (!g_err.empty()) return IMMESH_E_INVALID;
    // k_trv_sample
    *n_batches = 0;
    auto sample = [&](int k_lo, int k_hi, const std::vector<BakeImg>& imgs) {
        for (int i = 0; i < npx; ++i) {
            const int r = prow[i];
            if (r < 0 || facet_cam[r] < k_lo || facet_cam[r] > k_hi) continue;
            bake_bilinear(imgs[facet_cam[r]], src[2 * (size_t)i], src[2 * (size_t)i + 1], &d_rgb[3 * (size_t)i]);
        }
    };
    if (colour) {
        std::vector<BakeImg> himg(n_cams);
        for (int k = 0; k < n_cams; ++k) himg[k] = BakeImg{need[k] ? images[k].data : nullptr, images[k].width, images[k].height, (long long)images[k].pitch};
        if (on_device) {
            sample(0, n_cams - 1, himg);
        } else {
            long long arena_bytes = 0;
            const std::vector<int> start = bake_batches(images, need.data(), n_cams, bake_arena_bytes(cfg->max_image_bytes), &arena_bytes);
            std::vector<unsigned char> arena[2];
            for (size_t bi = 0; bi + 1 < start.size(); ++bi) {
                std::vector<unsigned char>& A = arena[bi & 1];
                A.assign((size_t)arena_bytes, 0);
                long long o = 0;
                int first = -1, last = -1;
                for (int k = start[bi]; k < start[bi + 1]; ++k) {
                    if (!need[k]) continue;
                    const immesh_texture_image& im = images[k];
                    for (int y = 0; y < im.height; ++y) std::memcpy(&A[o + 3LL * im.width * y], im.data + (long long)y * im.pitch, 3 * (size_t)im.width);
                    himg[k] = BakeImg{&A[o], im.width, im.height, 3LL * im.width};
                    o += bake_image_bytes(im);
                    if (first < 0) first = k;
                    last = k;
                }
                sample(first, last, himg);
                ++*n_batches;
            }
        }
    }
    // k_trv_score
    long long e[4] = {0, 0, 0, 0};
    if (truth)
        for (int i = 0; i < npx; ++i)
            if (prow[i] >= 0 && facet_cam[prow[i]] >= 0)
                trv_error(&d_rgb[3 * (size_t)i], truth->data + (long long)(i / w) * truth->pitch + 3 * (i % w), e, e + 3);
    if (rgb) std::memcpy(rgb, d_rgb.data(), 3 * (size_t)npx);
    if (depth) std::memcpy(depth, d_depth.data(), (size_t)npx * sizeof(float));
    if (facet) std::memcpy(facet, prow.data(), (size_t)npx * sizeof(int32_t));
    if (needed) std::memcpy(needed, need.data(), (size_t)n_cams);
    if (counts) {
        long long sampled = 0;
        for (int k = 0; k < n_cams; ++k) sampled += need[k];
        counts[0] = pc[0]; counts[1] = pc[1]; counts[2] = pc[2]; counts[3] = sampled;
        for (int i = 0; i < 4; ++i) counts[4 + i] = e[i];
    }
    return IMMESH_OK;
}
}  // extern "C"
