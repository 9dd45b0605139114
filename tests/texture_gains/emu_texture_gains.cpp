// TEST INFRASTRUCTURE (not product code): immesh_mesh_texture_gains' __host__ __device__ bodies (immesh_b200/csrc/texture_gains_core.cuh,
// texture_bake_core.cuh, texture_core.cuh, reinforce.cuh), its argument check and its host solve run on the CPU with the device call's
// orchestration: the chosen side per batch (k_tg_chosen), then per observer camera in index order the binning passes at the rule's
// positions (count, exclusive scan, fill in reverse slot order, or every slot when the bins overflow), every tile's pixels over its bin
// in batches of IM_RT_THREADS set-ups with the view's tie-break (k_tex_tile: covered and won pixels per row), the per-row "seen" test
// and samples into a dense row per chosen camera (k_tg_observe), its compaction in ascending camera (k_tg_compact), and the solve.  Host
// images go batch by batch (bake_batches), each batch's images packed into an arena at pitch 3 width as tex_upload_batches lays them
// out: one batch serves both phases, more batches are swept twice.  Also immesh_texture_apply_gains' host loop.  The shipped library
// never links or calls this.
#include <cstring>
#include <string>
#include <vector>

#include "../../immesh_b200/csrc/texture_gains_core.cuh"

using namespace immesh;

static std::string g_err;

extern "C" {
const char* emu_texture_gains_error() { return g_err.c_str(); }

// verts [nv][3] float; smooth [nv][3] / flags [nv] (or NULL); tris [nt][3] ascending triples and flips [nt], every one live, in the rows'
// (snapshot) order; bin_cap: bin entries beyond it walk every slot; shard_n: the handle's shards.  The other arguments and outputs as
// immesh_mesh_texture_gains'; *n_batches: the host-image batches (0 for device images).
int emu_texture_gains(const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device, const int32_t* facet_cam,
                      const float* facet_uv, int64_t n_facets, const immesh_texture_gains_config* cfg, const float* verts, const double* smooth,
                      const unsigned char* flags, int nv, const int* tris, const int* flips, int nt, long long bin_cap, int shard_n, double* gains,
                      int32_t* pair_cam, int64_t* pair_sums, int64_t* n_pairs, int64_t* counts, int* n_batches) {
    std::vector<unsigned char> have;
    g_err = tg_check(cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, cfg, gains, nt, shard_n, have);
    if (!g_err.empty()) return IMMESH_E_INVALID;
    const immesh_texture_config& sel = cfg->sel;
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    auto vtx = [&](int i) { return view_vertex(vpos.data(), smooth, flags, sel.positions, i); };
    const TexRule rule = tex_rule(sel);
    std::vector<BakeImg> himg(n_cams, BakeImg{nullptr, 1, 1, 3});
    std::vector<unsigned char> chosen((size_t)(3 * IM_TG_POINTS) * (nt > 0 ? nt : 1), 0);
    std::vector<long long> prow((size_t)IM_TG_SUMS * n_cams, 0), ps;
    std::vector<int> pc;
    long long used = 0, clipped = 0, pixels = 0;
    int n_obs = 0;
    auto scale = [&](int k, const float* uv, double* p) { bake_scaled(uv, images[k].width, images[k].height, cams[k].width, cams[k].height, p); };
    // k_tg_chosen
    auto chosen_side = [&](int k_lo, int k_hi) {
        for (int i = 0; i < nt; ++i) {
            const int c = facet_cam[i];
            if (c < k_lo || c > k_hi) continue;
            double p[6];
            scale(c, facet_uv + 6 * (size_t)i, p);
            tg_sample(himg[c], p, &chosen[(size_t)(3 * IM_TG_POINTS) * i]);
        }
    };
    // one observer pass: binning, k_tex_tile, k_tg_observe, k_tg_compact
    auto pass = [&](int k) {
        const DepthCam C = tex_camera(cams[k], sel.z_near, sel.z_far);
        const int w = C.w, h = C.h;
        ++n_obs;
        pixels += (long long)w * h;
        auto setup = [&](int t, DepthTri* T) { return depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), T); };
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
        std::vector<int> won(nt > 0 ? nt : 1, 0), cov(won);
        std::vector<DepthTri> S(IM_RT_THREADS);
        std::vector<int> Q(IM_RT_THREADS * 4);
        for (int tile = 0; tile < ntiles; ++tile) {
            const long long lo = all ? 0 : off[tile], hi = all ? nt : off[tile + 1];
            unsigned int best[IM_RT_THREADS];
            int ba[IM_RT_THREADS], bb[IM_RT_THREADS], bc[IM_RT_THREADS], brow[IM_RT_THREADS];
            for (int p = 0; p < IM_RT_THREADS; ++p) { best[p] = 0x7f800000u; ba[p] = bb[p] = bc[p] = 0x7fffffff; brow[p] = -1; }
            for (long long b = lo; b < hi; b += IM_RT_THREADS) {
                for (int p = 0; p < IM_RT_THREADS; ++p) {
                    const long long i = b + p;
                    bool ok = false;
                    if (i < hi) {
                        const int t = all ? (int)i : bin[i];
                        ok = setup(t, &S[p]);
                        Q[p * 4] = tris[t * 3]; Q[p * 4 + 1] = tris[t * 3 + 1]; Q[p * 4 + 2] = tris[t * 3 + 2]; Q[p * 4 + 3] = ok ? t : -1;
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
                        if (bits >= 0x7f800000u) continue;
                        const int* q = &Q[j * 4];
                        ++cov[q[3]];
                        if (view_better(bits, q[0], q[1], q[2], best[p], ba[p], bb[p], bc[p])) { best[p] = bits; ba[p] = q[0]; bb[p] = q[1]; bc[p] = q[2]; brow[p] = q[3]; }
                    }
                }
            }
            for (int p = 0; p < IM_RT_THREADS; ++p)
                if (brow[p] >= 0) ++won[brow[p]];
        }
        for (int i = 0; i < nt; ++i) {
            const int fc = facet_cam[i];
            if (won[i] < 1 || fc < 0 || fc == k) continue;
            float4 q[3];
            tex_corners(vtx(tris[i * 3]), vtx(tris[i * 3 + 1]), vtx(tris[i * 3 + 2]), flips[i] != 0, q);
            double e2;
            if (!tex_seen(C, q, won[i], cov[i], rule, &e2)) continue;
            float uv[6];
            tex_uv(C, q, uv);
            double p[6];
            scale(k, uv, p);
            unsigned char ok[3 * IM_TG_POINTS];
            tg_sample(himg[k], p, ok);
            int sum[IM_TG_SUMS] = {0, 0, 0, 0, 0, 0, 0}, cl = 0;
            tg_accumulate(ok, &chosen[(size_t)(3 * IM_TG_POINTS) * i], sum, &cl);
            clipped += cl;
            used += sum[0];
            for (int v = 0; sum[0] > 0 && v < IM_TG_SUMS; ++v) prow[(size_t)IM_TG_SUMS * fc + v] += sum[v];
        }
        for (int c = 0; c < n_cams; ++c) {
            long long* e = &prow[(size_t)IM_TG_SUMS * c];
            if (!e[0]) continue;
            pc.push_back(k); pc.push_back(c);
            for (int v = 0; v < IM_TG_SUMS; ++v) { ps.push_back(e[v]); e[v] = 0; }
        }
    };
    auto observe = [&](int k_lo, int k_hi) {
        for (int k = k_lo; nt > 0 && k <= k_hi; ++k)
            if (have[k]) pass(k);
    };
    *n_batches = 0;
    if (on_device) {
        for (int k = 0; k < n_cams; ++k)
            if (have[k]) himg[k] = BakeImg{images[k].data, images[k].width, images[k].height, (long long)images[k].pitch};
        chosen_side(0, n_cams - 1);
        observe(0, n_cams - 1);
    } else {
        std::vector<unsigned char> want(n_cams, 0);
        if (nt > 0) want = have;
        long long arena_bytes = 0;
        const std::vector<int> start = bake_batches(images, want.data(), n_cams, bake_arena_bytes(cfg->max_image_bytes), &arena_bytes);
        std::vector<unsigned char> arena[2];
        const int sweeps = start.size() == 2 ? 1 : 2;
        *n_batches = (int)start.size() - 1;
        for (int sw = 0; sw < sweeps; ++sw)
            for (size_t bi = 0; bi + 1 < start.size(); ++bi) {
                std::vector<unsigned char>& A = arena[bi & 1];
                A.assign((size_t)arena_bytes, 0);
                long long o = 0;
                int first = -1, last = -1;
                for (int k = start[bi]; k < start[bi + 1]; ++k) {
                    if (!want[k]) continue;
                    const immesh_texture_image& im = images[k];
                    for (int y = 0; y < im.height; ++y) std::memcpy(&A[o + 3LL * im.width * y], im.data + (long long)y * im.pitch, 3 * (size_t)im.width);
                    himg[k] = BakeImg{&A[o], im.width, im.height, 3LL * im.width};
                    o += bake_image_bytes(im);
                    if (first < 0) first = k;
                    last = k;
                }
                if (sweeps == 1 || sw == 0) chosen_side(first, last);
                if (sweeps == 1 || sw == 1) observe(first, last);
            }
    }
    const long long np = (long long)pc.size() / 2;
    int iters = 0, left = 0;
    auto fill_counts = [&]() {
        if (n_pairs) *n_pairs = np;
        if (counts) {
            counts[0] = np; counts[1] = used; counts[2] = clipped; counts[3] = n_obs; counts[4] = left; counts[5] = iters; counts[6] = pixels; counts[7] = 0;
        }
    };
    if (np > cfg->max_pairs) {
        fill_counts();
        g_err = "more pairs than max_pairs";
        return IMMESH_E_CAPACITY;
    }
    tg_solve(n_cams, pc.data(), ps.data(), np, cfg->sigma_n, cfg->sigma_g, gains, &iters, &left);
    if (pair_cam && np > 0) std::memcpy(pair_cam, pc.data(), 2 * (size_t)np * sizeof(int32_t));
    if (pair_sums && np > 0) std::memcpy(pair_sums, ps.data(), (size_t)IM_TG_SUMS * np * sizeof(int64_t));
    fill_counts();
    return IMMESH_OK;
}

// immesh_texture_apply_gains' argument check and host loop
int emu_apply_gains(const immesh_texture_image* in, const immesh_texture_image* out, int n, int on_device, const double* gains) {
    g_err = tg_apply_check(in, out, n, on_device, gains);
    if (!g_err.empty()) return IMMESH_E_INVALID;
    for (int k = 0; k < n; ++k) {
        if (!in[k].data) continue;
        unsigned char* o = const_cast<unsigned char*>(out[k].data);
        for (int y = 0; y < in[k].height; ++y)
            for (int x = 0; x < 3 * in[k].width; ++x) o[y * out[k].pitch + x] = tg_apply(in[k].data[y * in[k].pitch + x], gains[3 * k + x % 3]);
    }
    return IMMESH_OK;
}
}  // extern "C"
