// TEST INFRASTRUCTURE (not product code): immesh_mesh_texture_select's __host__ __device__ bodies (immesh_b200/csrc/texture_core.cuh,
// reinforce.cuh) run on the CPU with the device chain's orchestration: per camera in index order the binning passes at the rule's
// positions (count, exclusive scan, fill in reverse slot order, or every slot when the bins overflow), every tile's pixels over its bin
// in batches of IM_RT_THREADS set-ups with the view's tie-break (k_tex_tile: covered samples per facet, one won pixel for the winner),
// then the per-facet "seen" test with the nearest camera kept by a strict < (k_tex_facet), and the rows (k_tex_rows).  The shipped
// library never links or calls this.
#include <cmath>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/texture_core.cuh"

using namespace immesh;

extern "C" {
// verts [nv][3] float; smooth [nv][3] / flags [nv] (or NULL); tris [nt][3] ascending triples and flips [nt] (all live, the rows'
// order); bin_cap: bin entries beyond it walk every slot.  Outputs as immesh_mesh_texture_select: facet_cam [nt], facet_uv [nt][6]
// (untextured rows untouched), facet_px [nt][2], counts [4]; overflow [n_cams]: the bins of camera k overflowed.
int emu_texture_select(const immesh_texture_camera* cams, int n_cams, const immesh_texture_config* cfg, const float* verts, const double* smooth,
                       const unsigned char* flags, int nv, const int* tris, const int* flips, int nt, long long bin_cap, int* facet_cam, float* facet_uv,
                       int* facet_px, long long* counts, int* overflow) {
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    auto vtx = [&](int i) { return view_vertex(vpos.data(), smooth, flags, cfg->positions, i); };
    auto corners = [&](int t, float4* q) { tex_corners(vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), flips[t] != 0, q); };
    std::vector<int> won(nt > 0 ? nt : 1, 0), cov(nt > 0 ? nt : 1, 0), best_cam(nt > 0 ? nt : 1, -1), best_won(won), best_cov(won);
    std::vector<double> best_e2(nt > 0 ? nt : 1, INFINITY);
    const TexRule rule = tex_rule(*cfg);
    long long pixels = 0;
    for (int k = 0; k < n_cams; ++k) {
        const DepthCam C = tex_camera(cams[k], cfg->z_near, cfg->z_far);
        const int w = C.w, h = C.h;
        pixels += (long long)w * h;
        auto setup = [&](int t, DepthTri* T) { return depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), T); };
        const int ntx = (w + IM_RT_TILE - 1) / IM_RT_TILE, nty = (h + IM_RT_TILE - 1) / IM_RT_TILE, ntiles = ntx * nty;
        // k_rf_count / k_rf_scan
        std::vector<long long> cnt(ntiles, 0), off(ntiles + 1, 0);
        for (int t = 0; t < nt; ++t) {
            DepthTri T;
            if (!setup(t, &T)) continue;
            for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
                for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) ++cnt[ty * ntx + tx];
        }
        for (int i = 0; i < ntiles; ++i) off[i + 1] = off[i] + cnt[i];
        const bool all = off[ntiles] > bin_cap;
        overflow[k] = all ? 1 : 0;
        // k_rf_fill (the device fills a bin in any order: reversed here)
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
        // k_tex_tile
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
        // k_tex_facet
        for (int t = 0; t < nt; ++t) {
            const int wn = won[t], cv = cov[t];
            won[t] = 0; cov[t] = 0;
            if (wn < 1) continue;
            float4 q[3];
            corners(t, q);
            double e2;
            if (tex_seen(C, q, wn, cv, rule, &e2) && e2 < best_e2[t]) { best_e2[t] = e2; best_cam[t] = k; best_won[t] = wn; best_cov[t] = cv; }
        }
    }
    // k_tex_rows
    long long c[3] = {0, 0, 0};
    std::vector<int> used(n_cams, 0);
    for (int t = 0; t < nt; ++t) {
        const int k = best_cam[t];
        facet_cam[t] = k;
        facet_px[2 * t] = k >= 0 ? best_won[t] : 0;
        facet_px[2 * t + 1] = k >= 0 ? best_cov[t] : 0;
        if (k < 0) { ++c[1]; continue; }
        float4 q[3];
        corners(t, q);
        tex_uv(tex_camera(cams[k], cfg->z_near, cfg->z_far), q, facet_uv + 6 * (size_t)t);
        ++c[0];
        if (!used[k]) { used[k] = 1; ++c[2]; }
    }
    counts[0] = c[0]; counts[1] = c[1]; counts[2] = c[2]; counts[3] = pixels;
    return 0;
}
}  // extern "C"
