// TEST INFRASTRUCTURE (not product code): the shaded view's __host__ __device__ bodies (immesh_b200/csrc/reinforce.cuh) run on the
// CPU with the device chain's orchestration: the binning passes of the depth image at the view's positions (count, exclusive scan,
// fill in reverse slot order, or every slot when the bins overflow), k_view_zrange's automatic z range, then every tile's pixels over
// its bin in batches of IM_RT_THREADS set-ups with the triple tie-break and the shading of the winner (k_view_tile), and the queued
// view's camera (k_rf_pose's rf_frame_pose).  The shipped library never links or calls this.
#include <cmath>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/reinforce.cuh"

using namespace immesh;

extern "C" {
// cam = fx fy cx cy z_near z_far R[9] t[3]; verts [nv][3] float; smooth [nv][3] / flags [nv] (or NULL); tris [nt][3] (all live, in
// slot order); zr = the caller's range or NaN, NaN; bin_cap: bin entries beyond it walk every slot.  Outputs as
// immesh_mesh_render_view: rgba [h][w][4], depth [h][w]; *bin_entries: bin entries of the count pass, *overflow: the bins overflowed.
int emu_view_render(const double* cam, int w, int h, const float* verts, const double* smooth, const unsigned char* flags, int nv, const int* tris, int nt,
                    int pos_mode, int color, const double* zr_in, long long bin_cap, unsigned char* rgba, float* depth, long long* bin_entries, int* overflow) {
    DepthCam C;
    C.fx = cam[0]; C.fy = cam[1]; C.cx = cam[2]; C.cy = cam[3]; C.z_near = cam[4]; C.z_far = cam[5];
    for (int i = 0; i < 9; ++i) C.R[i] = cam[6 + i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam[15 + i];
    C.w = w; C.h = h;
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    auto vtx = [&](int i) { return view_vertex(vpos.data(), smooth, flags, pos_mode, i); };
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
    *bin_entries = off[ntiles];
    const bool all = off[ntiles] > bin_cap;
    *overflow = all ? 1 : 0;
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
    // k_view_zrange
    float zr[2] = {0.f, 0.f};
    if (color) {
        if (std::isnan(zr_in[0]) && std::isnan(zr_in[1])) {
            unsigned int lo = 0xffffffffu, hi = 0u;
            for (int t = 0; t < nt * 3; ++t) {
                const unsigned int u = view_ordered(vtx(tris[t]).z);
                lo = u < lo ? u : lo; hi = u > hi ? u : hi;
            }
            zr[0] = view_unordered(lo); zr[1] = view_unordered(hi);
        } else {
            zr[0] = (float)zr_in[0]; zr[1] = (float)zr_in[1];
        }
    }
    // k_view_tile
    std::vector<DepthTri> S(IM_RT_THREADS);
    std::vector<int> Q(IM_RT_THREADS * 4);
    for (int tile = 0; tile < ntiles; ++tile) {
        const long long lo = all ? 0 : off[tile], hi = all ? nt : off[tile + 1];
        unsigned int best[IM_RT_THREADS];
        int ba[IM_RT_THREADS], bb[IM_RT_THREADS], bc[IM_RT_THREADS], bs[IM_RT_THREADS];
        for (int k = 0; k < IM_RT_THREADS; ++k) { best[k] = 0x7f800000u; ba[k] = bb[k] = bc[k] = 0x7fffffff; bs[k] = -1; }
        for (long long b = lo; b < hi; b += IM_RT_THREADS) {
            for (int k = 0; k < IM_RT_THREADS; ++k) {
                const long long i = b + k;
                bool ok = false;
                if (i < hi) {
                    const int t = all ? (int)i : bin[i];
                    ok = setup(t, &S[k]);
                    Q[k * 4] = tris[t * 3]; Q[k * 4 + 1] = tris[t * 3 + 1]; Q[k * 4 + 2] = tris[t * 3 + 2]; Q[k * 4 + 3] = t;
                }
                if (!ok) { S[k].x_lo = 1; S[k].x_hi = 0; }
            }
            const int n = hi - b < IM_RT_THREADS ? (int)(hi - b) : IM_RT_THREADS;
            for (int k = 0; k < IM_RT_THREADS; ++k) {
                const int x = (tile % ntx) * IM_RT_TILE + k % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + k / IM_RT_TILE;
                for (int j = 0; j < n; ++j) {
                    const DepthTri& T = S[j];
                    if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
                    float zf;
                    if (!depth_sample(T, x, y, &zf)) continue;
                    unsigned int bits;
                    std::memcpy(&bits, &zf, 4);
                    const int* q = &Q[j * 4];
                    if (bits < 0x7f800000u && view_better(bits, q[0], q[1], q[2], best[k], ba[k], bb[k], bc[k])) {
                        best[k] = bits; ba[k] = q[0]; bb[k] = q[1]; bc[k] = q[2]; bs[k] = q[3];
                    }
                }
            }
        }
        for (int k = 0; k < IM_RT_THREADS; ++k) {
            const int x = (tile % ntx) * IM_RT_TILE + k % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + k / IM_RT_TILE;
            if (x >= w || y >= h) continue;
            const size_t px = (size_t)y * w + x;
            float val;
            std::memcpy(&val, &best[k], 4);
            depth[px] = depth_valid(C, val) ? val : -1.0f;
            uchar4 c = make_uchar4(0, 0, 0, 255);
            if (bs[k] >= 0) {
                const int t = bs[k];
                const float4 p[3] = {vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2])};
                DepthTri T;
                depth_tri_setup(C, p[0], p[1], p[2], &T);
                double col[3][3];
                for (int v = 0; v < 3; ++v) view_color(color, p[v].z, zr[0], zr[1], col[v]);
                c = view_shade(T, x, y, p, col, C.t);
            }
            rgba[px * 4] = c.x; rgba[px * 4 + 1] = c.y; rgba[px * 4 + 2] = c.z; rgba[px * 4 + 3] = c.w;
        }
    }
    return 0;
}
// the height colour of each z [n] with the range lo, hi (floats) -> rgb [n][3]
int emu_view_heat(const float* z, int n, float lo, float hi, unsigned char* rgb) {
    for (int i = 0; i < n; ++i) view_heat(z[i], lo, hi, rgb + (size_t)i * 3);
    return 0;
}
// poses [n_frames][12] of frames 1..n_frames (has[f - 1] = 0: none); the queued camera of frame `frame` by source mode -> R [9], t [3]
int emu_view_pose(const double* poses, const int* has, int n_frames, int frame, int win, int mode, const double* R_in, const double* t_in, double* R, double* t) {
    double ring[IM_RF_RING][12];
    int ring_frame[IM_RF_RING];
    std::memset(ring, 0, sizeof(ring));
    std::memset(ring_frame, 0, sizeof(ring_frame));
    for (int f = 1; f <= n_frames && f < frame + 1; ++f) {
        if (!has[f - 1]) continue;
        std::memcpy(ring[f % IM_RF_RING], poses + (size_t)(f - 1) * 12, 12 * sizeof(double));
        ring_frame[f % IM_RF_RING] = f;
    }
    rf_frame_pose(ring, ring_frame, frame, win, mode, R_in, t_in, R, t);
    return 0;
}
}  // extern "C"
