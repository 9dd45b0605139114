// TEST INFRASTRUCTURE (not product code): the reinforcement's __host__ __device__ bodies (immesh_b200/csrc/reinforce.cuh) run on
// the CPU with the device chain's orchestration: k_rf_pose's camera pose from a frame ring, and the tiled rasteriser -- count pass,
// exclusive scan, fill pass, then every tile's pixels over its bin in batches of IM_RT_THREADS set-ups (k_rf_tile) -- followed by
// the ascending-pixel compaction of k_rf_fcount / k_rf_emit.  The shipped library never links or calls this.
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/reinforce.cuh"

using namespace immesh;

extern "C" {
// poses [n_frames][12] of frames 1..n_frames (has[f - 1] = 0: the frame recorded none); the camera of frame `frame` -> R [9], t [3]
int emu_rf_pose(const double* poses, const int* has, int n_frames, int frame, int win, double* R, double* t) {
    double ring[IM_RF_RING][12];
    int ring_frame[IM_RF_RING];
    std::memset(ring, 0, sizeof(ring));
    std::memset(ring_frame, 0, sizeof(ring_frame));
    for (int f = 1; f <= n_frames && f < frame + 1; ++f) {   // what the frames' transform kernels left behind by frame `frame`
        if (!has[f - 1]) continue;
        std::memcpy(ring[f % IM_RF_RING], poses + (size_t)(f - 1) * 12, 12 * sizeof(double));
        ring_frame[f % IM_RF_RING] = f;
    }
    rf_avr_pose(ring, ring_frame, frame, win, R, t);
    return 0;
}
// cam = fx fy cx cy z_near z_far R[9] t[3]; verts [nv][3]; tris [nt][3] (all live).  Outputs as immesh_mesh_reinforced_cloud:
// depth [h][w], points [n][3], pixel [n]; returns n.  *bin_entries: bin entries of the count pass.
int emu_rf_raster(const double* cam, int w, int h, const float* verts, const int* tris, int nt, float* depth, float* points, int* pixel, long long* bin_entries) {
    DepthCam C;
    C.fx = cam[0]; C.fy = cam[1]; C.cx = cam[2]; C.cy = cam[3]; C.z_near = cam[4]; C.z_far = cam[5];
    for (int i = 0; i < 9; ++i) C.R[i] = cam[6 + i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam[15 + i];
    C.w = w; C.h = h;
    auto vtx = [&](int i) { return make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f); };
    const int ntx = (w + IM_RT_TILE - 1) / IM_RT_TILE, nty = (h + IM_RT_TILE - 1) / IM_RT_TILE, ntiles = ntx * nty;
    // k_rf_count
    std::vector<int> cnt(ntiles, 0), off(ntiles + 1, 0);
    for (int t = 0; t < nt; ++t) {
        DepthTri T;
        if (!depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), &T)) continue;
        for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
            for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) ++cnt[ty * ntx + tx];
    }
    // k_rf_scan
    for (int i = 0; i < ntiles; ++i) off[i + 1] = off[i] + cnt[i];
    *bin_entries = off[ntiles];
    // k_rf_fill (the device fills a bin in any order: reversed here)
    std::vector<int> cur(off.begin(), off.end() - 1), bin(off[ntiles] > 0 ? off[ntiles] : 1);
    for (int t = nt - 1; t >= 0; --t) {
        DepthTri T;
        if (!depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), &T)) continue;
        for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
            for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) bin[cur[ty * ntx + tx]++] = t;
    }
    // k_rf_tile
    std::vector<unsigned int> bits((size_t)w * h, 0x7f800000u);
    std::vector<DepthTri> S(IM_RT_THREADS);
    for (int tile = 0; tile < ntiles; ++tile) {
        const int lo = off[tile], hi = off[tile + 1];
        std::vector<unsigned int> acc(IM_RT_THREADS, 0x7f800000u);
        for (int b = lo; b < hi; b += IM_RT_THREADS) {
            for (int k = 0; k < IM_RT_THREADS; ++k) {
                const int i = b + k;
                const int t = i < hi ? bin[i] : -1;
                if (t < 0 || !depth_tri_setup(C, vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2]), &S[k])) { S[k].x_lo = 1; S[k].x_hi = 0; }
            }
            const int nb = hi - b < IM_RT_THREADS ? hi - b : IM_RT_THREADS;
            for (int k = 0; k < IM_RT_THREADS; ++k) {
                const int x = (tile % ntx) * IM_RT_TILE + k % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + k / IM_RT_TILE;
                acc[k] = rt_pixel_min(S.data(), nb, x, y, acc[k]);
            }
        }
        for (int k = 0; k < IM_RT_THREADS; ++k) {
            const int x = (tile % ntx) * IM_RT_TILE + k % IM_RT_TILE, y = (tile / ntx) * IM_RT_TILE + k / IM_RT_TILE;
            if (x < w && y < h) bits[(size_t)y * w + x] = acc[k];
        }
    }
    // k_rf_fcount / k_rf_scan / k_rf_emit: ascending pixel order
    int n = 0;
    for (int i = 0; i < w * h; ++i) {
        float val;
        std::memcpy(&val, &bits[i], 4);
        const bool ok = depth_valid(C, val);
        depth[i] = ok ? val : -1.0f;
        if (!ok) continue;
        depth_unproject(C, i % w, i / w, val, points + (size_t)n * 3);
        pixel[n++] = i;
    }
    return n;
}
}  // extern "C"
