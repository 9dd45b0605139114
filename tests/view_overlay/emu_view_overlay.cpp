// TEST INFRASTRUCTURE (not product code): the queued view's overlays (immesh_b200/csrc/view_overlay.cuh) run on the CPU with the
// device chain's orchestration: k_ov_begin's per-frame step over the frames since the overlay was set (trajectory ring, camera ring,
// frustum), the per-pixel keys of k_ov_points and k_ov_lines (the minimum over every fragment, as the atomics leave it), the binning
// passes at the view's positions (the wireframe's widened boxes with `wire`; fill in reverse slot order, or every slot when the bins
// overflow), then every tile's pixels over its bin in batches of IM_RT_THREADS set-ups (k_view_tile or k_view_wire_tile) with the
// keys resolved against the mesh's winner.  The shipped library never links or calls this.
#include <cmath>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/view_overlay.cuh"

using namespace immesh;

extern "C" {
// cam = fx fy cx cy z_near z_far R[9] t[3]; verts [nv][3] float; tris [nt][3] (all live, ascending, in slot order); zr = the caller's
// range or NaN, NaN; bin_cap: bin entries beyond it walk every slot; wire: the wireframe instead of the faces.
// Overlays: scan [ns][3] (frame nf's world points), rf [nr][3] (its reinforced points), sizes 0 = off; axis_and_grid; frames 1..nf
// with poses [nf][12] (rot_end row-major, pos_end; has[f - 1] = 0: a world-frame push without one) and pose_t [nf][3]; the overlay
// set before frame path_from; camera_size; path_w, path_cap.  Outputs: rgba [h][w][4], depth [h][w], keys [h][w] (the overlay keys
// or NULL), *bin_entries, *overflow.
int emu_ov_render(const double* cam, int w, int h, const float* verts, int nv, const int* tris, int nt, int color, const double* zr_in,
                  long long bin_cap, int wire, const float* scan, int ns, int scan_size, const float* rf, int nr, int rf_size, int axis_and_grid,
                  const double* poses, const int* has, const double* pose_t, int nf, int path_from, double camera_size, int path_w, int path_cap,
                  unsigned char* rgba, float* depth, unsigned long long* keys_out, long long* bin_entries, int* overflow) {
    DepthCam C;
    C.fx = cam[0]; C.fy = cam[1]; C.cx = cam[2]; C.cy = cam[3]; C.z_near = cam[4]; C.z_far = cam[5];
    for (int i = 0; i < 9; ++i) C.R[i] = cam[6 + i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam[15 + i];
    C.w = w; C.h = h;
    const int npx = w * h;
    // the overlay's buffers and k_ov_begin over the frames since it was set
    std::vector<double> path((size_t)(path_w > 0 ? path_cap : 1) * 3), fr(33);
    std::vector<unsigned long long> key(npx, OV_NONE);
    int path_n = 0, frustum_on = 0;
    ViewOverlay O = {};
    O.on = 1; O.wire = wire; O.scan_size = scan_size; O.reinforced_size = rf_size; O.axis_and_grid = axis_and_grid; O.path_width = path_w;
    O.path_cap = path_w > 0 ? path_cap : 1; O.npx = npx; O.camera_size = camera_size;
    O.path = (double (*)[3])path.data(); O.path_n = &path_n; O.frustum = (double (*)[3])fr.data(); O.frustum_on = &frustum_on; O.key = key.data();
    double ring[IM_RF_RING][12];
    int ring_frame[IM_RF_RING];
    std::memset(ring, 0, sizeof(ring));
    std::memset(ring_frame, 0, sizeof(ring_frame));
    for (int f = 1; f <= nf; ++f) {
        if (has[f - 1]) {   // k_transform_full
            std::memcpy(ring[f % IM_RF_RING], poses + (size_t)(f - 1) * 12, 12 * sizeof(double));
            ring_frame[f % IM_RF_RING] = f;
        }
        if (f >= path_from) ov_begin_frame(O, f, pose_t + (size_t)(f - 1) * 3, ring, ring_frame);
    }
    // k_ov_points
    const int n_scan = scan_size > 0 && nf >= 2 ? ns : 0, n_rf = rf_size > 0 ? nr : 0;
    for (int i = 0; i < n_scan + n_rf; ++i) {
        const bool sc = i < n_scan;
        const int j = sc ? i : i - n_scan, layer = sc ? OV_SCAN : OV_REINFORCED;
        const float* q = (sc ? scan : rf) + (size_t)j * 3;
        const double p[3] = {(double)q[0], (double)q[1], (double)q[2]};
        ov_point_raster(C, p, sc ? scan_size : rf_size, [&](int x, int y, float zf) {
            unsigned long long& k = key[(size_t)y * w + x];
            const unsigned long long v = ov_key(zf, layer, (unsigned)j);
            k = v < k ? v : k;
        });
    }
    // k_ov_lines (a warp's 32 lanes split the major coordinates; together they cover them all)
    const int nseg = (axis_and_grid ? OV_N_AXIS + OV_N_GRID : 0) + (frustum_on ? OV_N_CAMERA : 0) + std::max(ov_path_kept(O, path_n) - 1, 0);
    for (int i = 0; i < nseg; ++i) {
        int layer, idx, width;
        double p0[3], p1[3];
        OvSeg S;
        if (!ov_line(O, frustum_on, path_n, i, &layer, &idx, &width, p0, p1) || !ov_seg_setup(C, p0, p1, &S)) continue;
        for (int lane = 0; lane < 32; ++lane)
            ov_seg_raster(C, S, width, lane, 32, [&](int x, int y, float zf, double) {
                unsigned long long& k = key[(size_t)y * w + x];
                const unsigned long long v = ov_key(zf, layer, (unsigned)idx);
                k = v < k ? v : k;
            });
    }
    if (keys_out) std::memcpy(keys_out, key.data(), (size_t)npx * sizeof(unsigned long long));
    // the mesh: k_rf_count / k_rf_scan / k_rf_fill at the set-up of the mode
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    auto vtx = [&](int i) { return vpos[i]; };
    auto setup = [&](int t, DepthTri* T, int4* fb) {
        const float4 p0 = vtx(tris[t * 3]), p1 = vtx(tris[t * 3 + 1]), p2 = vtx(tris[t * 3 + 2]);
        return wire ? view_wire_setup(C, p0, p1, p2, T, fb) : depth_tri_setup(C, p0, p1, p2, T);
    };
    const int ntx = (w + IM_RT_TILE - 1) / IM_RT_TILE, nty = (h + IM_RT_TILE - 1) / IM_RT_TILE, ntiles = ntx * nty;
    std::vector<long long> cnt(ntiles, 0), off(ntiles + 1, 0);
    for (int t = 0; t < nt; ++t) {
        DepthTri T;
        int4 fb;
        if (!setup(t, &T, &fb)) continue;
        for (int ty = T.y_lo / IM_RT_TILE; ty <= T.y_hi / IM_RT_TILE; ++ty)
            for (int tx = T.x_lo / IM_RT_TILE; tx <= T.x_hi / IM_RT_TILE; ++tx) ++cnt[ty * ntx + tx];
    }
    for (int i = 0; i < ntiles; ++i) off[i + 1] = off[i] + cnt[i];
    *bin_entries = off[ntiles];
    const bool all = off[ntiles] > bin_cap;
    *overflow = all ? 1 : 0;
    std::vector<int> bin(all || off[ntiles] == 0 ? 1 : (size_t)off[ntiles]);
    if (!all) {
        std::vector<long long> cur(off.begin(), off.end() - 1);
        for (int t = nt - 1; t >= 0; --t) {
            DepthTri T;
            int4 fb;
            if (!setup(t, &T, &fb)) continue;
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
    // k_view_tile / k_view_wire_tile
    std::vector<DepthTri> S(IM_RT_THREADS);
    std::vector<int4> FB(IM_RT_THREADS);
    std::vector<int> Q(IM_RT_THREADS * 4);
    for (int tile = 0; tile < ntiles; ++tile) {
        const long long lo = all ? 0 : off[tile], hi = all ? nt : off[tile + 1];
        unsigned int face[IM_RT_THREADS], best[IM_RT_THREADS];
        int ba[IM_RT_THREADS], bb[IM_RT_THREADS], bc[IM_RT_THREADS], be[IM_RT_THREADS], bs[IM_RT_THREADS];
        for (int k = 0; k < IM_RT_THREADS; ++k) { face[k] = best[k] = 0x7f800000u; ba[k] = bb[k] = bc[k] = 0x7fffffff; be[k] = 3; bs[k] = -1; }
        for (long long b = lo; b < hi; b += IM_RT_THREADS) {
            for (int k = 0; k < IM_RT_THREADS; ++k) {
                const long long i = b + k;
                bool ok = false;
                if (i < hi) {
                    const int t = all ? (int)i : bin[i];
                    ok = setup(t, &S[k], &FB[k]);
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
                    const int* q = &Q[j * 4];
                    if (wire) {
                        view_wire_pixel(T, FB[j], q[0], q[1], q[2], q[3], x, y, &face[k], &best[k], &ba[k], &bb[k], &bc[k], &be[k], &bs[k]);
                        continue;
                    }
                    float zf;
                    if (!depth_sample(T, x, y, &zf)) continue;
                    unsigned int bits;
                    std::memcpy(&bits, &zf, 4);
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
            std::memcpy(&val, wire ? &face[k] : &best[k], 4);
            depth[px] = depth_valid(C, val) ? val : -1.0f;
            uchar4 c = make_uchar4(0, 0, 0, 255);
            if (ov_over_mesh(key[px], best[k])) {
                c = ov_color(key[px]);
            } else if (bs[k] >= 0) {
                const int t = bs[k];
                const float4 p[3] = {vtx(tris[t * 3]), vtx(tris[t * 3 + 1]), vtx(tris[t * 3 + 2])};
                double col[3][3];
                for (int v = 0; v < 3; ++v) view_color(color, p[v].z, zr[0], zr[1], col[v]);
                if (wire) {
                    c = view_wire_color(C, p, col, be[k], x, y);
                } else {
                    DepthTri T;
                    depth_tri_setup(C, p[0], p[1], p[2], &T);
                    c = view_shade(T, x, y, p, col, C.t);
                }
            }
            rgba[px * 4] = c.x; rgba[px * 4 + 1] = c.y; rgba[px * 4 + 2] = c.z; rgba[px * 4 + 3] = c.w;
        }
    }
    return 0;
}
// the frustum's 11 world vertices of rot_end R [9], pos_end t [3] at camera size cs -> out [11][3]
int emu_ov_frustum(const double* R, const double* t, double cs, double* out) {
    ov_frustum(R, t, cs, (double (*)[3])out);
    return 0;
}
}  // extern "C"
