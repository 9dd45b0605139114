// TEST INFRASTRUCTURE (not product code): the texturing queued behind every frame (immesh_mesh_texture_enable / _rows) with its
// __host__ __device__ bodies (immesh_b200/csrc/texture_core.cuh, the rasteriser of reinforce.cuh) in the device stage's orchestration:
// per frame the camera (k_txo_cam: the caller's, the rig on the sensor pose, or none), every pixel over the live slots with the view's
// tie-break counting covered and won pixels per slot (k_tex_tile with the slot as the count index), the per-slot update (k_txo_update);
// the state grown along the pool (txo_state_migrate: fresh slots, the allocated records copied); then the rows in the caller's order
// (k_txo_rows) and the frames any record holds, ascending (k_txo_keys, the sort and k_txo_unique).  The shipped library never links or
// calls this.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/texture_core.cuh"

using namespace immesh;

extern "C" {
// verts [nv][3] float (the positions never move); per frame f (n_frames of them): number[f], kind[f] (0 no camera, 1 the rig on
// pose[f], 2 the caller's camera pose[f]; pose[f] = R row-major then t), cap[f] (the pool's capacity from that frame on, never
// smaller), and the slots live at its end: slot / abc [3] / flip over [off[f], off[f + 1]).  A slot's triple is the same in every frame.
// n_alloc: slots allocated at the end.  Rows: row_slot [nr] in snapshot order.  Outputs as immesh_mesh_texture_rows: facet_cam [nr],
// facet_uv [nr][6] (untextured rows untouched), facet_px [nr][2], counts [4], frames [n_alloc] with *n_frames_out.
int emu_texture_online(const immesh_texture_camera* rig, const immesh_texture_config* cfg, const float* verts, int nv, int n_frames, const int* number,
                       const int* kind, const double* pose, const int* cap, const int* off, const int* slot, const int* abc, const int* flip, int n_alloc,
                       const int* row_slot, int nr, int* facet_cam, float* facet_uv, int* facet_px, long long* counts, int* frames, int* n_frames_out) {
    std::vector<float4> vpos(nv > 0 ? nv : 1);
    for (int i = 0; i < nv; ++i) vpos[i] = make_float4(verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], 0.f);
    const TxoRecord fresh = {-1, INFINITY, 0, 0, {0, 0, 0, 0, 0, 0}};
    std::vector<TxoRecord> rec;
    std::vector<int> won, cov, tri(3 * (size_t)std::max(n_alloc, 1), 0), live_flip(std::max(n_alloc, 1), 0), live(std::max(n_alloc, 1), 0);
    int alloc = 0;   // slots allocated so far (the pool's counter)
    const TexRule rule = tex_rule(*cfg);
    long long pixels = 0;
    for (int f = 0; f < n_frames; ++f) {
        if ((size_t)cap[f] > rec.size()) {   // txo_state_migrate: fresh slots, then the allocated records
            std::vector<TxoRecord> nrec(cap[f], fresh);
            std::copy(rec.begin(), rec.begin() + std::min<size_t>(alloc, rec.size()), nrec.begin());
            rec.swap(nrec);
            won.assign(cap[f], 0);
            cov.assign(cap[f], 0);
        }
        std::fill(live.begin(), live.end(), 0);
        for (int e = off[f]; e < off[f + 1]; ++e) {
            const int s = slot[e];
            for (int k = 0; k < 3; ++k) tri[3 * (size_t)s + k] = abc[3 * (size_t)e + k];
            live[s] = 1;
            live_flip[s] = flip[e];
            alloc = std::max(alloc, s + 1);
        }
        // k_txo_cam
        if (kind[f] == 0) continue;
        const double* P = pose + 12 * (size_t)f;
        const immesh_texture_camera c = kind[f] == 2 ? txo_fixed_camera(*rig, P, P + 9) : txo_camera(*rig, P, P + 9);
        const DepthCam C = tex_camera(c, cfg->z_near, cfg->z_far);
        pixels += (long long)rig->width * rig->height;
        // k_tex_tile over every live slot (the result does not depend on the bins)
        auto corner = [&](int s, int k) { return vpos[tri[3 * (size_t)s + k]]; };
        std::vector<DepthTri> T(alloc);
        std::vector<int> ok(alloc, 0);
        for (int s = 0; s < alloc; ++s) ok[s] = live[s] && depth_tri_setup(C, corner(s, 0), corner(s, 1), corner(s, 2), &T[s]);
        for (int y = 0; y < C.h; ++y)
            for (int x = 0; x < C.w; ++x) {
                unsigned int best = 0x7f800000u;
                int ba = 0x7fffffff, bb = 0x7fffffff, bc = 0x7fffffff, bs = -1;
                for (int s = 0; s < alloc; ++s) {
                    if (!ok[s]) continue;
                    const DepthTri& D = T[s];
                    if (x < D.x_lo || x > D.x_hi || y < D.y_lo || y > D.y_hi) continue;
                    float zf;
                    if (!depth_sample(D, x, y, &zf)) continue;
                    unsigned int bits;
                    std::memcpy(&bits, &zf, 4);
                    if (bits >= 0x7f800000u) continue;
                    ++cov[s];
                    const int* q = &tri[3 * (size_t)s];
                    if (view_better(bits, q[0], q[1], q[2], best, ba, bb, bc)) { best = bits; ba = q[0]; bb = q[1]; bc = q[2]; bs = s; }
                }
                if (bs >= 0) ++won[bs];
            }
        // k_txo_update
        for (int s = 0; s < alloc; ++s) {
            const int wn = won[s], cv = cov[s];
            won[s] = 0; cov[s] = 0;
            if (wn < 1) continue;
            const float4 p[3] = {corner(s, 0), corner(s, 1), corner(s, 2)};
            txo_observe(C, p, live_flip[s], wn, cv, rule, number[f], &rec[s]);
        }
    }
    // k_txo_rows
    long long c0 = 0, c1 = 0;
    std::vector<int> used;
    for (int i = 0; i < nr; ++i) {
        const int s = row_slot[i];
        const TxoRecord& r = rec[s];
        facet_cam[i] = r.frame;
        facet_px[2 * i] = r.frame >= 0 ? r.won : 0;
        facet_px[2 * i + 1] = r.frame >= 0 ? r.cov : 0;
        if (r.frame < 0) { ++c1; continue; }
        txo_face_uv(r.uv, live_flip[s], facet_uv + 6 * (size_t)i);
        ++c0;
        used.push_back(r.frame);
    }
    std::sort(used.begin(), used.end());
    // k_txo_keys, the sort, k_txo_unique
    std::vector<int> all;
    for (int s = 0; s < std::min<int>(alloc, (int)rec.size()); ++s)
        if (rec[s].frame >= 0) all.push_back(rec[s].frame);
    std::sort(all.begin(), all.end());
    all.erase(std::unique(all.begin(), all.end()), all.end());
    for (size_t i = 0; i < all.size(); ++i) frames[i] = all[i];
    *n_frames_out = (int)all.size();
    counts[0] = c0; counts[1] = c1; counts[2] = (long long)(std::unique(used.begin(), used.end()) - used.begin()); counts[3] = pixels;
    return 0;
}
}  // extern "C"
