// TEST INFRASTRUCTURE (not product code): executes the __host__ __device__ bodies of the CUDA mesher
// (immesh_b200/csrc/mesh_core.cuh, mesh_voxel.cuh) on the CPU, one thread at a time, for the CPU-only logic
// tests.  The shipped library never links or calls this.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "../../immesh_b200/csrc/mesh_voxel.cuh"

using namespace immesh;

struct immesh_mesh {
    MeshParams P;
    MeshDev M;
    FrameBuf F;
    std::vector<float4> vpos, vchunk_pts;
    std::vector<double> vsmooth;
    std::vector<int> v_tri_head, gval, vox_chunk, cand_pos, vox_count, vox_mt, vox_na, vox_frame, tri_next, thash, cnt;
    std::vector<unsigned long long> gkeys, vkeys, tri_flip, ckeys, cand_gkey, add_flip;
    std::vector<int4> tri;
    std::vector<float> pts;
    std::vector<int> cand_vslot, cand_status, cand_scan, cand_conf, cand_nconf, cand_next, chead, act, work, work_n, work_ids, add_tri, rem_tri, work_nf, all_vref, fset, pulled, work_ring, work_done, ditem;
    std::vector<unsigned int> work_bits;
    std::vector<int4> all_faces;
    std::vector<double> work_axes;
    std::vector<XSmooth> x_smooth;
    std::vector<int4> x_face, x_rem;
    std::vector<unsigned long long> x_word;
    FramePose fp_storage;
    int nw = 0;
    int frame_counter = 0;
    int last_cnt[IM_MC_HOST];
};
static size_t p2(size_t v) { size_t p = 1; while (p < v) p <<= 1; return p; }

extern "C" {
int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    immesh_mesh* h = new immesh_mesh();
    MeshParams& P = h->P;
    P.xi = cfg->points_minimum_scale; P.res = cfg->voxel_resolution; P.accept = cfg->voxel_resolution * 1.25;
    P.knn_max = P.accept * 2 * 1.000001; P.inv_q = 4194304.0 / cfg->voxel_resolution; P.append_target = cfg->number_of_pts_append_to_map;
    const int max_v = cfg->max_vertices ? cfg->max_vertices : (1 << 20), max_t = cfg->max_triangles ? cfg->max_triangles : (1 << 22);
    const int max_vox = cfg->max_voxels ? cfg->max_voxels : (1 << 18), mfp = cfg->max_frame_points ? cfg->max_frame_points : (1 << 20);
    MeshDev& M = h->M;
    M.max_v = max_v; M.max_t = max_t;
    h->vpos.resize(max_v); h->vsmooth.resize((size_t)max_v * 3); h->v_tri_head.assign(max_v, -1);
    const size_t gcap = p2((size_t)max_v * 2), vcap = p2((size_t)max_vox * 2), tcap = p2((size_t)max_t * 2);
    h->gkeys.assign(gcap, IM_EMPTY_KEY); h->gval.assign(gcap, -1);
    h->vkeys.assign(vcap, IM_EMPTY_KEY); h->vox_chunk.assign(vcap * IM_VCHUNKS, -1); h->vox_count.assign(vcap, 0); h->vox_mt.assign(vcap, 0); h->vox_na.assign(vcap, 0); h->vox_frame.assign(vcap, -1);
    h->tri.resize(max_t); h->tri_next.resize((size_t)max_t * 3); h->tri_flip.resize(max_t); h->thash.assign(tcap, -1);
    h->cnt.assign(IM_MC_ALLOC, 0);
    mesh_cnt_init(h->cnt.data());
    M.vpos = h->vpos.data(); M.vsmooth = h->vsmooth.data(); M.v_tri_head = h->v_tri_head.data();
    M.gkeys = h->gkeys.data(); M.gval = h->gval.data(); M.gmask = (unsigned)(gcap - 1);
    M.vkeys = h->vkeys.data(); M.vmask = (unsigned)(vcap - 1); M.vox_chunk = h->vox_chunk.data(); M.vox_count = h->vox_count.data(); M.max_vchunks = max_v / 4 + 1024; h->vchunk_pts.resize((size_t)M.max_vchunks * 16); M.vchunk_pts = h->vchunk_pts.data();
    M.vox_meshing_times = h->vox_mt.data(); M.vox_new_added = h->vox_na.data(); M.vox_frame = h->vox_frame.data(); M.vox_short_axis = nullptr;
    M.tri = h->tri.data(); M.tri_next = h->tri_next.data(); M.tri_flip = h->tri_flip.data(); M.thash = h->thash.data(); M.tmask = (unsigned)(tcap - 1);
    M.cnt = h->cnt.data();
    FrameBuf& F = h->F;
    const size_t mc = mfp;
    F.max_cand = mfp; F.max_work = std::min(max_vox, 1 << 14); F.max_act = std::min<size_t>(max_vox, mc); F.max_list = 1 << 20;
    h->pts.resize(mc * 3); h->cand_gkey.resize(mc); h->cand_vslot.resize(mc); h->cand_status.resize(mc); h->cand_scan.resize(mc);
    h->cand_conf.resize(mc * IM_CONF_K); h->cand_nconf.resize(mc); h->cand_next.resize(mc); h->cand_pos.resize(mc);
    const size_t ccap = p2(mc * 2);
    h->ckeys.resize(ccap); h->chead.resize(ccap);
    h->act.resize(F.max_act); h->work.resize(F.max_work); h->work_n.resize(F.max_work); h->work_ids.resize((size_t)F.max_work * IM_MAXD);
    h->work_nf.resize(F.max_work); h->work_bits.assign((size_t)F.max_work * (IM_MAXG / 32), 0u); h->work_ring.assign(F.max_work, 0); h->work_done.assign(F.max_work, 0); F.max_ditem = F.max_work * 4; h->ditem.resize(F.max_ditem); F.max_vref = 1 << 21; h->all_faces.resize(F.max_list); h->all_vref.resize(F.max_vref); h->pulled.resize((size_t)F.max_list * 2); F.fset_mask = (1u << 19) - 1; h->fset.assign((size_t)F.fset_mask + 1, -1); h->work_axes.resize((size_t)F.max_work * 9);
    h->add_tri.resize((size_t)F.max_list * 3); h->add_flip.resize(F.max_list); h->rem_tri.resize(F.max_list);
    F.pts = h->pts.data(); F.cand_gkey = h->cand_gkey.data(); F.cand_vslot = h->cand_vslot.data(); F.cand_status = h->cand_status.data();
    F.cand_scan = h->cand_scan.data(); F.cand_conf = h->cand_conf.data(); F.cand_nconf = h->cand_nconf.data(); F.cand_next = h->cand_next.data(); F.cand_pos = h->cand_pos.data();
    F.ckeys = h->ckeys.data(); F.chead = h->chead.data(); F.scan_block = nullptr;
    F.act = h->act.data(); F.work = h->work.data(); F.work_n_ids = h->work_n.data(); F.work_ids = h->work_ids.data(); F.work_nfaces = h->work_nf.data(); F.work_bits = h->work_bits.data(); F.work_ring = h->work_ring.data(); F.work_done = h->work_done.data(); F.ditem = h->ditem.data(); F.all_faces = h->all_faces.data(); F.all_vref = h->all_vref.data(); F.pulled = h->pulled.data(); F.fset = h->fset.data(); F.work_axes = h->work_axes.data();
    F.add_tri = h->add_tri.data(); F.add_flip = h->add_flip.data(); F.rem_tri = h->rem_tri.data();
    F.shard_rank = 0; F.shard_n = 1; F.x_cap = 0; F.x_smooth = nullptr; F.x_face = nullptr; F.x_word = nullptr; F.x_rem = nullptr;
    std::memset(h->last_cnt, 0, sizeof(h->last_cnt));
    *out = h;
    return 0;
}
int immesh_mesh_destroy(immesh_mesh_t* h) { delete h; return 0; }
// ---- one frame in three phases (the sharded test exchanges the lists between them, like the device path does with NCCL)
// A: append (replicated) + activation + dilation of the voxels this rank owns
int emu_mesh_phase_a(immesh_mesh_t* h, const float* world_xyz, int n, const double* pose_t) {
    FrameBuf& F = h->F;
    MeshDev& M = h->M;
    const MeshParams& P = h->P;
    const int step = std::max(1, (int)std::lround((double)(n / P.append_target)));
    F.n = n; F.step = step; F.m = n > 0 ? (n + step - 1) / step : 0; F.frame = ++h->frame_counter;
    for (int j = 0; j < 3; ++j) { h->fp_storage.pose_t[j] = pose_t[j]; h->fp_storage.prio_origin[j] = (long long)std::floor(pose_t[j] / P.res) - 1024; }
    F.fp = &h->fp_storage;
    F.cmask = (unsigned)(p2((size_t)std::max(F.m, 1) * 2) - 1);
    if (n > 0) std::memcpy(h->pts.data(), world_xyz, (size_t)n * 12);
    for (unsigned i = 0; i <= F.cmask; ++i) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    mesh_cnt_frame_begin(M);
    for (unsigned i = 0; i <= F.fset_mask; ++i) F.fset[i] = -1;
    for (int c = 0; c < F.m; ++c) cand_init(M, P, F, c);
    for (int c = 0; c < F.m; ++c) cand_conflicts(M, P, F, c);
    for (int c = 0; c < F.m; ++c)
        if (F.cand_status[c] == CAND_UNDECIDED && !cand_poll(M, P, F, c)) return -100;
    int run = 0;
    for (int c = 0; c < F.m; ++c) { F.cand_scan[c] = run; run += F.cand_status[c] == CAND_ACCEPT; }
    const int base = M.cnt[IM_MC_VERTICES];
    for (int c = 0; c < F.m; ++c) cand_commit(M, P, F, c, base);
    for (int c = 0; c < F.m; ++c) cand_place(M, F, c, base);
    const int na = std::min(M.cnt[IM_MC_ACT], F.max_act);
    for (int a = 0; a < na; ++a) voxel_select(M, F, a);
    h->nw = work_total(M, F);
    DilateSmem* DS = new DilateSmem();
    for (int i = 0; i < std::min(M.cnt[IM_MC_DITEMS], F.max_ditem); ++i) voxel_dilate(M, P, F, F.ditem[i], DS, 0, 1);
    delete DS;
    return 0;
}
// B: triangulation + pull + commit decisions of the owned voxels
int emu_mesh_phase_b(immesh_mesh_t* h) {
    FrameBuf& F = h->F;
    MeshDev& M = h->M;
    const MeshParams& P = h->P;
    const int nw = h->nw;
    MeshSmem<256>* S1 = new MeshSmem<256>();
    MeshSmem<1024>* S2 = new MeshSmem<1024>();
    MeshWarpSmem<128>* SW = new MeshWarpSmem<128>();
    for (int i = 0; i < nw; ++i) voxel_mesh_warp<128>(M, P, F, work_slot(M, F, i), SW, 0, 1, 96);   // same split as the device
    delete SW;
    for (int i = 0; i < nw; ++i) {
        const int w = work_slot(M, F, i);
        const int nd = F.work_n_ids[w];
        if (nd > 96 && nd <= 256) voxel_mesh<256>(M, P, F, w, S1, 0, 1, 1);
    }
    for (int f = 0; f < std::min(M.cnt[IM_MC_FACES], F.max_list); ++f) commit_face(M, P, F, f);
    for (int r = 0; r < std::min(M.cnt[IM_MC_VREFS], F.max_vref); ++r) pull_vertex(M, P, F, r);
    for (int e = 0; e < std::min(M.cnt[IM_MC_PULLED], F.max_list); ++e) pull_check(M, F, e);
    for (int i = 0; i < nw; ++i) {
        const int w = work_slot(M, F, i);
        const int nd = F.work_n_ids[w];
        if (nd < 0 || nd > 256) voxel_mesh<1024>(M, P, F, w, S2, 0, 1);
    }
    delete S1; delete S2;
    return 0;
}
// C: push (all removals, then all insertions)
int emu_mesh_phase_c(immesh_mesh_t* h) {
    FrameBuf& F = h->F;
    MeshDev& M = h->M;
    const int nr = std::min(M.cnt[IM_MC_REMOVE], F.max_list), nadd = std::min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = 0; e < nr; ++e) tri_remove(M, F.rem_tri[e]);
    for (int e = 0; e < nadd; ++e) tri_add(M, F.add_tri[(size_t)e * 3], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
    mesh_cnt_frame_end(M);
    std::memcpy(h->last_cnt, M.cnt, sizeof(h->last_cnt));
    return M.cnt[IM_MC_ERR] ? IMMESH_E_CAPACITY : 0;
}
int immesh_mesh_push_frame(immesh_mesh_t* h, const float* world_xyz, int n, const double* pose_t, int) {
    int rc = emu_mesh_phase_a(h, world_xyz, n, pose_t);
    if (rc) return rc;
    emu_mesh_phase_b(h);
    return emu_mesh_phase_c(h);
}
// ---- sharded per-voxel stage: exchange lists
int emu_mesh_set_shard(immesh_mesh_t* h, int rank, int nranks) {
    FrameBuf& F = h->F;
    F.shard_rank = rank; F.shard_n = nranks; F.x_cap = 1 << 16;
    h->x_smooth.resize(F.x_cap); h->x_face.resize(F.x_cap); h->x_word.resize(F.x_cap); h->x_rem.resize(F.x_cap);
    F.x_smooth = h->x_smooth.data(); F.x_face = h->x_face.data(); F.x_word = h->x_word.data(); F.x_rem = h->x_rem.data();
    return 0;
}
int emu_mesh_xcounts(immesh_mesh_t* h, int* out) {   // smooth, face, remove
    out[0] = std::min(h->M.cnt[IM_MC_X_SMOOTHS], h->F.x_cap); out[1] = std::min(h->M.cnt[IM_MC_X_FACES], h->F.x_cap); out[2] = std::min(h->M.cnt[IM_MC_X_REMS], h->F.x_cap);
    return 0;
}
int emu_mesh_xget(immesh_mesh_t* h, void* smooth32, int* face4, unsigned long long* word, int* rem4) {
    int c[3];
    emu_mesh_xcounts(h, c);
    if (smooth32) std::memcpy(smooth32, h->x_smooth.data(), (size_t)c[0] * sizeof(XSmooth));
    if (face4) std::memcpy(face4, h->x_face.data(), (size_t)c[1] * sizeof(int4));
    if (word) std::memcpy(word, h->x_word.data(), (size_t)c[1] * 8);
    if (rem4) std::memcpy(rem4, h->x_rem.data(), (size_t)c[2] * sizeof(int4));
    return 0;
}
int emu_mesh_xapply_smooth(immesh_mesh_t* h, const void* smooth32, int n) {
    const XSmooth* e = (const XSmooth*)smooth32;
    for (int i = 0; i < n; ++i) { h->M.vsmooth[(size_t)e[i].id * 3] = e[i].x; h->M.vsmooth[(size_t)e[i].id * 3 + 1] = e[i].y; h->M.vsmooth[(size_t)e[i].id * 3 + 2] = e[i].z; }
    return 0;
}
int emu_mesh_xapply_lists(immesh_mesh_t* h, const int* face4, const unsigned long long* word, int nf, const int* rem4, int nr) {
    for (int i = 0; i < nf; ++i) apply_face(h->M, h->F, face4[i * 4], face4[i * 4 + 1], face4[i * 4 + 2], word[i]);
    for (int i = 0; i < nr; ++i) apply_remove(h->M, h->F, rem4[i * 4], rem4[i * 4 + 1], rem4[i * 4 + 2]);
    return 0;
}
int emu_mesh_error_word(immesh_mesh_t* h) { return h->last_cnt[IM_MC_ERR]; }   // IM_MERR_* flags of the last frame
// keys (x, y, z) of the voxels the last frame meshed (its work list, in work-list order); returns their number
int emu_mesh_frame_voxels(immesh_mesh_t* h, int32_t* keys) {
    const int nw = work_total(h->M, h->F);
    for (int i = 0; keys && i < nw; ++i) {
        int x, y, z;
        unpack_ikey(h->M.vkeys[h->F.work[work_slot(h->M, h->F, i)]], &x, &y, &z);
        keys[i * 3] = x; keys[i * 3 + 1] = y; keys[i * 3 + 2] = z;
    }
    return nw;
}
int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out) {
    const int* c = h->last_cnt;
    out[0] = c[IM_MC_VERTICES]; out[1] = c[IM_MC_TRIS_LIVE]; out[2] = c[IM_MC_NEW_VERTICES]; out[3] = c[IM_MC_WORK_FRONT] + c[IM_MC_WORK_BACK];
    out[4] = c[IM_MC_ADD]; out[5] = c[IM_MC_REMOVE]; out[6] = c[IM_MC_VOXELS]; out[7] = c[IM_MC_ACT];
    return 0;
}
int immesh_mesh_snapshot(immesh_mesh_t* h, float* vertices, int32_t* triangles, int32_t* flips) {
    const MeshDev& M = h->M;
    const int nv = M.cnt[IM_MC_VERTICES], nalloc = M.cnt[IM_MC_TRIS_ALLOC];
    if (vertices)
        for (int i = 0; i < nv; ++i) { vertices[i * 3] = M.vpos[i].x; vertices[i * 3 + 1] = M.vpos[i].y; vertices[i * 3 + 2] = M.vpos[i].z; }
    std::vector<std::array<int, 4>> rows;
    for (int t = 0; t < nalloc; ++t)
        if (M.tri[t].w) rows.push_back({M.tri[t].x, M.tri[t].y, M.tri[t].z, (int)(M.tri_flip[t] & 1ull)});
    std::sort(rows.begin(), rows.end());
    for (size_t i = 0; i < rows.size(); ++i) {
        if (triangles) for (int j = 0; j < 3; ++j) triangles[i * 3 + j] = rows[i][j];
        if (flips) flips[i] = rows[i][3];
    }
    return 0;
}
}
