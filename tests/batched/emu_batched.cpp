// TEST INFRASTRUCTURE (not product code): the host emulation of the mesher (tests/emu/emu_mesh.cpp) with the m_smoothed flags
// (MeshDev::vsmoothed) attached, plus immesh_mesh_push_frame_batched: the orchestration of the CUDA library's batched frame
// (mesh_capi.cu, mesh_push_batched) on the same __host__ __device__ bodies, one thread at a time -- append chunks, the activation rule
// after the last chunk, the meshed voxels in key order (rank = flip priority), pass 1 (every dilation's smoothing), pass 2 (dilation
// lists again, triangulation, pull / commit, the batch's additions), removals after the last batch.  Built as its own library; the
// per-handle batch state lives beside the handle and is dropped with it.
#define immesh_mesh_create emu_base_mesh_create
#define immesh_mesh_destroy emu_base_mesh_destroy
#include "../emu/emu_mesh.cpp"
#undef immesh_mesh_create
#undef immesh_mesh_destroy

#include <unordered_map>

namespace {
struct BatchState {
    int max_vox = 0;
    std::vector<unsigned char> smoothed;   // MeshDev::vsmoothed
    std::vector<int> act, rank, fset;      // frame-wide activated voxels, ranks of a batch's work voxels, the batch's facet set
    std::vector<unsigned char> mark;       // FrameBuf::tri_mark
};
std::unordered_map<immesh_mesh*, BatchState*> g_batch;

void batch_reset(MeshDev& M) {   // per-batch lists: work, dilation items, facets, vertex refs, pulls, add list
    for (int k : {6, 7, 17, 19, 24, 25, 26, 28, 29}) M.cnt[k] = 0;
}
void batch_fill(immesh_mesh* h, const FrameBuf& F, std::vector<int>& rank, const std::vector<int>& sel, size_t lo, size_t hi) {
    for (size_t r = lo; r < hi; ++r) {
        const int w = voxel_enqueue(h->M, F, sel[r]);
        if (w >= 0) rank[w] = (int)r;
    }
}
}  // namespace

extern "C" {
int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    const int rc = emu_base_mesh_create(cfg, out);
    if (rc) return rc;
    immesh_mesh* h = *out;
    BatchState* s = new BatchState();
    s->max_vox = cfg->max_voxels ? cfg->max_voxels : (1 << 18);   // emu_mesh.cpp's default
    s->smoothed.assign((size_t)h->M.max_v, 0);
    h->M.vsmoothed = s->smoothed.data();
    g_batch[h] = s;
    return 0;
}
int immesh_mesh_destroy(immesh_mesh_t* h) {
    auto it = g_batch.find(h);
    if (it != g_batch.end()) { delete it->second; g_batch.erase(it); }
    return emu_base_mesh_destroy(h);
}
// the flags and smoothed positions of the vertices (test access)
int emu_mesh_smooth_state(immesh_mesh_t* h, unsigned char* flags, double* smooth) {
    const int nv = h->M.cnt[0];
    if (flags) std::memcpy(flags, h->M.vsmoothed, (size_t)nv);
    if (smooth) std::memcpy(smooth, h->M.vsmooth, (size_t)nv * 3 * sizeof(double));
    return nv;
}
// size of the batched frame's facet set (tests of the bounded probe)
int emu_mesh_set_batch_fset_bits(immesh_mesh_t* h, int bits) {
    g_batch.at(h)->fset.assign((size_t)1 << bits, -1);
    return 0;
}
int immesh_mesh_push_frame_batched(immesh_mesh_t* h, const float* xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels,
                                   int64_t* stats) {
    (void)on_device;   // host memory either way
    if (!h || (!xyz && n > 0) || n < 0 || !pose_t || batch_points < 0 || batch_points > h->F.max_cand || batch_voxels < 0 || batch_voxels > h->F.max_work) return IMMESH_E_INVALID;
    if (h->F.shard_n > 1) return IMMESH_E_INVALID;
    BatchState& S = *g_batch.at(h);
    MeshDev& M = h->M;
    const MeshParams& P = h->P;
    const int B = batch_points ? batch_points : h->F.max_cand, V = batch_voxels ? batch_voxels : h->F.max_work;
    if (S.act.empty()) {
        S.act.resize(S.max_vox); S.rank.resize(h->F.max_work); S.mark.assign(M.max_t, 0);
        if (S.fset.empty()) S.fset.assign(p2((size_t)h->F.max_list * 2), -1);
    }
    FrameBuf F = h->F;
    F.act = S.act.data(); F.max_act = S.max_vox;
    F.work_rank = S.rank.data(); F.tri_mark = S.mark.data();
    F.fset = S.fset.data(); F.fset_mask = (unsigned)(S.fset.size() - 1);
    const long long step = std::max(1LL, (long long)std::lround((double)(n / P.append_target)));
    const long long m_total = n > 0 ? (n + step - 1) / step : 0;
    F.frame = ++h->frame_counter;
    for (int j = 0; j < 3; ++j) { h->fp_storage.pose_t[j] = pose_t[j]; h->fp_storage.prio_origin[j] = 0; }
    F.fp = &h->fp_storage;
    for (int k = 5; k <= 10; ++k) M.cnt[k] = 0;
    for (int k = 17; k <= 26; ++k) M.cnt[k] = 0;
    for (int k = 28; k <= 35; ++k) M.cnt[k] = 0;
    // append, chunk by chunk: candidates [c B, (c + 1) B) of the frame (candidate i = point i step)
    long long chunks = 0;
    for (long long c0 = 0; c0 < m_total; c0 += B, ++chunks) {
        const int m = (int)std::min<long long>(B, m_total - c0);
        for (int i = 0; i < m; ++i) std::memcpy(&h->pts[(size_t)i * 3], xyz + (size_t)(c0 + i) * step * 3, 12);
        F.pts = h->pts.data(); F.step = 1; F.m = m; F.n = m;
        F.cmask = (unsigned)(p2((size_t)std::max(m, 1) * 2) - 1);
        for (unsigned i = 0; i <= F.cmask; ++i) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
        M.cnt[9] = 0; M.cnt[18] = 0;
        for (int c = 0; c < m; ++c) cand_init(M, P, F, c);
        for (int c = 0; c < m; ++c) cand_conflicts(M, P, F, c);
        for (int c = 0; c < m; ++c)
            if (F.cand_status[c] == CAND_UNDECIDED && !cand_poll(M, P, F, c)) return -100;
        int run = 0;
        for (int c = 0; c < m; ++c) { F.cand_scan[c] = run; run += F.cand_status[c] == CAND_ACCEPT; }
        const int base = M.cnt[0];
        for (int c = 0; c < m; ++c) cand_commit(M, P, F, c, base);
        for (int c = 0; c < m; ++c) cand_place(M, F, c, base);
        M.cnt[0] += M.cnt[10]; M.cnt[33] += M.cnt[10]; M.cnt[10] = 0;
    }
    // activation rule over the frame's activated voxels; the meshed ones in ascending key order (their rank = flip priority)
    std::vector<int> sel;
    for (int a = 0; a < std::min(M.cnt[5], F.max_act); ++a)
        if (voxel_activate(M, F, F.act[a])) sel.push_back(F.act[a]);
    std::sort(sel.begin(), sel.end(), [&](int a, int b) { return M.vkeys[a] < M.vkeys[b]; });
    const size_t nbat = (sel.size() + V - 1) / V;
    DilateSmem* DS = new DilateSmem();
    // pass 1: every dilation's smoothing before any orientation
    for (size_t b = 0; b < nbat; ++b) {
        batch_reset(M);
        batch_fill(h, F, S.rank, sel, b * V, std::min(sel.size(), (b + 1) * V));
        for (int i = 0; i < std::min(M.cnt[29], F.max_ditem); ++i) voxel_dilate(M, P, F, F.ditem[i], DS, 0, 1);
    }
    // pass 2: dilation lists again (the re-stored smoothing writes the same bits), triangulation, pull + commit, this batch's additions
    MeshSmem<256>* S1 = new MeshSmem<256>();
    MeshSmem<1024>* S2 = new MeshSmem<1024>();
    MeshWarpSmem<128>* SW = new MeshWarpSmem<128>();
    for (size_t b = 0; b < nbat; ++b) {
        batch_reset(M);
        for (unsigned i = 0; i <= F.fset_mask; ++i) F.fset[i] = -1;
        batch_fill(h, F, S.rank, sel, b * V, std::min(sel.size(), (b + 1) * V));
        for (int i = 0; i < std::min(M.cnt[29], F.max_ditem); ++i) voxel_dilate(M, P, F, F.ditem[i], DS, 0, 1);
        const int nw = work_total(M, F);
        for (int i = 0; i < nw; ++i) voxel_mesh_warp<128>(M, P, F, work_slot(M, F, i), SW, 0, 1, 96);
        for (int i = 0; i < nw; ++i) {
            const int w = work_slot(M, F, i);
            const int nd = F.work_n_ids[w];
            if (nd > 96 && nd <= 256) voxel_mesh<256>(M, P, F, w, S1, 0, 1, 1);
        }
        for (int f = 0; f < std::min(M.cnt[25], F.max_list); ++f) commit_face(M, P, F, f);
        for (int r = 0; r < std::min(M.cnt[26], F.max_vref); ++r) pull_vertex(M, P, F, r);
        for (int e = 0; e < std::min(M.cnt[28], F.max_list); ++e) pull_check(M, F, e);
        for (int i = 0; i < nw; ++i) {
            const int w = work_slot(M, F, i);
            const int nd = F.work_n_ids[w];
            if (nd < 0 || nd > 256) voxel_mesh<1024>(M, P, F, w, S2, 0, 1);
        }
        const int nadd = std::min(M.cnt[7], F.max_list);
        for (int e = 0; e < nadd; ++e) {
            const int t = tri_add(M, F.add_tri[(size_t)e * 3], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
            if (t >= 0) F.tri_mark[t] = IM_TRI_BORN;
        }
        M.cnt[34] += M.cnt[7]; M.cnt[35] += M.cnt[6] + M.cnt[17];
    }
    delete DS; delete S1; delete S2; delete SW;
    // deferred removals; marks cleared for the next frame
    for (int t = 0; t < std::min(M.cnt[1], M.max_t); ++t) {
        if (F.tri_mark[t] == IM_TRI_REMOVE) tri_remove(M, t);
        F.tri_mark[t] = 0;
    }
    M.cnt[10] = M.cnt[33]; M.cnt[7] = M.cnt[34]; M.cnt[6] = M.cnt[35]; M.cnt[17] = 0;
    std::memcpy(h->last_cnt, M.cnt, 32 * sizeof(int));
    if (stats) {
        stats[0] = chunks; stats[1] = (int64_t)nbat;
        stats[2] = (int64_t)(S.act.size() * 4 + S.rank.size() * 4 + S.mark.size() + S.fset.size() * 4);
        stats[3] = M.cnt[7];
    }
    if (M.cnt[3] & ~(IM_MERR_KEY_RANGE | IM_MERR_PRIO_RANGE)) return IMMESH_E_CAPACITY;
    return M.cnt[3] ? IMMESH_E_RANGE : 0;
}
}  // extern "C"
