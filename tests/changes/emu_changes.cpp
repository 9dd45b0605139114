// TEST INFRASTRUCTURE (not product code): the host emulation of the mesher with the batched frame (tests/batched/emu_batched.cpp) and
// the change feed of immesh_mesh_changes_enable / immesh_mesh_changes.  The feed's __host__ __device__ bodies (mesh_changes.cuh, and
// chg_touch inside apply_face) run one thread at a time in the device's order (mesh_feeds.cu, mesh_changes_launch): the touched set
// after the push and before the frame's counter end (or the sweep), the rows against the published bytes, the ring append and the
// header.  Only the LSD radix sort is replaced by a sort of the rows' triples (the triples of a frame are distinct, so both give the
// same order).  The read side restates the host logic of immesh_mesh_changes.
#define immesh_mesh_push_frame emu_plain_push_frame
#define immesh_mesh_push_frame_batched emu_plain_push_frame_batched
#include "../batched/emu_batched.cpp"
#undef immesh_mesh_push_frame
#undef immesh_mesh_push_frame_batched

#include "../../immesh_b200/csrc/mesh_changes.cuh"

namespace {
struct Feed {
    int cap = 0, enable_frame = 0, last_frame = 0;
    std::vector<int> stamp, list, cnt;
    std::vector<unsigned char> pub;
    std::vector<int4> marked, rowbuf, ring;
    std::vector<ChgHdr> hdr;
    long long written = 0;
    ChgDev C = {};
};
std::unordered_map<immesh_mesh*, Feed*> g_feed;

Feed* feed_of(immesh_mesh* h) {   // (an entry left by a destroyed handle at the same address does not match its stamp buffer)
    auto it = g_feed.find(h);
    if (it == g_feed.end()) return nullptr;
    if (h->F.chg_stamp == it->second->stamp.data()) return it->second;
    delete it->second;
    g_feed.erase(it);
    return nullptr;
}
void feed_frame(immesh_mesh* h, const FrameBuf& F, bool batched) {
    Feed& d = *feed_of(h);
    const MeshDev& M = h->M;
    const ChgDev& C = d.C;
    const bool full = batched;
    if (!batched)
        for (int e = 0; e < chg_gather_count(M, F); ++e) chg_gather(M, F, e);
    if (chg_sweeping(F, full))
        for (int t = 0; t < std::min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t); ++t) chg_sweep_slot(M, F, C, t);
    const int n = std::min(chg_listed(F, full), F.chg_cap);
    for (int i = 0; i < n; ++i) chg_row_mark(M, F, C, i);
    int run = 0;
    for (int i = 0; i < n; ++i) run += chg_row_emit(C, i, run);
    F.chg_cnt[IM_CH_ROWS] = run;
    std::vector<unsigned int> order(run);
    for (int i = 0; i < run; ++i) order[i] = (unsigned)i;
    std::sort(order.begin(), order.end(), [&](unsigned a, unsigned b) {
        const int4 x = C.rowbuf[a], y = C.rowbuf[b];
        return x.x != y.x ? x.x < y.x : x.y != y.y ? x.y < y.y : x.z < y.z;
    });
    if (!chg_lost(F, C, full))
        for (int i = 0; i < run; ++i) chg_append(C, order.data(), i);
    chg_frame_end(M, F, C, full, full);
    d.last_frame = F.frame;
}
}  // namespace

extern "C" {
int immesh_mesh_push_frame(immesh_mesh_t* h, const float* world_xyz, int n, const double* pose_t, int) {
    if (!feed_of(h)) return emu_plain_push_frame(h, world_xyz, n, pose_t, 0);
    const int rc = emu_mesh_phase_a(h, world_xyz, n, pose_t);
    if (rc) return rc;
    emu_mesh_phase_b(h);
    FrameBuf& F = h->F;
    MeshDev& M = h->M;
    const int nr = std::min(M.cnt[IM_MC_REMOVE], F.max_list), nadd = std::min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = 0; e < nr; ++e) tri_remove(M, F.rem_tri[e]);
    for (int e = 0; e < nadd; ++e) tri_add(M, F.add_tri[(size_t)e * 3], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
    feed_frame(h, F, false);
    mesh_cnt_frame_end(M);
    std::memcpy(h->last_cnt, M.cnt, sizeof(h->last_cnt));
    return M.cnt[IM_MC_ERR] ? IMMESH_E_CAPACITY : 0;
}
int immesh_mesh_push_frame_batched(immesh_mesh_t* h, const float* xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels,
                                   int64_t* stats) {
    const int rc = emu_plain_push_frame_batched(h, xyz, n, on_device, pose_t, batch_points, batch_voxels, stats);
    if (rc == IMMESH_E_INVALID || !feed_of(h)) return rc;
    FrameBuf F = h->F;
    F.frame = h->frame_counter;
    feed_frame(h, F, true);
    return rc;
}
int immesh_mesh_changes_enable(immesh_mesh_t* h, int64_t max_rows, int max_frames) {
    if (!h || max_rows < 0 || max_rows > (1LL << 30) || (max_rows > 0 && (max_frames < 1 || max_frames > (1 << 20)))) return IMMESH_E_INVALID;
    if (h->F.shard_n > 1) return IMMESH_E_INVALID;
    if (Feed* f = feed_of(h)) { delete f; g_feed.erase(h); }
    h->F.chg_stamp = nullptr; h->F.chg_list = nullptr; h->F.chg_cnt = nullptr; h->F.chg_cap = 0;
    if (max_rows == 0) return 0;
    Feed* d = new Feed();
    const int max_t = h->M.max_t;
    d->cap = (int)std::min<int64_t>(max_rows, 1 << 21);
    d->stamp.assign(max_t, -1); d->pub.assign(max_t, 0); d->list.assign(d->cap, 0); d->cnt.assign(IM_CH_SIZE, 0);
    d->marked.resize(d->cap); d->rowbuf.resize(d->cap); d->ring.resize((size_t)max_rows);
    ChgHdr none; none.frame = -1; none.v_begin = none.v_end = none.r_begin = none.r_end = none.lost = -1;
    d->hdr.assign(max_frames, none);
    d->C.pub = d->pub.data(); d->C.marked = d->marked.data(); d->C.rowbuf = d->rowbuf.data(); d->C.hdr = d->hdr.data(); d->C.ring = d->ring.data(); d->C.written = &d->written;
    d->C.max_rows = max_rows; d->C.max_frames = max_frames;
    for (int t = 0; t < std::min(h->M.cnt[IM_MC_TRIS_ALLOC], max_t); ++t) d->pub[t] = chg_state(h->M, t);
    d->enable_frame = d->last_frame = h->frame_counter;
    g_feed[h] = d;
    h->F.chg_stamp = d->stamp.data(); h->F.chg_list = d->list.data(); h->F.chg_cnt = d->cnt.data(); h->F.chg_cap = d->cap;
    return 0;
}
int immesh_mesh_changes(immesh_mesh_t* h, int64_t since, int64_t* frames, int cap_frames, int32_t* rows, int64_t cap_rows, float* vertices, int64_t cap_vertices,
                        int64_t* counts) {
    if (!h || !counts || cap_frames < 0 || cap_rows < 0 || cap_vertices < 0 || (cap_frames > 0 && !frames) || (cap_rows > 0 && !rows) || (cap_vertices > 0 && !vertices))
        return IMMESH_E_INVALID;
    for (int i = 0; i < 4; ++i) counts[i] = 0;
    Feed* d = feed_of(h);
    if (h->F.shard_n > 1 || !d) return IMMESH_E_INVALID;
    const ChgDev& C = d->C;
    const int64_t newest = d->last_frame, nf = newest - since;
    counts[3] = newest;
    if (since > newest) return IMMESH_E_INVALID;
    if (since < d->enable_frame || nf > C.max_frames) return IMMESH_E_RANGE;
    if (nf == 0) return 0;
    for (int64_t f = since + 1; f <= newest; ++f) {
        const ChgHdr& r = C.hdr[f % C.max_frames];
        if (r.frame != f || r.lost || r.r_begin < d->written - C.max_rows) return IMMESH_E_RANGE;
    }
    const ChgHdr& first = C.hdr[(since + 1) % C.max_frames];
    const ChgHdr& last = C.hdr[newest % C.max_frames];
    const int64_t nrows = last.r_end - first.r_begin, nverts = last.v_end - first.v_begin;
    counts[0] = nf; counts[1] = nrows; counts[2] = nverts;
    if (nf > cap_frames || nrows > cap_rows || nverts > cap_vertices) return IMMESH_E_CAPACITY;
    for (int64_t f = since + 1, k = 0; f <= newest; ++f, ++k) {
        const ChgHdr& r = C.hdr[f % C.max_frames];
        frames[k * 4] = f; frames[k * 4 + 1] = r.v_begin; frames[k * 4 + 2] = r.v_end; frames[k * 4 + 3] = r.r_end - first.r_begin;
    }
    for (int64_t g = first.r_begin; g < last.r_end; ++g) std::memcpy(rows + (g - first.r_begin) * 4, &C.ring[g % C.max_rows], 16);
    for (int64_t i = 0; i < nverts; ++i) {
        const float4 p = h->M.vpos[first.v_begin + i];
        vertices[i * 3] = p.x; vertices[i * 3 + 1] = p.y; vertices[i * 3 + 2] = p.z;
    }
    return 0;
}
int immesh_mesh_wait(immesh_mesh_t*) { return 0; }   // one thread: every frame has finished
}  // extern "C"
