// immesh_b200 -- the mesh's change feed (immesh_mesh_changes_enable / immesh_mesh_changes): per frame, the net difference of the
// live triangle set and its flips against the state the feed last published, as (a, b, c, code) rows in ascending triple order,
// appended with a frame header to a device ring.  The bodies below run one thread each in the kernels of mesh_capi.cu (k_chg_*)
// and in the host emulation of the tests.
//
// Touched set of a frame: every slot whose live flag or flip word a writer of the frame changed -- the "existing" branch of
// apply_face (chg_touch), the removal and addition lists of the push (chg_gather) -- deduplicated by a per-slot stamp of the frame
// number.  A batched frame, and a frame whose touched list overflowed, take the sweep instead: every allocated slot whose state
// differs from its published byte.
#pragma once
#include "mesh_core.cuh"

namespace immesh {

struct ChgHdr { long long frame, v_begin, v_end, r_begin, r_end, lost; };   // rows [r_begin, r_end) in ring positions since enable
struct ChgDev {
    unsigned char* pub;   // [max_t] state last published per triangle slot: bit 0 live, bit 1 flip (chg_state)
    int4* marked;         // [chg_cap] per listed slot: its row, or w = -1
    int4* rowbuf;         // [chg_cap] the frame's rows in list order
    ChgHdr* hdr;          // [max_frames] frame f at f % max_frames
    int4* ring;           // [max_rows] row g (since enable) at g % max_rows
    long long* written;   // rows appended since enable
    long long max_rows;
    int max_frames;
};
enum : int { IM_CHG_REMOVED = 0, IM_CHG_ADDED = 2, IM_CHG_FLIPPED = 4 };   // row codes; | flip for the last two

IM_HD unsigned char chg_state(const MeshDev& M, int t) {
    return M.tri[t].w ? (unsigned char)(1u | ((unsigned)(M.tri_flip[t] & 1ull) << 1)) : (unsigned char)0;
}
// code of the row of a slot whose state went from `was` to `now`; -1: no row
IM_HD int chg_code(unsigned char was, unsigned char now) {
    if (was == now) return -1;
    if (!(now & 1)) return IM_CHG_REMOVED;
    return ((was & 1) ? IM_CHG_FLIPPED : IM_CHG_ADDED) | ((now >> 1) & 1);
}
// entry e of the frame's removal list followed by its addition list (after the push: an added triple is in the store)
IM_HDN inline void chg_gather(const MeshDev& M, const FrameBuf& F, int e) {
    const int nr = M.cnt[IM_MC_REMOVE] < F.max_list ? M.cnt[IM_MC_REMOVE] : F.max_list;
    if (e < nr) { chg_touch(F, F.rem_tri[e]); return; }
    e -= nr;
    const int t = tri_find(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2]);
    if (t >= 0) chg_touch(F, t);
}
IM_HD int chg_gather_count(const MeshDev& M, const FrameBuf& F) {
    const int nr = M.cnt[IM_MC_REMOVE] < F.max_list ? M.cnt[IM_MC_REMOVE] : F.max_list;
    const int na = M.cnt[IM_MC_ADD] < F.max_list ? M.cnt[IM_MC_ADD] : F.max_list;
    return nr + na;
}
// the frame lists its slots by the sweep: a batched frame (full), or a touched list that overflowed
IM_HD bool chg_sweeping(const FrameBuf& F, bool full) { return full || F.chg_cnt[IM_CH_TOUCHED] > F.chg_cap; }
IM_HD int chg_listed(const FrameBuf& F, bool full) { return chg_sweeping(F, full) ? F.chg_cnt[IM_CH_SWEPT] : F.chg_cnt[IM_CH_TOUCHED]; }
IM_HD void chg_sweep_slot(const MeshDev& M, const FrameBuf& F, const ChgDev& C, int t) {
    const unsigned char now = chg_state(M, t);
    if (now == C.pub[t]) return;
    const int e = im_atomic_add(&F.chg_cnt[IM_CH_SWEPT], 1);
    if (e < F.chg_cap) F.chg_list[e] = t;
    else C.pub[t] = now;   // the frame is lost to the feed, but the published state stays that of the store
}
// lost to the feed: more listed slots than the list holds, or more rows than the ring
IM_HD bool chg_lost(const FrameBuf& F, const ChgDev& C, bool full) {
    return chg_listed(F, full) > F.chg_cap || (long long)F.chg_cnt[IM_CH_ROWS] > C.max_rows;
}
// listed slot i: its row (w = code, -1: none) into marked[i], its published byte updated
IM_HD void chg_row_mark(const MeshDev& M, const FrameBuf& F, const ChgDev& C, int i) {
    const int t = F.chg_list[i];
    const unsigned char now = chg_state(M, t);
    const int code = chg_code(C.pub[t], now);
    int4 r = make_int4(0, 0, 0, -1);
    if (code >= 0) {
        C.pub[t] = now;
        r = M.tri[t];
        r.w = code;
    }
    C.marked[i] = r;
}
// compaction of the marked rows in list order: 1 when entry i is a row (count), then the row at position pos (emit)
IM_HD int chg_row_count(const ChgDev& C, int i) { return C.marked[i].w >= 0 ? 1 : 0; }
IM_HD int chg_row_emit(const ChgDev& C, int i, int pos) {
    const int4 r = C.marked[i];
    if (r.w < 0) return 0;
    C.rowbuf[pos] = r;
    return 1;
}
// LSD sort word w of row v: the triple's c, b, a
IM_HD unsigned int chg_word(const ChgDev& C, int w, int v) {
    const int4 r = C.rowbuf[v];
    return (unsigned int)(w == 0 ? r.z : w == 1 ? r.y : r.x);
}
// row i of the frame in ascending triple order (order: positions in rowbuf) into the ring
IM_HD void chg_append(const ChgDev& C, const unsigned int* order, int i) {
    C.ring[(*C.written + i) % C.max_rows] = C.rowbuf[order[i]];
}
// after the rows: the frame's header, the ring position, the counters cleared for the next frame.  v_after: the vertex counter
// already includes the frame's new vertices (the batched frame's end)
IM_HD void chg_frame_end(const MeshDev& M, const FrameBuf& F, const ChgDev& C, bool full, bool v_after) {
    ChgHdr h;
    h.frame = F.frame;
    const long long nv = M.cnt[IM_MC_NEW_VERTICES];
    h.v_begin = v_after ? M.cnt[IM_MC_VERTICES] - nv : M.cnt[IM_MC_VERTICES];
    h.v_end = h.v_begin + nv;
    h.lost = chg_lost(F, C, full) ? 1 : 0;
    h.r_begin = *C.written;
    h.r_end = h.r_begin + (h.lost ? 0 : F.chg_cnt[IM_CH_ROWS]);
    C.hdr[F.frame % C.max_frames] = h;
    *C.written = h.r_end;
    F.chg_cnt[IM_CH_TOUCHED] = 0; F.chg_cnt[IM_CH_SWEPT] = 0; F.chg_cnt[IM_CH_ROWS] = 0;
}

}  // namespace immesh
