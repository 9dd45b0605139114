// immesh_b200 -- the two per-voxel thread-block stages of the incremental mesher:
//   stage A  voxel_dilate : in-voxel vertices -> exact 20-NN each (ring-expanding neighbourhood gather staged
//                           in shared memory) -> dilated vertex set + smoothed positions
//                           (retrieve_pts_in_voxels + retrieve_neighbor_pts_kdtree)
//   stage B  voxel_mesh   : PCA -> 2-D projection -> exact Delaunay -> 150-degree filter -> pull / commit ->
//                           add / remove lists + orientation flags (delaunay_triangulation, triangle_compare,
//                           correct_triangle_index)
// Stage A of every voxel completes before stage B of any voxel starts (kernel boundary), which is the defined
// replacement of the reference's racy smoothing / orientation interplay (DESIGN.md).
#pragma once
#include "mesh_core.cuh"

namespace immesh {

#if defined(__CUDA_ARCH__)
#define IM_NLANES 32
IM_HD void warp_min_pair(float* d, int* id, int* aux) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, *d, o);
        const int oi = __shfl_xor_sync(0xffffffffu, *id, o);
        const int oa = __shfl_xor_sync(0xffffffffu, *aux, o);
        if (od < *d || (od == *d && oi < *id)) { *d = od; *id = oi; *aux = oa; }
    }
}
IM_HD unsigned im_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
IM_HD unsigned im_lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
#else
#define IM_NLANES 1
IM_HD void warp_min_pair(float*, int*, int*) {}
IM_HD unsigned im_ballot(bool p) { return p ? 1u : 0u; }
IM_HD unsigned im_lanemask_lt() { return 0u; }
#endif
IM_HD int im_popc(unsigned m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}

// ------------------------------------------------------------------ results of the per-voxel stage
// One GPU: applied directly.  Sharded (F.shard_n > 1): recorded in the exchange lists; every rank applies the
// all-gathered lists of all ranks to its replica (apply_*), so the replicas stay set-identical.
IM_HD void apply_face(const MeshDev& M, const FrameBuf& F, int a, int b, int c, unsigned long long word) {
    // commit, faces side (triangle_compare): a face already live in the store is "existing" (its flip priority word is
    // raised), otherwise it goes to the add list.  Batched frame: a triangle an earlier batch added is not "in the store" yet.
    const int t = tri_find(M, a, b, c);
    if (t >= 0 && M.tri[t].w && tri_pre_frame(F, t)) {
        im_atomic_max64(&M.tri_flip[t], word);
        chg_touch(F, t);   // its orientation may change
    } else {
        const int e = im_atomic_add(&M.cnt[IM_MC_ADD], 1);
        if (e < F.max_list) {
            F.add_tri[(size_t)e * 3 + 0] = a; F.add_tri[(size_t)e * 3 + 1] = b; F.add_tri[(size_t)e * 3 + 2] = c;
            F.add_flip[e] = word;
        } else {
            im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
        }
    }
}
IM_HD void emit_face(const MeshDev& M, const FrameBuf& F, int a, int b, int c, unsigned long long word) {
    if (F.shard_n > 1) {
        const int e = im_atomic_add(&M.cnt[IM_MC_X_FACES], 1);
        if (e < F.x_cap) { F.x_face[e] = make_int4(a, b, c, 0); F.x_word[e] = word; }
        else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
        return;
    }
    apply_face(M, F, a, b, c, word);
}
IM_HD void emit_remove(const MeshDev& M, const FrameBuf& F, int t) {
    if (F.shard_n > 1) {
        const int4 tr = M.tri[t];
        const int e = im_atomic_add(&M.cnt[IM_MC_X_REMS], 1);
        if (e < F.x_cap) F.x_rem[e] = make_int4(tr.x, tr.y, tr.z, 0); else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
        return;
    }
    if (F.tri_mark) {   // batched frame: counted now, removed after the last batch (only pre-frame triangles are pulled)
        im_atomic_add(&M.cnt[IM_MC_REMOVE], 1);
        F.tri_mark[t] = IM_TRI_REMOVE;
        return;
    }
    const int e = im_atomic_add(&M.cnt[IM_MC_REMOVE], 1);
    if (e < F.max_list) F.rem_tri[e] = t; else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
}
IM_HD void apply_remove(const MeshDev& M, const FrameBuf& F, int a, int b, int c) {
    const int t = tri_find(M, a, b, c);
    if (t < 0 || !M.tri[t].w) return;
    const int e = im_atomic_add(&M.cnt[IM_MC_REMOVE], 1);
    if (e < F.max_list) F.rem_tri[e] = t; else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
}
IM_HD void emit_smooth(const MeshDev& M, const FrameBuf& F, int v, double x, double y, double z) {
    store_smooth(M, v, x, y, z);
    if (F.shard_n > 1) {
        const int e = im_atomic_add(&M.cnt[IM_MC_X_SMOOTHS], 1);
        if (e < F.x_cap) { XSmooth r; r.id = v; r.pad = 0; r.x = x; r.y = y; r.z = z; F.x_smooth[e] = r; }
        else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
    }
}

struct DilateSmem {
    float4 cand[IM_MAXG];      // gathered neighbourhood vertices: xyz + id (bit-cast in w)
    unsigned char flag[IM_MAXG];  // member of the dilated set (byte stores of 1 only, so concurrent warps do not race)
    int cell_slot[344];        // per shell cell: voxel slot (-1 none) / running candidate offset
    int cell_off[344];
    int q[IM_MAXIN];           // in-voxel vertex ids (the kNN queries)
    int qdone[IM_MAXIN];       // query finished at an earlier ring (its 20-NN are provably complete)
    int ids[IM_MAXD];          // output, ascending
    int n_cand, n_q, n_out, need_more, overflow;
    // per-warp scratch of the kNN fast path: compacted (d2 bits << 32 | id) keys + candidate indices, ranked output
    unsigned long long wl_key[4][64];
    unsigned short wl_idx[4][64];
    float wl_outd[4][20];
    unsigned short wl_outi[4][20];
};

IM_HD int f2i(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_int(f);
#else
    int i; memcpy(&i, &f, 4); return i;
#endif
}
IM_HD float i2f(int i) {
#if defined(__CUDA_ARCH__)
    return __int_as_float(i);
#else
    float f; memcpy(&f, &i, 4); return f;
#endif
}

// deterministic gather of the shell of Chebyshev radius `ring` around voxel (kx,ky,kz) behind the candidates already staged:
// cells in lexicographic order, a cell's vertices in chunk order -> every block working on the same voxel in this frame builds
// the identical candidate array (indices are shared through a per-voxel bitmap)
IM_HDN inline void dilate_gather_ring(const MeshDev& M, DilateSmem* S, int kx, int ky, int kz, int ring, int tid, int nthreads) {
    const int side = 2 * ring + 1, ncell = side * side * side;
    for (int c = tid; c < ncell; c += nthreads) {
        const int dx = c / (side * side) - ring, dy = (c / side) % side - ring, dz = c % side - ring;
        const int ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy, az = dz < 0 ? -dz : dz;
        int slot = -1, cntv = 0;
        if ((ax > ay ? (ax > az ? ax : az) : (ay > az ? ay : az)) == ring && ikey_ok(kx + dx, ky + dy, kz + dz)) {
            slot = table_find(M.vkeys, M.vmask, pack_ikey(kx + dx, ky + dy, kz + dz));
            if (slot >= 0) {
                cntv = M.vox_count[slot];
                if (cntv > IM_VCHUNKS * 16) cntv = IM_VCHUNKS * 16;
            }
        }
        S->cell_slot[c] = slot;
        S->cell_off[c] = cntv;
    }
    IM_SYNCBLOCK_M();
    if (tid == 0) {
        int run = S->n_cand;
        for (int c = 0; c < ncell; ++c) { const int k = S->cell_off[c]; S->cell_off[c] = run; run += k; }
        S->cell_off[ncell] = run;
        if (run > IM_MAXG) S->overflow = 1;
        S->n_cand = run < IM_MAXG ? run : IM_MAXG;
    }
    IM_SYNCBLOCK_M();
    for (int c = tid; c < ncell; c += nthreads) {
        const int slot = S->cell_slot[c];
        if (slot < 0) continue;
        const int o = S->cell_off[c], cntv = S->cell_off[c + 1] - o;
        for (int k = 0; k < cntv; ++k)
            if (o + k < IM_MAXG) S->cand[o + k] = M.vchunk_pts[(size_t)im_chunk_or0(M.vox_chunk[(size_t)slot * IM_VCHUNKS + (k >> 4)]) * 16 + (k & 15)];
    }
    IM_SYNCBLOCK_M();
}

// stage A for one dilation item = (work slot w, group g of up to 8 queries).  All groups of a voxel stage the same
// candidate array; each runs the exact 20-NN of its own queries and ORs the indices of the dilation members into the
// voxel's global bitmap; the last group to finish turns the bitmap into the ascending id list of the dilated set.
IM_HDN inline void voxel_dilate(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int item, DilateSmem* S, int tid, int nthreads) {
    const int w = item >> 5, grp = item & 31;
    const int vs = F.work[w];
    int kx, ky, kz;
    unpack_ikey(M.vkeys[vs], &kx, &ky, &kz);
    if (tid == 0) { S->n_cand = 0; S->n_q = 0; S->n_out = 0; S->overflow = 0; }
    IM_SYNCBLOCK_M();
    // ring 0 = the voxel's own vertices (retrieve_pts_in_voxels): candidates for everybody, queries for their group
    int nqt = M.vox_count[vs];
    if (nqt > IM_VCHUNKS * 16) nqt = IM_VCHUNKS * 16;
    if (nqt > IM_MAXIN) { nqt = IM_MAXIN; if (tid == 0) S->overflow = 1; }
    for (int k = tid; k < nqt; k += nthreads) {
        const float4 p = M.vchunk_pts[(size_t)im_chunk_or0(M.vox_chunk[(size_t)vs * IM_VCHUNKS + (k >> 4)]) * 16 + (k & 15)];
        S->q[k] = f2i(p.w);
        S->cand[k] = p;
    }
    if (tid == 0) { S->n_q = nqt; S->n_cand = nqt; }
    IM_SYNCBLOCK_M();
    const int ngroups = (nqt + 7) >> 3;
    const int q_lo = grp * 8, q_hi = (q_lo + 8 < nqt) ? q_lo + 8 : nqt;
    for (int i = tid; i < nqt; i += nthreads) { S->qdone[i] = 0; S->flag[i] = 0; }
    int flag_init = nqt;   // candidates [0, flag_init) have an initialised flag
    const double max_d2 = P.knn_max * P.knn_max;
    const int lane = tid % IM_NLANES, warp = tid / IM_NLANES, nwarps = (nthreads + IM_NLANES - 1) / IM_NLANES;
    int ring_used = 0;
    for (int ring = 1; ring <= 3; ++ring) {
        dilate_gather_ring(M, S, kx, ky, kz, ring, tid, nthreads);
        ring_used = ring;
        const int nc = S->n_cand < IM_MAXG ? S->n_cand : IM_MAXG;
        for (int i = flag_init + tid; i < nc; i += nthreads) S->flag[i] = 0;
        flag_init = nc;
        if (tid == 0) S->need_more = 0;
        IM_SYNCBLOCK_M();
        // after gathering rings 0..ring, every unseen vertex is at least ring*res away from any query of this voxel
        const double lb = (double)ring * P.res;
        for (int qi = q_lo + warp; qi < q_hi; qi += nwarps) {
            if (S->qdone[qi]) continue;   // complete at an earlier ring: more candidates cannot change its 20-NN
            const int qv = S->q[qi];
            const float4 qp = M.vpos[qv];
#if defined(__CUDA_ARCH__)
            {
                // Warp-cooperative exact 20-NN.  Candidates are consumed in chunks of 512: every lane holds the squared
                // distances of its <= 16 chunk candidates in registers (computed once) plus, as a 17th slot, the entry of the
                // running best-20 list it carries (lane r carries the r-th nearest so far).  Per chunk, 20 rounds of warp
                // arg-min on (d2, id) over the lanes' current minima rebuild the best-20 list; the winning lane retires its
                // entry and rescans its slots.
                float cd = INFINITY;           // carried list entry of this lane
                int cid = 0x7fffffff, cidx = 0, have = 0;
                // Fast path.  The 20 nearest are the 20 smallest (d2, id) keys of ANY candidate subset {d2 <= T} that holds
                // at least 20 of them, so: count the candidates under a ladder of radii (one pass), compact those under the
                // first radius with >= 20 members (normally 20..40 of ~400) into a per-warp list, and rank the list by
                // all-pairs comparison of its 64-bit keys -- no serial selection rounds.  Lists longer than 64 fall through
                // to the general chunked selection below.
                bool fast_done = false;
                {
                    const float r2 = (float)(P.res * P.res);
                    float mf = (float)max_d2;                    // dd <= mf  <=>  (double)dd <= max_d2
                    if ((double)mf > max_d2) mf = __uint_as_float(__float_as_uint(mf) - 1u);
                    const float T0 = 0.30f * r2, T1 = 0.49f * r2, T2 = 0.72f * r2, T3 = 1.0f * r2, T4 = 2.25f * r2;
                    int c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0;
                    for (int i = lane; i < nc; i += 32) {
                        const float4 cp = S->cand[i];
                        const float dd = dist2f(qp.x, qp.y, qp.z, cp.x, cp.y, cp.z);
                        c0 += (dd <= T0); c1 += (dd <= T1); c2 += (dd <= T2); c3 += (dd <= T3); c4 += (dd <= T4); c5 += (dd <= mf);
                    }
                    c0 = __reduce_add_sync(0xffffffffu, c0); c1 = __reduce_add_sync(0xffffffffu, c1);
                    c2 = __reduce_add_sync(0xffffffffu, c2); c3 = __reduce_add_sync(0xffffffffu, c3);
                    c4 = __reduce_add_sync(0xffffffffu, c4); c5 = __reduce_add_sync(0xffffffffu, c5);
                    float T = mf; int C = c5;
                    if (c4 >= 20) { T = T4; C = c4; }
                    if (c3 >= 20) { T = T3; C = c3; }
                    if (c2 >= 20) { T = T2; C = c2; }
                    if (c1 >= 20) { T = T1; C = c1; }
                    if (c0 >= 20) { T = T0; C = c0; }
                    if (T > mf) { T = mf; C = c5; }
                    if (C <= 64) {
                        unsigned long long* wkey = S->wl_key[warp];
                        unsigned short* widx = S->wl_idx[warp];
                        const unsigned lt = im_lanemask_lt();
                        int pos = 0;
                        for (int i0 = 0; i0 < nc; i0 += 32) {
                            const int i = i0 + lane;
                            bool in = false;
                            float dd = 0.f;
                            int id = 0;
                            if (i < nc) {
                                const float4 cp = S->cand[i];
                                dd = dist2f(qp.x, qp.y, qp.z, cp.x, cp.y, cp.z);
                                id = f2i(cp.w);
                                in = dd <= T;
                            }
                            const unsigned m = __ballot_sync(0xffffffffu, in);
                            if (in) {
                                const int k = pos + __popc(m & lt);
                                wkey[k] = ((unsigned long long)__float_as_uint(dd) << 32) | (unsigned int)id;
                                widx[k] = (unsigned short)i;
                            }
                            pos += __popc(m);
                        }
                        __syncwarp();
                        const unsigned long long k0 = (lane < C) ? wkey[lane] : ~0ull, k1 = (lane + 32 < C) ? wkey[lane + 32] : ~0ull;
                        int rk0 = 0, rk1 = 0;
                        for (int j = 0; j < C; ++j) {
                            const unsigned long long kj = wkey[j];
                            rk0 += (kj < k0); rk1 += (kj < k1);
                        }
                        if (lane < C && rk0 < 20) { S->wl_outd[warp][rk0] = __uint_as_float((unsigned int)(k0 >> 32)); S->wl_outi[warp][rk0] = widx[lane]; }
                        if (lane + 32 < C && rk1 < 20) { S->wl_outd[warp][rk1] = __uint_as_float((unsigned int)(k1 >> 32)); S->wl_outi[warp][rk1] = widx[lane + 32]; }
                        __syncwarp();
                        have = C < 20 ? C : 20;
                        if (lane < have) { cd = S->wl_outd[warp][lane]; cidx = S->wl_outi[warp][lane]; }
                        __syncwarp();
                        fast_done = true;
                    }
                }
                for (int base = 0; base < nc && !fast_done; base += 512) {
                    float dreg[17];
                    int ireg[17];
                    const int nsl = (min(nc - base, 512) + 31) >> 5;   // occupied register slots (warp-uniform)
#pragma unroll
                    for (int sl = 0; sl < 16; ++sl) {
                        const int i = base + lane + 32 * sl;
                        float d2 = INFINITY;
                        int id = 0x7fffffff;
                        if (sl < nsl && i < nc) {
                            const float4 cp = S->cand[i];
                            const float dd = dist2f(qp.x, qp.y, qp.z, cp.x, cp.y, cp.z);
                            if ((double)dd <= max_d2) { d2 = dd; id = f2i(cp.w); }
                        }
                        dreg[sl] = d2; ireg[sl] = id;
                    }
                    dreg[16] = (lane < have) ? cd : INFINITY;
                    ireg[16] = (lane < have) ? cid : 0x7fffffff;
                    float nd = INFINITY;
                    int nid = 0x7fffffff, nidx = 0, found = 0;
                    for (int r = 0; r < 20; ++r) {
                        float bd = dreg[16];
                        int bid = ireg[16], bsl = 16;
#pragma unroll
                        for (int sl = 0; sl < 16; ++sl)
                            if (sl < nsl && (dreg[sl] < bd || (dreg[sl] == bd && ireg[sl] < bid))) { bd = dreg[sl]; bid = ireg[sl]; bsl = sl; }
                        // aux packs the winner's candidate index (11 bits), slot (5 bits) and lane (5 bits)
                        int aux = ((bsl == 16) ? cidx : (base + bsl * 32 + lane)) | (bsl << 11) | (lane << 16);
                        warp_min_pair(&bd, &bid, &aux);
                        if (bid == 0x7fffffff) break;
                        if ((aux >> 16) == lane) {
                            const int wsl = (aux >> 11) & 31;
#pragma unroll
                            for (int sl = 0; sl < 17; ++sl)
                                if (sl == wsl) { dreg[sl] = INFINITY; ireg[sl] = 0x7fffffff; }
                        }
                        if (lane == r) { nd = bd; nid = bid; nidx = aux & 2047; }
                        ++found;
                    }
                    cd = nd; cid = nid; cidx = nidx; have = found;
                }
                // ordered pass over the final list: dilation membership and the smoothing mean (ascending distance)
                double sv0 = 0.0, sv1 = 0.0, sv2 = 0.0;
                int cnt = 0;
                float last_d = 0.f;
                if (have > 0) last_d = __shfl_sync(0xffffffffu, cd, have - 1);
                {
                    const unsigned m2 = __ballot_sync(0xffffffffu, lane < have && (double)sqrtf(cd) < P.accept * 2);
                    cnt = __popc(m2);
                    const float4 mine = S->cand[cidx];
                    for (unsigned mm = m2; mm; mm &= mm - 1) {
                        const int r = __ffs(mm) - 1;
                        const float x = __shfl_sync(0xffffffffu, mine.x, r), y = __shfl_sync(0xffffffffu, mine.y, r), z = __shfl_sync(0xffffffffu, mine.z, r);
                        sv0 = sv0 + (double)x; sv1 = sv1 + (double)y; sv2 = sv2 + (double)z;
                    }
                }
                const bool complete = (lb > P.knn_max) || (have >= 20 && (double)last_d < lb * lb * 0.999999);
                if (!complete) {
                    if (lane == 0) S->need_more = 1;   // retried with the next ring; nothing is published yet
                } else {
                    if (lane < have && (double)sqrtf(cd) < P.accept) S->flag[cidx] = 1;
                    if (lane == 0) {
                        S->qdone[qi] = 1;
                        emit_smooth(M, F, qv, (sv0 / (double)cnt) * (double)1.0f + (double)qp.x * (double)(1 - 1.0f),
                                    (sv1 / (double)cnt) * (double)1.0f + (double)qp.y * (double)(1 - 1.0f),
                                    (sv2 / (double)cnt) * (double)1.0f + (double)qp.z * (double)(1 - 1.0f));
                    }
                }
                continue;
            }
#endif
            float prev_d = -1.0f;
            int prev_id = -1;
            double sv0 = 0.0, sv1 = 0.0, sv2 = 0.0;
            int cnt = 0, found = 0;
            float last_d = 0.f;
            int widx_a[20];
            float wd_a[20];
            for (int r = 0; r < 20; ++r) {
                float bd = INFINITY;
                int bid = 0x7fffffff, bidx = -1;
                for (int i = lane; i < nc; i += IM_NLANES) {
                    const float4 cp = S->cand[i];
                    const float d2 = dist2f(qp.x, qp.y, qp.z, cp.x, cp.y, cp.z);
                    const int id = f2i(cp.w);
                    if (!((double)d2 <= max_d2)) continue;
                    if (d2 < prev_d || (d2 == prev_d && id <= prev_id)) continue;  // already reported
                    if (d2 < bd || (d2 == bd && id < bid)) { bd = d2; bid = id; bidx = i; }
                }
                warp_min_pair(&bd, &bid, &bidx);
                if (bidx < 0) break;
                prev_d = bd; prev_id = bid;
                last_d = bd;
                widx_a[found] = bidx; wd_a[found] = bd;
                ++found;
                const float sd = sqrtf(bd);
                if ((double)sd < P.accept * 2) {
                    ++cnt;
                    const float4 cp = S->cand[bidx];
                    sv0 = sv0 + (double)cp.x; sv1 = sv1 + (double)cp.y; sv2 = sv2 + (double)cp.z;
                }
            }
            const bool complete = (lb > P.knn_max) || (found >= 20 && (double)last_d < lb * lb * 0.999999);
            if (!complete) {
                if (lane == 0) S->need_more = 1;
            } else if (lane == 0) {
                for (int r = 0; r < found; ++r)
                    if ((double)sqrtf(wd_a[r]) < P.accept) S->flag[widx_a[r]] = 1;
                S->qdone[qi] = 1;
                // smooth_factor = 1.0f (mesh_rec_geometry.cpp:334,367-369)
                emit_smooth(M, F, qv, (sv0 / (double)cnt) * (double)1.0f + (double)qp.x * (double)(1 - 1.0f),
                            (sv1 / (double)cnt) * (double)1.0f + (double)qp.y * (double)(1 - 1.0f),
                            (sv2 / (double)cnt) * (double)1.0f + (double)qp.z * (double)(1 - 1.0f));
            }
        }
        IM_SYNCBLOCK_M();
        if (!S->need_more) break;
    }
    // publish this group's dilation members in the voxel's bitmap
    {
        const int nc = S->n_cand < IM_MAXG ? S->n_cand : IM_MAXG;
        unsigned int* bits = F.work_bits + (size_t)w * (IM_MAXG / 32);
        for (int i = tid; i < nc; i += nthreads)
            if (S->flag[i]) {
#if defined(__CUDA_ARCH__)
                atomicOr(&bits[i >> 5], 1u << (i & 31));
#else
                bits[i >> 5] |= 1u << (i & 31);
#endif
            }
        if (tid == 0) {
            im_atomic_max(&F.work_ring[w], ring_used);
            if (S->overflow) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VOXEL_CAP);
        }
    }
    im_fence();
    IM_SYNCBLOCK_M();
    if (tid == 0) S->need_more = (im_atomic_add(&F.work_done[w], 1) == ngroups - 1) ? 1 : 0;
    IM_SYNCBLOCK_M();
    if (!S->need_more) return;
    // ---- last group of the voxel: dilated set = union of all groups' members, ascending by id (std::set<long>,
    // ImMesh_mesh_reconstruction.cpp:157-170)
    im_fence();
    const int ring_all = im_vload(&F.work_ring[w]);
    for (int ring = ring_used + 1; ring <= ring_all; ++ring) dilate_gather_ring(M, S, kx, ky, kz, ring, tid, nthreads);
    {
        const int nc = S->n_cand < IM_MAXG ? S->n_cand : IM_MAXG;
        unsigned int* bits = F.work_bits + (size_t)w * (IM_MAXG / 32);
        for (int i = tid; i < nc; i += nthreads) {
            const unsigned int word = (unsigned int)im_vload((const int*)&bits[i >> 5]);
            if ((word >> (i & 31)) & 1u) {
                const int k = im_atomic_add(&S->n_out, 1);
                if (k < IM_MAXD) S->ids[k] = f2i(S->cand[i].w); else S->overflow = 1;
            }
        }
        IM_SYNCBLOCK_M();
        for (int i = tid; i < IM_MAXG / 32; i += nthreads) bits[i] = 0u;   // clean for the next frame
        if (tid == 0) { F.work_ring[w] = 0; F.work_done[w] = 0; }
    }
    IM_SYNCBLOCK_M();
    int n = S->n_out < IM_MAXD ? S->n_out : IM_MAXD;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = n + tid; i < np2; i += nthreads) S->ids[i] = 0x7fffffff;
    IM_SYNCBLOCK_M();
    for (int k = 2; k <= np2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < np2; i += nthreads) {
                const int l = i ^ j;
                if (l > i) {
                    const int a = S->ids[i], b = S->ids[l];
                    const bool up = ((i & k) == 0);
                    if ((a > b) == up) { S->ids[i] = b; S->ids[l] = a; }
                }
            }
            IM_SYNCBLOCK_M();
        }
    for (int i = tid; i < n; i += nthreads) F.work_ids[(size_t)w * IM_MAXD + i] = S->ids[i];
    // frame-wide list of (voxel, dilated vertex) references for the flat pull stage
    if (tid == 0) S->need_more = (n >= 3) ? im_atomic_add(&M.cnt[IM_MC_VREFS], n) : -1;
    IM_SYNCBLOCK_M();
    {
        const int voff = S->need_more;
        if (voff >= 0) {
            if (voff + n > F.max_vref) { if (tid == 0) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); }
            else for (int i = tid; i < n; i += nthreads) F.all_vref[voff + i] = (w << 10) | i;
        }
    }
    if (tid == 0) {
        F.work_nfaces[w] = 0;
        F.work_n_ids[w] = n;
        if (S->overflow) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VOXEL_CAP);
        // work accounting for the roofline (DESIGN.md): gathered candidates, queries, dilated vertices
        im_atomic_add(&M.cnt[IM_MC_STAT_GATHERED], S->n_cand);
        im_atomic_add(&M.cnt[IM_MC_STAT_QUERIES], nqt);
        im_atomic_add(&M.cnt[IM_MC_STAT_DILATED], n);
    }
}

// ------------------------------------------------------------------ stage B
// commit (triangle_compare) + orientation (correct_triangle_index) + pull (find_relative_triangulation_combination) of one
// voxel, given its ascending dilated id list, its new facets (sorted id triples) and a hash set over them.
IM_HDN inline void voxel_commit_common(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int w, int n, const int* ids, int nf,
                                       const int (*faces)[3], const int* fhash, unsigned int hmask, const double* axes, int tid, int nthreads) {
    const unsigned long long prio = voxel_prio(M, F, w, tid == 0);
    const unsigned long long word_base = ((unsigned long long)F.frame << 34) | (prio << 1);
    // commit, faces side (triangle_compare): a face already live in the store is "existing", otherwise "to add"
    for (int k = tid; k < nf; k += nthreads) {
        const int a = faces[k][0], b = faces[k][1], c = faces[k][2];
        const unsigned long long word = word_base | (unsigned long long)compute_flip(M, a, b, c, F.fp->pose_t, axes);
        emit_face(M, F, a, b, c, word);
    }
    // pull (find_relative_triangulation_combination) + commit, store side: live triangles with all three vertices in
    // the dilated set that the new triangulation does not contain are removed.  Each triangle is visited from its
    // smallest vertex only.
    for (int i = tid; i < n; i += nthreads) {
        const int v = ids[i];
        for (int t = M.v_tri_head[v]; t >= 0;) {
            const int4 r = M.tri[t];
            const int slot = (r.x == v) ? 0 : ((r.y == v) ? 1 : 2);
            const int nx = M.tri_next[(size_t)t * 3 + slot];
            if (r.w && r.x == v && tri_pre_frame(F, t)) {
                // binary search y and z in the ascending id list
                bool in_set = true;
                for (int pass = 0; pass < 2 && in_set; ++pass) {
                    const int key = pass == 0 ? r.y : r.z;
                    int lo = 0, hi = n - 1;
                    bool hit = false;
                    while (lo <= hi) {
                        const int mid = (lo + hi) >> 1;
                        const int val = ids[mid];
                        if (val == key) { hit = true; break; }
                        if (val < key) lo = mid + 1; else hi = mid - 1;
                    }
                    in_set = hit;
                }
                if (in_set) {
                    bool in_new = false;
                    unsigned int hs = tri_hash(r.x, r.y, r.z) & hmask;
                    for (int probe = 0; probe <= (int)hmask; ++probe) {
                        const int k = fhash[hs];
                        if (k < 0) break;
                        if (faces[k][0] == r.x && faces[k][1] == r.y && faces[k][2] == r.z) { in_new = true; break; }
                        hs = (hs + 1) & hmask;
                    }
                    if (!in_new) emit_remove(M, F, t);
                }
            }
            t = nx;
        }
    }
}

template <int MAXD>
struct MeshSmem {
    int ids[MAXD];
    float pos[MAXD][3];
    double uv[MAXD][2];
    int2 snap[MAXD];
    DTri tris[3 * MAXD + 8];
    int faces[2 * MAXD][3];       // global ids, a<b<c
    int fhash[4 * MAXD];          // open-addressed set of face indices
    int scratch[8 + 256 + 520];
    float circ[(MAXD <= 256) ? (3 * MAXD + 8) : 1][3];   // circumcircle cache (mid-size variant only)
    double axes[9];               // short, mid, long
    double centre[3];
    int ntri, nface;
};

template <int MAXD>
IM_HDN inline void voxel_mesh(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int w, MeshSmem<MAXD>* S, int tid, int nthreads, int store_only = 0) {
    const int nraw = F.work_n_ids[w];
    const int n = nraw < 0 ? -nraw : nraw;   // negative: handed over to the large variant after a capacity overflow
    if (store_only && tid == 0) F.work_nfaces[w] = (n > MAXD) ? -1 : 0;   // -1: left to the large (monolithic) variant
    if (n < 3 || n > MAXD) return;
    for (int i = tid; i < n; i += nthreads) {
        const int id = F.work_ids[(size_t)w * IM_MAXD + i];
        S->ids[i] = id;
        const float4 p = M.vpos[id];
        S->pos[i][0] = p.x; S->pos[i][1] = p.y; S->pos[i][2] = p.z;
    }
    if (!store_only) for (int i = tid; i < 4 * MAXD; i += nthreads) S->fhash[i] = -1;
    if (tid == 0) S->nface = 0;
    IM_SYNCBLOCK_M();
    if (tid == 0) {
        // centroid, covariance, principal axes (mesh_rec_geometry.cpp:193-213); sequential sums: bit-reproducible
        double c[3] = {0, 0, 0};
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < 3; ++j) c[j] = c[j] + (double)S->pos[i][j];
        for (int j = 0; j < 3; ++j) c[j] = c[j] / (double)n;
        double cov[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < n; ++i) {
            const double d[3] = {(double)S->pos[i][0] - c[0], (double)S->pos[i][1] - c[1], (double)S->pos[i][2] - c[2]};
            cov[0] += d[0] * d[0]; cov[1] += d[0] * d[1]; cov[2] += d[0] * d[2];
            cov[3] += d[1] * d[1]; cov[4] += d[1] * d[2]; cov[5] += d[2] * d[2];
        }
        for (int k = 0; k < 6; ++k) cov[k] = cov[k] / (double)n;
        double ev[3], U[9];
        jacobi3(cov, ev, U);
        int order[3];  // ascending eigenvalues (SelfAdjointEigenSolver order)
        order3(ev, order);
        double s[3], m[3];
        for (int j = 0; j < 3; ++j) { s[j] = col3(U, j, order[0]); m[j] = col3(U, j, order[1]); }
        const double d0[3] = {(double)S->pos[0][0] - c[0], (double)S->pos[0][1] - c[1], (double)S->pos[0][2] - c[2]};
        const double d1[3] = {(double)S->pos[1][0] - c[0], (double)S->pos[1][1] - c[1], (double)S->pos[1][2] - c[2]};
        if (dot3(d0, s) < 0) { s[0] = -s[0]; s[1] = -s[1]; s[2] = -s[2]; }
        if (dot3(d1, m) < 0) { m[0] = -m[0]; m[1] = -m[1]; m[2] = -m[2]; }
        S->axes[0] = s[0]; S->axes[1] = s[1]; S->axes[2] = s[2];
        S->axes[3] = m[0]; S->axes[4] = m[1]; S->axes[5] = m[2];
        S->axes[6] = s[1] * m[2] - s[2] * m[1];
        S->axes[7] = s[2] * m[0] - s[0] * m[2];
        S->axes[8] = s[0] * m[1] - s[1] * m[0];
        S->centre[0] = c[0]; S->centre[1] = c[1]; S->centre[2] = c[2];
    }
    IM_SYNCBLOCK_M();
    for (int i = tid; i < n; i += nthreads) {
        const double d[3] = {(double)S->pos[i][0] - S->centre[0], (double)S->pos[i][1] - S->centre[1], (double)S->pos[i][2] - S->centre[2]};
        const double u = dot3(d, S->axes + 6), v = dot3(d, S->axes + 3);
        S->uv[i][0] = u; S->uv[i][1] = v;
        S->snap[i] = make_int2((int)im_llrint(u * P.inv_q), (int)im_llrint(v * P.inv_q));
    }
    IM_SYNCBLOCK_M();
    delaunay_block(S->snap, n, S->tris, 3 * MAXD + 8, &S->ntri, S->scratch, tid, nthreads, (MAXD <= 256) ? S->circ : nullptr);
    IM_SYNCBLOCK_M();
    if (S->scratch[4] == 0) return;  // all points collinear: T.number_of_faces() == 0 (mesh_rec_geometry.cpp:257-260)
    if (S->scratch[6]) {   // cavity capacity exceeded
        if (store_only) { if (tid == 0) { F.work_nfaces[w] = -1; F.work_n_ids[w] = -n; } }
        else if (tid == 0) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VOXEL_CAP);
        return;
    }
    // finite faces passing the 150-degree filter (is_face_is_ok), as sorted global id triples
    const int nt = S->ntri;
    for (int t = tid; t < nt; t += nthreads) {
        const DTri& tr = S->tris[t];
        if (!tr.alive || tr.v[0] < 0 || tr.v[1] < 0 || tr.v[2] < 0) continue;
        const int i0 = tr.v[0], i1 = tr.v[1], i2 = tr.v[2];
        if (angle_bad(S->uv[i0][0], S->uv[i0][1], S->uv[i1][0], S->uv[i1][1], S->uv[i2][0], S->uv[i2][1])) continue;
        if (angle_bad(S->uv[i1][0], S->uv[i1][1], S->uv[i2][0], S->uv[i2][1], S->uv[i0][0], S->uv[i0][1])) continue;
        if (angle_bad(S->uv[i2][0], S->uv[i2][1], S->uv[i0][0], S->uv[i0][1], S->uv[i1][0], S->uv[i1][1])) continue;
        int a = S->ids[i0], b = S->ids[i1], c = S->ids[i2];
        if (a > b) { const int x = a; a = b; b = x; }
        if (b > c) { const int x = b; b = c; c = x; }
        if (a > b) { const int x = a; a = b; b = x; }
        const int k = im_atomic_add(&S->nface, 1);
        S->faces[k][0] = a; S->faces[k][1] = b; S->faces[k][2] = c;
        if (!store_only) {   // the monolithic variant looks new facets up in shared memory; the fused path uses the frame-wide set
            unsigned int hs = tri_hash(a, b, c) & (4 * MAXD - 1);
            while (im_atomic_cas32(&S->fhash[hs], -1, k) != -1) hs = (hs + 1) & (4 * MAXD - 1);
        }
    }
    IM_SYNCBLOCK_M();
    const int nf = S->nface;
    if (tid == 0) im_atomic_add(&M.cnt[IM_MC_STAT_FACETS], nf);
    if (store_only) {
        // fused dilate+triangulate kernel: the facets and the voxel's principal axes go to global memory; commit / orientation
        // run in a later kernel, once the smoothed positions of ALL voxels of the frame are final
        // compact frame-wide lists (arbitrary order): facets (a,b,c,w) and vertex references (w,i)
        if (tid == 0) S->scratch[0] = im_atomic_add(&M.cnt[IM_MC_FACES], nf);
        IM_SYNCBLOCK_M();
        const int foff = S->scratch[0];
        if (foff + nf > F.max_list) {
            if (tid == 0) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
        } else {
            for (int k = tid; k < nf; k += nthreads) F.all_faces[foff + k] = make_int4(S->faces[k][0], S->faces[k][1], S->faces[k][2], w);
        }
        for (int k = tid; k < 9; k += nthreads) F.work_axes[(size_t)w * 9 + k] = S->axes[k];
        if (tid == 0) F.work_nfaces[w] = nf;
        return;
    }
    voxel_commit_common(M, P, F, w, n, S->ids, nf, S->faces, S->fhash, 4 * MAXD - 1, S->axes, tid, nthreads);
}

// ------------------------------------------------------------------ stage B, warp-level variant (small dilated sets)
// One warp per voxel (n <= MAXD dilated vertices), __syncwarp only.  The Bowyer-Watson conflict search is pruned with a
// cached float circumcircle per triangle (conservative margin; every survivor still goes through the exact predicate),
// which removes ~90% of the exact in-circle evaluations.  Cavity / boundary capacity is 64 triangles; a voxel that
// exceeds it is handed to the large block-level variant (work_n_ids[w] negated).  Triangulation only: the facets go to
// the frame-wide lists, commit / orientation / pull are done by the flat stage-C kernels.
template <int MAXD>
struct MeshWarpSmem {
    int ids[MAXD];
    double uv[MAXD][2];
    int2 snap[MAXD];
    DTri tris[3 * MAXD + 8];          // after face extraction: reused as the face hash (4*MAXD ints)
    float circ[3 * MAXD + 8][3];      // before the triangulation: vertex positions; after it: faces (2*MAXD int3)
    int scratch[8 + 64 + 2 * 192];
    double axes[9];
    double centre[3];
    int ntri, nface;
};

template <int MAXD>
IM_HDN inline void voxel_mesh_warp(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int w, MeshWarpSmem<MAXD>* S, int lane, int nlanes, int n_max) {
    const int n = F.work_n_ids[w];
    if (n < 3 || n > n_max || n > MAXD) return;
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 32, n);
    float (*pos)[3] = S->circ;  // alias: positions are dead once projected
    for (int i = lane; i < n; i += nlanes) {
        const int id = F.work_ids[(size_t)w * IM_MAXD + i];
        S->ids[i] = id;
        const float4 p = M.vpos[id];
        pos[i][0] = p.x; pos[i][1] = p.y; pos[i][2] = p.z;
    }
    if (lane == 0) S->nface = 0;
    IM_SYNCWARP();
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 33, 0);
    if (lane == 0) {
        double c[3] = {0, 0, 0};
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < 3; ++j) c[j] = c[j] + (double)pos[i][j];
        for (int j = 0; j < 3; ++j) c[j] = c[j] / (double)n;
        double cov[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < n; ++i) {
            const double d[3] = {(double)pos[i][0] - c[0], (double)pos[i][1] - c[1], (double)pos[i][2] - c[2]};
            cov[0] += d[0] * d[0]; cov[1] += d[0] * d[1]; cov[2] += d[0] * d[2];
            cov[3] += d[1] * d[1]; cov[4] += d[1] * d[2]; cov[5] += d[2] * d[2];
        }
        for (int k = 0; k < 6; ++k) cov[k] = cov[k] / (double)n;
        IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 51, __double_as_longlong(cov[5] + cov[0]));
        double ev[3], U[9];
        jacobi3(cov, ev, U);
        IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 52, __double_as_longlong(ev[0] + U[8]));
        int order[3];
        order3(ev, order);
        double sx[3], m[3];
        for (int j = 0; j < 3; ++j) { sx[j] = col3(U, j, order[0]); m[j] = col3(U, j, order[1]); }
        const double d0[3] = {(double)pos[0][0] - c[0], (double)pos[0][1] - c[1], (double)pos[0][2] - c[2]};
        const double d1[3] = {(double)pos[1][0] - c[0], (double)pos[1][1] - c[1], (double)pos[1][2] - c[2]};
        if (dot3(d0, sx) < 0) { sx[0] = -sx[0]; sx[1] = -sx[1]; sx[2] = -sx[2]; }
        if (dot3(d1, m) < 0) { m[0] = -m[0]; m[1] = -m[1]; m[2] = -m[2]; }
        S->axes[0] = sx[0]; S->axes[1] = sx[1]; S->axes[2] = sx[2];
        S->axes[3] = m[0]; S->axes[4] = m[1]; S->axes[5] = m[2];
        S->axes[6] = sx[1] * m[2] - sx[2] * m[1];
        S->axes[7] = sx[2] * m[0] - sx[0] * m[2];
        S->axes[8] = sx[0] * m[1] - sx[1] * m[0];
        S->centre[0] = c[0]; S->centre[1] = c[1]; S->centre[2] = c[2];
    }
    IM_SYNCWARP();
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 34, 0);
    for (int i = lane; i < n; i += nlanes) {
        const double d[3] = {(double)pos[i][0] - S->centre[0], (double)pos[i][1] - S->centre[1], (double)pos[i][2] - S->centre[2]};
        const double u = dot3(d, S->axes + 6), v = dot3(d, S->axes + 3);
        S->uv[i][0] = u; S->uv[i][1] = v;
        S->snap[i] = make_int2((int)im_llrint(u * P.inv_q), (int)im_llrint(v * P.inv_q));
    }
    IM_SYNCWARP();
    // ---- Bowyer-Watson, warp-synchronous
    const int2* Pt = S->snap;
    DTri* tris = S->tris;
    int* s_cav_n = S->scratch;
    int* s_edge_n = S->scratch + 1;
    int* s_seed = S->scratch + 2;   // i1, i2, ok
    int* s_ovf = S->scratch + 6;
    int* s_cav = S->scratch + 8;    // [64]
    int* s_edges = S->scratch + 72; // [68*2]
    const int max_tris = 3 * MAXD + 8;
    if (lane == 0) {
        *s_ovf = 0;
        int i1 = -1, i2 = -1;
        for (int i = 1; i < n; ++i)
            if (Pt[i].x != Pt[0].x || Pt[i].y != Pt[0].y) { i1 = i; break; }
        if (i1 >= 0)
            for (int i = 1; i < n; ++i)
                if (i != i1 && orient2d_i(Pt[0].x, Pt[0].y, Pt[i1].x, Pt[i1].y, Pt[i].x, Pt[i].y) != 0) { i2 = i; break; }
        s_seed[0] = i1; s_seed[1] = i2; s_seed[2] = (i1 >= 0 && i2 >= 0) ? 1 : 0;
        S->ntri = 0;
        if (s_seed[2]) {
            int a = 0, b = i1, c = i2;
            if (orient2d_i(Pt[a].x, Pt[a].y, Pt[b].x, Pt[b].y, Pt[c].x, Pt[c].y) < 0) { const int t = b; b = c; c = t; }
            const short tv[4][3] = {{(short)a, (short)b, (short)c}, {(short)c, (short)b, IM_GHOST}, {(short)a, (short)c, IM_GHOST}, {(short)b, (short)a, IM_GHOST}};
            for (int k = 0; k < 4; ++k) { tris[k].v[0] = tv[k][0]; tris[k].v[1] = tv[k][1]; tris[k].v[2] = tv[k][2]; tris[k].alive = 1; }
            circumcircle_f(Pt, a, b, c, S->circ[0]);
            S->ntri = 4;
        }
    }
    IM_SYNCWARP();
    if (!s_seed[2]) return;
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 35, 0);
    const int i1 = s_seed[0], i2 = s_seed[1];
    // per insertion: (1) conflict scan, compacted with ballots; (2) directed edge list of the cavity; (3) boundary edges
    // (those whose reverse is not in the list) ranked with ballots, each writes its new triangle -- cavity slots first,
    // then the pool tail.  Three warp barriers, no atomics.
    int* s_ea = s_edges;            // [192] directed cavity edges: tails
    int* s_eb = s_edges + 192;      // [192] heads
    (void)s_cav_n; (void)s_edge_n;
    const unsigned lt = im_lanemask_lt();
    bool ovf = false;
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
    long long ph_a = 0, ph_b = 0, ph_c = 0, ph_d = 0, ph_t = 0, ph_nm = 0, ph_nc = 0, ph_nt = 0;
#define IM_PH(acc) do { const long long now_ = clock64(); acc += now_ - ph_t; ph_t = now_; } while (0)
#else
#define IM_PH(acc) do { } while (0)
#endif
    for (int p = 1; p < n && !ovf; ++p) {
        if (p == i1 || p == i2) continue;
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
        ph_t = clock64();
#endif
        const int nt = S->ntri;
        const float pxf = (float)Pt[p].x, pyf = (float)Pt[p].y;
        // (1a) cheap pass over the whole pool: live triangles whose cached circumcircle does not exclude p (ghosts always
        // qualify) are compacted into a short list; (1b) the exact predicates then run on that list only, all lanes busy
        int nm = 0;
        int* s_may = s_ea;   // [<= 192] reused: the edge arrays are filled after the scan
        for (int t0 = 0; t0 < nt; t0 += nlanes) {
            const int t = t0 + lane;
            bool maybe = false;
            if (t < nt) {
                const DTri tr = tris[t];
                if (tr.alive) {
                    maybe = true;
                    if (tr.v[0] != IM_GHOST && tr.v[1] != IM_GHOST && tr.v[2] != IM_GHOST) {
                        const float dx = pxf - S->circ[t][0], dy = pyf - S->circ[t][1];
                        if (dx * dx + dy * dy > S->circ[t][2]) maybe = false;   // certainly outside the circumcircle
                    }
                }
            }
            const unsigned m = im_ballot(maybe);
            if (maybe) {
                const int k = nm + im_popc(m & lt);
                if (k < 192) s_may[k] = t;
            }
            nm += im_popc(m);
        }
        if (nm > 192) { ovf = true; break; }   // warp-uniform
        IM_SYNCWARP();
        IM_PH(ph_a);
        int nc = 0;
        for (int j0 = 0; j0 < nm; j0 += nlanes) {
            const int j = j0 + lane;
            bool c = false;
            int t = 0;
            if (j < nm) {
                t = s_may[j];
                c = dt_conflict(tris[t], Pt, p);
            }
            const unsigned m = im_ballot(c);
            if (c) {
                const int k = nc + im_popc(m & lt);
                if (k < 64) s_cav[k] = t;
            }
            nc += im_popc(m);
        }
        if (nc > 64) { ovf = true; break; }   // warp-uniform
        IM_SYNCWARP();
        IM_PH(ph_b);
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
        ph_nm += nm; ph_nc += nc; ph_nt += nt;
#endif
        if (nc == 0) continue;                // duplicate point: skipped (CGAL does the same)
        const int ne3 = nc * 3;
#if defined(__CUDA_ARCH__)
        const bool one_pass = ne3 <= 32;   // every cavity edge in one lane: interior edges pair up through match.any
#else
        const bool one_pass = false;
#endif
        if (!one_pass) {
            for (int e = lane; e < ne3; e += nlanes) {
                const DTri& t = tris[s_cav[e / 3]];
                s_ea[e] = t.v[(e % 3 + 1) % 3];
                s_eb[e] = t.v[(e % 3 + 2) % 3];
            }
            IM_SYNCWARP();
        }
        int nb = 0;
        for (int e0 = 0; e0 < ne3; e0 += nlanes) {
            const int e = e0 + lane;
            bool isb = false;
            int a = 0, b = 0;
#if defined(__CUDA_ARCH__)
            if (one_pass) {
                unsigned key = 0xfffe0000u | (unsigned)lane;
                if (e < ne3) {
                    const DTri t = tris[s_cav[e / 3]];
                    const int k3 = e % 3;
                    a = (k3 == 0) ? t.v[1] : (k3 == 1) ? t.v[2] : t.v[0];
                    b = (k3 == 0) ? t.v[2] : (k3 == 1) ? t.v[0] : t.v[1];
                    const unsigned ua = (unsigned)a & 0xffffu, ub = (unsigned)b & 0xffffu;
                    key = ua < ub ? (ua << 16 | ub) : (ub << 16 | ua);
                }
                const unsigned peers = __match_any_sync(0xffffffffu, key);
                isb = (e < ne3) && __popc(peers) == 1;
                __syncwarp();   // all edge reads done before any cavity slot is overwritten
            } else
#endif
            if (e < ne3) {
                a = s_ea[e]; b = s_eb[e];
                isb = true;
                for (int f = 0; f < ne3; ++f)
                    if (s_ea[f] == b && s_eb[f] == a) { isb = false; break; }
            }
            const unsigned m = im_ballot(isb);
            if (isb) {
                const int k = nb + im_popc(m & lt);
                const int slot = (k < nc) ? s_cav[k] : (nt + (k - nc));
                if (slot < max_tris) {
                    tris[slot].v[0] = (short)a; tris[slot].v[1] = (short)b; tris[slot].v[2] = (short)p; tris[slot].alive = 1;
                    if (a != IM_GHOST && b != IM_GHOST) circumcircle_f(Pt, a, b, p, S->circ[slot]);
                }
            }
            nb += im_popc(m);
        }
        IM_PH(ph_c);
        // every cavity slot is reused (a valid cavity has nc + 2 boundary edges); kill leftovers defensively
        for (int k = nb + lane; k < nc; k += nlanes) tris[s_cav[k]].alive = 0;
        if (nb > nc) {
            if (nt + (nb - nc) <= max_tris) { if (lane == 0) S->ntri = nt + (nb - nc); }
            else ovf = true;
        }
        IM_SYNCWARP();
        IM_PH(ph_d);
    }
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        immesh::g_stamps[44] = ph_a; immesh::g_stamps[45] = ph_b; immesh::g_stamps[46] = ph_c; immesh::g_stamps[47] = ph_d;
        immesh::g_stamps[48] = ph_nm; immesh::g_stamps[49] = ph_nc; immesh::g_stamps[50] = ph_nt;
    }
#endif
    if (lane == 0) *s_ovf = ovf ? 1 : 0;
    IM_SYNCWARP();
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 36, 0);
    if (*s_ovf) {  // hand this voxel to the block-level stage
        if (lane == 0) F.work_n_ids[w] = -n;
        return;
    }
    // ---- faces passing the 150-degree filter, as sorted global id triples (stored over the dead circumcircle cache)
    int (*faces)[3] = reinterpret_cast<int (*)[3]>(&S->circ[0][0]);
    const int nt = S->ntri;
    for (int t = lane; t < nt; t += nlanes) {
        const DTri& tr = tris[t];
        if (!tr.alive || tr.v[0] < 0 || tr.v[1] < 0 || tr.v[2] < 0) continue;
        const int j0 = tr.v[0], j1 = tr.v[1], j2 = tr.v[2];
        if (angle_bad(S->uv[j0][0], S->uv[j0][1], S->uv[j1][0], S->uv[j1][1], S->uv[j2][0], S->uv[j2][1])) continue;
        if (angle_bad(S->uv[j1][0], S->uv[j1][1], S->uv[j2][0], S->uv[j2][1], S->uv[j0][0], S->uv[j0][1])) continue;
        if (angle_bad(S->uv[j2][0], S->uv[j2][1], S->uv[j0][0], S->uv[j0][1], S->uv[j1][0], S->uv[j1][1])) continue;
        int a = S->ids[j0], b = S->ids[j1], c = S->ids[j2];
        if (a > b) { const int x = a; a = b; b = x; }
        if (b > c) { const int x = b; b = c; c = x; }
        if (a > b) { const int x = a; a = b; b = x; }
        const int k = im_atomic_add(&S->nface, 1);
        faces[k][0] = a; faces[k][1] = b; faces[k][2] = c;
    }
    IM_SYNCWARP();
    const int nf = S->nface;
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, 37, nf);
    // facets + principal axes to the frame-wide lists; commit / orientation / pull run in the flat stage-C kernels
    if (lane == 0) {
        im_atomic_add(&M.cnt[IM_MC_STAT_FACETS], nf);
        S->scratch[0] = im_atomic_add(&M.cnt[IM_MC_FACES], nf);
    }
    IM_SYNCWARP();
    const int foff = S->scratch[0];
    if (foff + nf > F.max_list) {
        if (lane == 0) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
    } else {
        for (int k = lane; k < nf; k += nlanes) F.all_faces[foff + k] = make_int4(faces[k][0], faces[k][1], faces[k][2], w);
    }
    for (int k = lane; k < 9; k += nlanes) F.work_axes[(size_t)w * 9 + k] = S->axes[k];
    if (lane == 0) F.work_nfaces[w] = nf;
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
    if (blockIdx.x == 0 && threadIdx.x == 0) { immesh::g_stamps[38] = clock64(); immesh::g_stamps[39] = n; immesh::g_stamps[40] = nf; }
#endif
}

// ------------------------------------------------------------------ stage C, flat: one thread per new facet / per dilated vertex
// The per-voxel commit is a chain of dependent, DRAM-latency-bound accesses (triple-hash probes, smoothed positions,
// incidence lists); spreading it over one thread per facet and one thread per (voxel, vertex) pair exposes the
// memory-level parallelism instead.
IM_HD bool face_is(const int4& f, int a, int b, int c, int w) { return f.x == a && f.y == b && f.z == c && f.w == w; }
// C1: orientation + "existing / to add" decision of facet f, and registration in the frame's facet set
IM_HDN inline void commit_face(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int f) {
    const int4 fc = F.all_faces[f];
    const int w = fc.w;
    const unsigned long long word = ((unsigned long long)F.frame << 34) | (voxel_prio(M, F, w, true) << 1) |
                                    (unsigned long long)compute_flip(M, fc.x, fc.y, fc.z, F.fp->pose_t, F.work_axes + (size_t)w * 9);
    emit_face(M, F, fc.x, fc.y, fc.z, word);
    // bounded probe: a full set is a capacity error, never a spin
    unsigned int hs = (tri_hash(fc.x, fc.y, fc.z) + (unsigned int)w * 0x9E3779B1u) & F.fset_mask;
    for (unsigned int probe = 0;; ++probe) {
        if (probe > F.fset_mask) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); break; }
        if (im_atomic_cas32(&F.fset[hs], -1, f) == -1) break;
        hs = (hs + 1) & F.fset_mask;
    }
}
// C2a: pull (find_relative_triangulation_combination) for vertex reference r = (w, i): every live triangle whose smallest
// vertex is this one and whose other two vertices are in the voxel's dilated set.  Needs only the dilation result, so it
// runs concurrently with the triangulation kernels.
IM_HDN inline void pull_vertex(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int r) {
    const int ref = F.all_vref[r];
    const int w = ref >> 10, i = ref & 1023;
    const int n = F.work_n_ids[w];
    if (n > 256) return;   // large voxels pull inside the monolithic variant
    const int* ids = F.work_ids + (size_t)w * IM_MAXD;
    const int v = ids[i];
    for (int t = M.v_tri_head[v]; t >= 0;) {
        const int4 tr = M.tri[t];
        const int slot = (tr.x == v) ? 0 : ((tr.y == v) ? 1 : 2);
        const int nx = M.tri_next[(size_t)t * 3 + slot];
        if (tr.w && tr.x == v && tri_pre_frame(F, t)) {
            bool in_set = true;
            for (int pass = 0; pass < 2 && in_set; ++pass) {
                const int key = pass == 0 ? tr.y : tr.z;
                int lo = 0, hi = n - 1;
                bool hit = false;
                while (lo <= hi) {
                    const int mid = (lo + hi) >> 1;
                    const int val = ids[mid];
                    if (val == key) { hit = true; break; }
                    if (val < key) lo = mid + 1; else hi = mid - 1;
                }
                in_set = hit;
            }
            if (in_set) {
                const int e = im_atomic_add(&M.cnt[IM_MC_PULLED], 1);
                if (e < F.max_list) { F.pulled[2 * (size_t)e] = w; F.pulled[2 * (size_t)e + 1] = t; }
                else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
            }
        }
        t = nx;
    }
}
// C2b: commit, store side (triangle_compare): a pulled triangle that the voxel's new triangulation does not contain is removed
IM_HDN inline void pull_check(const MeshDev& M, const FrameBuf& F, int e) {
    const int w = F.pulled[2 * (size_t)e], t = F.pulled[2 * (size_t)e + 1];
    if (F.work_n_ids[w] < 0) return;   // handed over to the monolithic variant after a capacity overflow
    const int4 tr = M.tri[t];
    unsigned int hs = (tri_hash(tr.x, tr.y, tr.z) + (unsigned int)w * 0x9E3779B1u) & F.fset_mask;
    for (unsigned int probe = 0; probe <= F.fset_mask; ++probe) {
        const int k = F.fset[hs];
        if (k < 0) break;
        if (face_is(F.all_faces[k], tr.x, tr.y, tr.z, w)) return;
        hs = (hs + 1) & F.fset_mask;
    }
    emit_remove(M, F, t);
}

}  // namespace immesh
