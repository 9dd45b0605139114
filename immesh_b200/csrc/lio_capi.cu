// immesh_b200 -- CUDA kernels (sm_90a) and C-ABI host orchestration of the localization path.
// Kernel bodies live in lio_core.cuh / voxelmap.cuh; this file adds the launch geometry, the
// block-level integer reduction of the normal equations, stream/event plumbing and the C ABI.
// There is no CPU path: every entry point needs a CUDA device and fails loudly without one.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "peer_win.cuh"
#include "handles.hpp"
#include "map_dump.hpp"
#include "pool_growth.cuh"
#include "pdl.cuh"

using namespace immesh;

// ------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(128) k_prepare(LioParams P, ScanBuf sb_) {
    pdl_wait();
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) prepare_point(P, sb, i);
    pdl_trigger();
}

__global__ void k_reset_scan(ScanBuf sb, LioCtrl* ctrl, int copy_prop) {
    pdl_wait();
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int nt = gridDim.x * blockDim.x;
    unsigned long long* acc = &ctrl->acc[0][0];
    for (int i = tid; i < IM_MAX_ITER * IM_NTERMS * 2; i += nt) acc[i] = 0ull;
    if (copy_prop)
        for (int i = tid; i < IM_STATE_DOUBLES; i += nt) ctrl->state_prop[i] = ctrl->state[i];
    if (tid == 0) {
        ctrl->stop = 0;
        ctrl->iters_run = 0;
        ctrl->rematch_num = 0;
        for (int i = 0; i < IM_MAX_ITER; ++i) ctrl->blocks_done[i] = 0;
    }
    pdl_trigger();
}

// K2+K3.  Default (one GPU): two kernels per IESKF iteration.
//   k_match : 8 lanes per scan point.  The walk over a root voxel's octree (build_single_residual visits EVERY plane below the root,
//             up to 1 + 8 + 64 for max_layer 2, each a dependent chain of ~150 double operations behind a record load) is split by
//             first-level child over the 8 lanes and merged with three shuffles, in the serial walk's order (match_in_voxel_lane).
//   k_terms : one thread per scan point: the 29 fixed-point normal-equation terms of the matched points; the block's sums are reduced
//             with warp shuffles (integer adds: exact, order-free) and folded into the iteration's global accumulators with 60
//             atomics; the last block to finish runs the 6x6 IESKF update (ieskf_solve).
// k_residual is the two steps in one thread per point (used by immesh_residual_build).
#define RES_THREADS 128
#define MATCH_THREADS 128
#define MATCH_LANES 8
struct MatchCombine8 {
    unsigned int mask;   // the 8 lanes of this point inside the warp; 0: one lane per point
    __device__ void operator()(bool* ok, MatchResult* best) const {
        if (mask == 0u) return;   // one lane per point: nothing to merge
        const int lane = threadIdx.x & 31;
        *ok = (__ballot_sync(mask, *ok) & mask) != 0u;
        double prob = best->prob;
        int src = lane;
#pragma unroll
        for (int o = MATCH_LANES / 2; o > 0; o >>= 1) {
            const double op = __shfl_xor_sync(mask, prob, o);
            const int os = __shfl_xor_sync(mask, src, o);
            if (op > prob || (op == prob && os < src)) { prob = op; src = os; }   // first lane, in lane order, holding the largest probability
        }
        best->node = __shfl_sync(mask, best->node, src);
        best->layer = __shfl_sync(mask, best->layer, src);
        best->prob = prob;
    }
};
__global__ void __launch_bounds__(MATCH_THREADS, 8) k_match(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl) {
    __shared__ double s_state[24 + 6 * 18];
    pdl_wait();
    IM_STAMP(0, 0);
    // the stop flag, the scan's device-resident description and the state are loaded together (one trip to L2 instead of three)
    const int stop = ctrl->stop;
    const ScanBuf sb = scan_load_dyn(sb_);
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    const int n = sb.n;
    if (stop || n <= 0) return;
    IM_STAMP(1, n);
    // 8 lanes per point while the scan fits the machine about twice over (the grid is one resident wave); beyond that every SM has
    // more than enough points to hide the walk's latency and the lanes would only multiply the instruction count: one thread per point
    const long long threads = (long long)gridDim.x * blockDim.x;
    const int lanes = ((long long)n * MATCH_LANES <= 2 * threads) ? MATCH_LANES : 1;
    const int per_block = MATCH_THREADS / lanes;
    if ((long long)blockIdx.x * per_block >= n) return;   // block-uniform; the grid is sized for the machine, not for the scan
    __syncthreads();
    IM_STAMP(2, 0);
    const int sub = threadIdx.x & (lanes - 1);
    MatchCombine8 comb;
    comb.mask = (lanes == 1) ? 0u : 0xFFu << ((threadIdx.x & 31) & ~(MATCH_LANES - 1));
    for (int i = blockIdx.x * per_block + (threadIdx.x / lanes); i < n; i += gridDim.x * per_block)
        residual_match_lanes(map, P, sb, s_state, i, sub, lanes, comb);
    pdl_trigger();
    IM_STAMP(7, 0);
}

// Publish a block's normal-equation sums (2^-20 fixed point, DESIGN.md 3) into the (hi, lo) accumulator pairs `dst`: thread, warp and
// block sums in int64, the block's sum split into its 32-bit halves for the atomics.  The block sum of 128 thread sums cannot leave
// int64 while every thread sum is below 2^56 in magnitude, and a thread sum stays exact while it holds at most IM_FX_THREAD_TERMS
// terms (each below 1e10 * 2^20, residual_terms refuses larger ones).  Beyond either bound -- a dense scan with very large weights,
// where a block's int64 sum used to wrap silently -- the call fails with IMMESH_E_RANGE.  The flag is raised once per block after the
// warp sums (a global atomic in every thread ahead of the shuffles made k_terms 60 % slower).
#define IM_FX_THREAD_TERMS 879   // floor(2^63 / (1e10 * 2^20))
__device__ __forceinline__ void publish_terms(const long long (&acc)[IM_NTERMS], unsigned long long* dst, int* err) {
    __shared__ long long s_part[RES_THREADS / 32][IM_NTERMS];
    long long mag = 0;   // bit 56 or above set iff some acc[k] lies outside [-2^56, 2^56) (x ^ (x >> 63) is x, or -x - 1 for negative x)
#pragma unroll
    for (int k = 0; k < IM_NTERMS - 1; ++k) mag |= acc[k] ^ (acc[k] >> 63);
    const int out_of_range = (acc[28] > IM_FX_THREAD_TERMS || mag >= (1LL << 56)) ? 1 : 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < IM_NTERMS - 1; ++k) {
        long long v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_part[warp][k] = v;
    }
    if (__syncthreads_or(out_of_range) && threadIdx.x == 0) atomicOr(err, IM_ERR_FX_RANGE);
    if (threadIdx.x < IM_NTERMS - 1) {
        long long v = 0;
        for (int w = 0; w < RES_THREADS / 32; ++w) v += s_part[w][threadIdx.x];
        if (v != 0) {
            atomicAdd(&dst[2 * threadIdx.x], (unsigned long long)(v >> 32));
            atomicAdd(&dst[2 * threadIdx.x + 1], (unsigned long long)(v & 0xffffffffLL));
        }
    }
}

template <bool MATCHED>
__device__ __forceinline__ void residual_block(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb_, LioCtrl* ctrl, int iter, int fused_solve) {
    __shared__ double s_state[24 + 6 * 18];
    pdl_wait();
    IM_STAMP(10, 0);
    // the stop flag, the scan's device-resident description and the state -- rot/pos and the 6x6 pose block of the covariance, the only
    // parts this pass reads -- are loaded together (one trip to L2 instead of three)
    const int stop = ctrl->stop;
    const ScanBuf sb = scan_load_dyn(sb_);
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    const int n = sb.n;
    if (stop || n <= 0) return;   // empty scan: no iteration runs (iters_run stays 0), as with an empty map
    // the grid is sized for the largest scan (constant launch sequence); blocks without points leave at once and are not counted
    const int nb_active = min((int)gridDim.x, (n + RES_THREADS - 1) / RES_THREADS);
    if ((int)blockIdx.x >= nb_active) return;
    __syncthreads();
    IM_STAMP(11, 0);
    long long acc[IM_NTERMS];
#pragma unroll
    for (int k = 0; k < IM_NTERMS; ++k) acc[k] = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        long long t[IM_NTERMS];
        const bool hit = MATCHED ? residual_point_matched(map, P, sb, s_state, i, t, map.err) : residual_point(map, P, sb, s_state, i, t, map.err);
        if (hit) {
#pragma unroll
            for (int k = 0; k < IM_NTERMS; ++k) acc[k] += t[k];
        }
    }
    IM_STAMP(12, acc[0] + acc[27]);
    publish_terms(acc, ctrl->acc[iter], map.err);
    IM_STAMP(13, 0);
    if (!fused_solve) return;
    // the last block to publish its sums runs the IESKF update of this iteration (6x6 form, lio_core.cuh: ieskf_solve)
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&ctrl->blocks_done[iter], 1) == nb_active - 1) ? 1 : 0;
    __syncthreads();
    IM_STAMP(14, s_last);
    if (s_last) {
        __shared__ SolveScratch S;
        __threadfence();
        ieskf_solve(P, ctrl, iter, &S, threadIdx.x, blockDim.x);
    }
    pdl_trigger();
}
__global__ void __launch_bounds__(RES_THREADS) k_residual(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, int iter, int fused_solve) {
    residual_block<false>(map, P, sb_, ctrl, iter, fused_solve);
}
__global__ void __launch_bounds__(RES_THREADS) k_terms(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, int iter, int fused_solve) {
    residual_block<true>(map, P, sb_, ctrl, iter, fused_solve);
}

// sharded VoxelMap: pass 1 (match where this rank owns the voxel, publish bits) and pass 2 (terms + integer reduction)
__global__ void __launch_bounds__(RES_THREADS) k_shard_pass1(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, unsigned int* bits, int words_cap) {
    __shared__ double s_state[24 + 6 * 18];
    if (ctrl->stop) return;
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    if (n <= 0) return;
    const int words = words_cap;
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) shard_pass1_point(map, P, sb, s_state, i, bits, bits + words);
}
__global__ void __launch_bounds__(RES_THREADS) k_shard_pass2(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, int iter, const unsigned int* bits, int words_cap) {
    __shared__ double s_state[24 + 6 * 18];
    if (ctrl->stop) return;
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    if (n <= 0) return;
    const int words = words_cap;
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    __syncthreads();
    long long acc[IM_NTERMS];
#pragma unroll
    for (int k = 0; k < IM_NTERMS; ++k) acc[k] = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        long long t[IM_NTERMS];
        if (shard_pass2_point(map, P, sb, s_state, i, bits, bits + words, t, map.err)) {
#pragma unroll
            for (int k = 0; k < IM_NTERMS; ++k) acc[k] += t[k];
        }
    }
    publish_terms(acc, ctrl->acc[iter], map.err);
}

// ---- sharded VoxelMap over peer windows (peer_win.cuh): the two exchanges of an iteration are fused into the kernels.
// Window of one rank:  flag[2][8] u64 | acc[8][IM_NTERMS*2] u64 (one row per source rank) | bits[8][2][words_cap] u32
struct LioPeers {
    unsigned char* w[IM_MAX_RANKS];
    int rank, n, words_cap, pad;
};
#define IM_LIOWIN_ACC_OFF 128
#define IM_LIOWIN_BITS_OFF 4096
__device__ __forceinline__ unsigned long long* liowin_flag(unsigned char* w, int phase, int src) { return (unsigned long long*)w + phase * IM_MAX_RANKS + src; }
__device__ __forceinline__ unsigned long long* liowin_acc(unsigned char* w, int src) { return (unsigned long long*)(w + IM_LIOWIN_ACC_OFF) + src * (IM_NTERMS * 2); }
__device__ __forceinline__ unsigned int* liowin_bits(unsigned char* w, int src, int which, int words_cap) { return (unsigned int*)(w + IM_LIOWIN_BITS_OFF) + (size_t)(src * 2 + which) * words_cap; }

// pass 1 + publish: every warp ballots the two bits of its 32 consecutive points and lane r stores the two words into rank
// r's window (row = this rank); the last block raises this rank's pass-1 flag in every peer window.
__global__ void __launch_bounds__(RES_THREADS) k_shard_pass1_p2p(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, LioPeers pe, int epoch_off) {
    __shared__ double s_state[24 + 6 * 18];
    __shared__ int s_last;
    if (ctrl->stop) return;
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    if (n <= 0) return;
    const unsigned long long epoch = ctrl->dyn.epoch + (unsigned long long)epoch_off;
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int n32 = (n + 31) & ~31;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n32; i += gridDim.x * blockDim.x) {
        bool ex = false, ok1 = false;
        if (i < n) shard_pass1_flags(map, P, sb, s_state, i, &ex, &ok1);
        const unsigned int we = __ballot_sync(0xffffffffu, ex), wo = __ballot_sync(0xffffffffu, ok1);
        if (lane < pe.n) {
            liowin_bits(pe.w[lane], pe.rank, 0, pe.words_cap)[i >> 5] = we;
            liowin_bits(pe.w[lane], pe.rank, 1, pe.words_cap)[i >> 5] = wo;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&ctrl->shard_cnt[0], 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (s_last) {
        if (threadIdx.x == 0) ctrl->shard_cnt[0] = 0;
        __threadfence_system();
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) immesh::st_release_sys(liowin_flag(pe.w[threadIdx.x], 0, pe.rank), epoch);
    }
}
// wait for the peers' bits + pass 2 + integer block reduction + publish: the last block copies this rank's 60 partial sums
// into row `rank` of every window and raises the pass-2 flag.
__global__ void __launch_bounds__(RES_THREADS) k_shard_pass2_p2p(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, int iter, LioPeers pe, int epoch_off) {
    __shared__ double s_state[24 + 6 * 18];
    __shared__ int s_last;
    if (ctrl->stop) return;
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    if (n <= 0) return;
    const unsigned long long epoch = ctrl->dyn.epoch + (unsigned long long)epoch_off;
    if (threadIdx.x < pe.n && threadIdx.x != pe.rank) {
        immesh::wait_epoch(liowin_flag(pe.w[pe.rank], 0, threadIdx.x), epoch, map.err, IM_ERR_PEER_TIMEOUT);
    }
    for (int i = threadIdx.x; i < 24 + 6 * 18; i += blockDim.x) s_state[i] = ctrl->state[i];
    __syncthreads();
    long long acc[IM_NTERMS];
#pragma unroll
    for (int k = 0; k < IM_NTERMS; ++k) acc[k] = 0;
    unsigned char* mine = pe.w[pe.rank];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        unsigned int we = 0, wo = 0;
        for (int r = 0; r < pe.n; ++r) {
            we |= __ldcg(liowin_bits(mine, r, 0, pe.words_cap) + (i >> 5));
            wo |= __ldcg(liowin_bits(mine, r, 1, pe.words_cap) + (i >> 5));
        }
        long long t[IM_NTERMS];
        if (shard_pass2_flags(map, P, sb, s_state, i, (we >> (i & 31)) & 1u, (wo >> (i & 31)) & 1u, t, map.err)) {
#pragma unroll
            for (int k = 0; k < IM_NTERMS; ++k) acc[k] += t[k];
        }
    }
    publish_terms(acc, ctrl->acc[iter], map.err);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&ctrl->shard_cnt[1], 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (s_last) {
        __threadfence();
        if (threadIdx.x == 0) ctrl->shard_cnt[1] = 0;
        if (threadIdx.x < IM_NTERMS * 2) {
            const unsigned long long v = *(volatile unsigned long long*)&ctrl->acc[iter][threadIdx.x];
            for (int r = 0; r < pe.n; ++r) liowin_acc(pe.w[r], pe.rank)[threadIdx.x] = v;
        }
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) immesh::st_release_sys(liowin_flag(pe.w[threadIdx.x], 1, pe.rank), epoch);
    }
}
// wait for the peers' sums, add the rows (integers: order-free, identical on every rank), then the usual solve
#define SOLVE_THREADS 128
__global__ void __launch_bounds__(SOLVE_THREADS) k_solve_p2p(LioParams P, LioCtrl* ctrl, int iter, LioPeers pe, int epoch_off, int* err) {
    __shared__ SolveScratch S;
    if (ctrl->stop || (ctrl->dyn.n_dev ? *ctrl->dyn.n_dev : ctrl->dyn.n) <= 0) return;
    const unsigned long long epoch = ctrl->dyn.epoch + (unsigned long long)epoch_off;
    if (threadIdx.x < pe.n && threadIdx.x != pe.rank) {
        immesh::wait_epoch(liowin_flag(pe.w[pe.rank], 1, threadIdx.x), epoch, err, IM_ERR_PEER_TIMEOUT);
    }
    __syncthreads();
    if (threadIdx.x < IM_NTERMS * 2) {
        unsigned long long v = 0;
        for (int r = 0; r < pe.n; ++r) v += __ldcg(liowin_acc(pe.w[pe.rank], r) + threadIdx.x);
        ctrl->acc[iter][threadIdx.x] = v;
    }
    __threadfence_block();
    __syncthreads();
    ieskf_solve(P, ctrl, iter, &S, threadIdx.x, blockDim.x);
}
// stand-alone solve (NCCL-sharded path: the sums are complete only after the all-reduce)
__global__ void __launch_bounds__(SOLVE_THREADS) k_solve(LioParams P, LioCtrl* ctrl, int iter) {
    __shared__ SolveScratch S;
    if (ctrl->stop || (ctrl->dyn.n_dev ? *ctrl->dyn.n_dev : ctrl->dyn.n) <= 0) return;
    ieskf_solve(P, ctrl, iter, &S, threadIdx.x, blockDim.x);
}

#define PREDICT_THREADS 352
__global__ void __launch_bounds__(PREDICT_THREADS) k_predict(LioCtrl* ctrl) {
    __shared__ double T[324], Fx[324];
    const double dt = ctrl->dyn.dt;
    if (!(dt > 0)) return;   // block-uniform
    predict_const_vel(ctrl->state, dt, ctrl->dyn.cov_gyr, ctrl->dyn.cov_acc, T, Fx, threadIdx.x, blockDim.x);
}

__global__ void __launch_bounds__(128) k_grow_point(VoxelMapDev map, LioParams P, ScanBuf sb_, LioCtrl* ctrl, int mode) {
    pdl_wait();
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) grow_point(map, P, sb, ctrl->state, i, mode);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_grow_segment(ScanBuf sb) {
    pdl_wait();
    const int nt = *sb.n_touched;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nt; t += gridDim.x * blockDim.x) grow_segment(sb, t);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_grow_scatter(ScanBuf sb_) {
    pdl_wait();
    const ScanBuf sb = scan_load_dyn(sb_);
    const int n = sb.n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) grow_scatter(sb, i);
    pdl_trigger();
}
// Most touched root voxels receive one or two points of a scan and stay in an append-only regime (a node still collecting its
// first points, or a planar node between two refits): no plane fit, no split, no descent.  k_grow_simple finishes those -- same
// appends, same order (ascending (var_contrast, index)), same arithmetic as update_octo_tree -- with a warp per voxel in a lean
// kernel (few registers: many more warps in flight than the general kernel below, which carries the plane fit and the octree
// split); only the other voxels go on to k_grow_voxel through a compact list.  At the 1M-point / 0.2 m configuration 175 k voxels
// are touched per scan and nearly all are of the first kind.  (A THREAD per simple voxel was measured and rejected: one thread's
// 60 dependent moment read-modify-writes take longer than the warp's two per lane.)
#define GROW_SIMPLE_MAX 4
__global__ void __launch_bounds__(128) k_grow_simple(VoxelMapDev map, LioParams P, ScanBuf sb, int mode, int* complex_list, int* n_complex) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int nt = *sb.n_touched;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < nt; t += nwarps) {
        const int slot = sb.touched[t];
        const int cnt = sb.slot_count[slot], off = sb.slot_offset[slot];
        const int root = map.root_node[slot];
        int kind = 0;   // 0: general kernel, 1: append all, 2: drop all (frozen planar node)
        if (root >= 0 && (mode & 1) == 0 && cnt <= GROW_SIMPLE_MAX) {
            const NodeRec& n = map.nodes[root];
            if (!n.init_octo) kind = (n.n_pts + cnt <= P.layer_init[n.layer]) ? 1 : 0;
            else if (map.planes[root].is_plane) kind = !n.update_enable ? 2 : ((n.new_points + cnt <= 5 && n.n_pts + cnt < P.max_points) ? 1 : 0);
        }
        kind = __shfl_sync(0xffffffffu, kind, 0);
        if (kind == 0) {
            if (lane == 0) complex_list[atomicAdd(n_complex, 1)] = t;
            continue;
        }
        if (kind == 1) {
            int idx[GROW_SIMPLE_MAX];
            double key[GROW_SIMPLE_MAX];
#pragma unroll
            for (int a = 0; a < GROW_SIMPLE_MAX; ++a) {
                idx[a] = 0x7fffffff; key[a] = 0.0;
                if (a < cnt) { idx[a] = sb.seg[off + a]; key[a] = sb.sortkey[idx[a]]; }
            }
#pragma unroll
            for (int a = 1; a < GROW_SIMPLE_MAX; ++a)       // insertion sort on (key, index): the order std::sort(var_contrast) with ties by index gives
#pragma unroll
                for (int b = a; b > 0; --b) {
                    const bool lt = b < cnt && (key[b] < key[b - 1] || (key[b] == key[b - 1] && idx[b] < idx[b - 1]));
                    if (lt) { const int ti = idx[b]; idx[b] = idx[b - 1]; idx[b - 1] = ti; const double tk = key[b]; key[b] = key[b - 1]; key[b - 1] = tk; }
                }
#pragma unroll
            for (int a = 0; a < GROW_SIMPLE_MAX; ++a) {
                if (a >= cnt) break;
                const int i = idx[a];
                const float px = sb.pw[(size_t)i * 3 + 0], py = sb.pw[(size_t)i * 3 + 1], pz = sb.pw[(size_t)i * 3 + 2];
                if (lane == 0) {
                    map.nodes[root].new_points += 1;
                    node_append(map, root, px, py, pz, sb.var + (size_t)i * 6);
                }
                node_moments_add(map, root, px, py, pz, sb.var + (size_t)i * 6, lane, 32);
                __syncwarp();
            }
        }
        if (lane == 0) {
            sb.slot_count[slot] = 0;
            sb.slot_cursor[slot] = 0;
        }
    }
    pdl_trigger();
}
// one warp per remaining touched root voxel, voxels claimed dynamically (their cost varies by orders of magnitude)
__global__ void __launch_bounds__(128) k_grow_voxel(VoxelMapDev map, LioParams P, ScanBuf sb, int mode, int* sorted_scratch, int* work_counter, const int* complex_list, const int* n_complex) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int nt = *n_complex;
    while (true) {
        int t = 0;
        if (lane == 0) t = atomicAdd(work_counter, 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= nt) break;
        grow_voxel(map, P, sb, complex_list[t], mode, lane, 32, sorted_scratch);
    }
    pdl_trigger();
}
// last kernel of a scan: recycle chunks, reset the per-scan counters, publish the converged pose for the mesher's frame (which
// runs behind on another stream) and assemble the block the host reads back with one D2H copy
__global__ void k_grow_finish(VoxelMapDev map, ScanBuf sb, LioCtrl* ctrl, int* counters) {
    pdl_wait();
    recycle_chunks(map, threadIdx.x, blockDim.x);
    if (threadIdx.x == 0) {
        *sb.n_touched = 0;
        *sb.seg_top = 0;
        counters[IM_LC_WORK] = 0;
        counters[IM_LC_COMPLEX] = 0;
    }
    if (ctrl) {
        const int si = ctrl->dyn.scan_idx;
        for (int i = threadIdx.x; i < IM_STATE_DOUBLES; i += blockDim.x) ctrl->out.state[i] = ctrl->state[i];
        if (threadIdx.x < 12) ctrl->pose_ring[si & (IM_POSE_RING - 1)][threadIdx.x] = ctrl->state[threadIdx.x];
        if (threadIdx.x < IM_LC_SIZE) ctrl->out.counters[threadIdx.x] = counters[threadIdx.x];
        if (threadIdx.x == 0) { ctrl->out.iters_run = ctrl->iters_run; ctrl->out.scan_idx = si; }
    }
    __syncthreads();
    if (threadIdx.x == 0 && map.stat) { map.stat[0] = 0; map.stat[1] = 0; }   // per-scan work counters (IM_LC_REFITS, IM_LC_REFIT_POINTS)
}
// BuildResidualListOMP on caller-supplied Point_with_var data (world point + covariance per point)
__global__ void __launch_bounds__(128) k_match_pv(VoxelMapDev map, LioParams P, ScanBuf sb, const double* pw, int n) {   // API call: explicit n
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const MatchResult mr = match_point(map, P, pw + (size_t)i * 3, sb.var + (size_t)i * 6);
        sb.match_node[i] = mr.node;
        sb.match_layer[i] = mr.layer;
    }
}
// ptpl payload of every matched point (diagnostic / drop-in immesh_residual_build)
__global__ void k_gather_ptpl(VoxelMapDev map, ScanBuf sb, int n, double* out /*[n][31]*/) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int nd = sb.match_node[i];
        if (nd < 0) continue;
        const PlaneRec& pl = map.planes[nd];
        double* o = out + (size_t)i * 31;
        for (int j = 0; j < 3; ++j) { o[j] = (double)sb.body[i * 3 + j]; o[3 + j] = pl.normal[j]; o[6 + j] = pl.center[j]; }
        o[9] = (double)pl.d;
        for (int j = 0; j < 21; ++j) o[10 + j] = pl.pv[j];
    }
}

// ---- plane-map publication (immesh_voxelmap_plane_markers): only the roots in the pending list are visited.
// The listed roots are ordered by their packed key with two stable radix sorts of the 32-bit halves (low half first), which is the
// signed (kx, ky, kz) order of the map dump; one thread per root then counts its rows (a walk that clears nothing), an exclusive
// scan places them, and -- once the host has checked the caller's room -- one thread per root writes its rows and settles its mark.
namespace {
#include "radix_sort.cuh"
}
#define PUB_THREADS 256
static_assert(IM_PUB_COLS == IMMESH_PLANE_MARKER_COLS, "plane-marker row width");
// n_dev (or null): the count is read on the device.  Every path waits for the predecessor first (launched with IM_LAUNCH_PDL in the
// scan feed's markers).
__global__ void __launch_bounds__(PUB_THREADS) k_pub_keys(VoxelMapDev map, int n, const int* n_dev, int hi, const unsigned int* order, unsigned int* kout,
                                                          unsigned int* vout) {
    pdl_wait();
    if (n_dev) n = *n_dev;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = order ? order[i] : (unsigned int)i;
        const unsigned long long key = map.keys[map.pub_list[v]];
        kout[i] = hi ? (unsigned int)(key >> 32) : (unsigned int)key;
        vout[i] = v;
    }
}
// per root (in key order): slot, row count; the four reference counters summed with integer atomics (order-free)
__global__ void __launch_bounds__(PUB_THREADS) k_pub_count(VoxelMapDev map, int n, const int* n_dev, const unsigned int* order, int* slots, int* cnt, int* counts) {
    pdl_wait();
    if (n_dev) n = *n_dev;
    int c[4] = {0, 0, 0, 0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int slot = map.pub_list[order[i]];
        const int root = map.root_node[slot];
        slots[i] = slot;
        cnt[i] = root >= 0 ? plane_pub_root(map, root, map.keys[slot], nullptr, c) : 0;
    }
    for (int k = 0; k < 4; ++k)
        if (c[k]) atomicAdd(counts + k, c[k]);
}
// per root: its rows at its offset, flags cleared; roots that stay pending go back on the (reset) list.  md (or null): the scan
// feed's markers -- nothing when the scan's rows were lost, else the rows at the ring cursor k_mark_head placed (row r in slot r % ring)
__global__ void __launch_bounds__(PUB_THREADS) k_pub_emit(VoxelMapDev map, int n, const int* slots, const int* off, double* rows, const LioMarkDev* md, long long ring) {
    pdl_wait();
    long long base = 0;
    if (md) {
        if (md->lost) return;
        n = md->n;
        base = md->base;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int slot = slots[i];
        if (plane_pub_commit(map, slot, rows, base + off[i], ring)) map.pub_list[atomicAdd(map.pub_n, 1)] = slot;
    }
}
// ---- the scan feed's plane-map markers (immesh_lio_feed_markers_enable): the publication above, queued in the scan's launch sequence
// with every count read on the device.  k_mark_begin takes the pending count; the key sort, k_pub_count and k_pub_scan run over it;
// k_mark_head places the rows at the ring cursor (or loses them all), writes the header and -- only when the rows fit -- resets the
// list (marker_header), so that k_pub_emit publishes and settles the marks; it returns at once for a lost scan (md->lost), the
// case where marker_header left the list as it was.  A lost scan consumes nothing.
__global__ void k_mark_begin(const int* pub_n, LioMarkDev* md) {
    pdl_wait();
    if (threadIdx.x == 0) md->n = *pub_n;
    if (threadIdx.x < 5) md->misc[threadIdx.x] = 0;
}
__global__ void __launch_bounds__(1024) k_pub_scan(int* cnt, const LioMarkDev* md, int* total) {
    pdl_wait();
    rs_scan_block(cnt, md->n, total);
}
// walk = 0: a record without a walk (the IMU chain's branch 1)
__global__ void k_mark_head(const LioFeedDev* fd, LioMarkDev* md, int* pub_n, long long* hdr, long long max_scans, long long max_rows, int walk) {
    pdl_wait();
    if (threadIdx.x != 0) return;
    const long long scan = fd->dyn.scan;
    md->started = scan;   // before any byte of the slot changes (a reader checks it after its copy)
    __threadfence();
    marker_header(*md, scan, walk, pub_n, max_rows, hdr + (scan - 1) % max_scans * IMMESH_LIO_FEED_MARKER_HDR);
    __threadfence();
    pdl_trigger();
}

// ---- scan publishers.  immesh_lio_effect_cloud: a scan-order compaction of match_node >= 0 -- per-tile counts, the one-block
// exclusive scan over the tiles (k_rs_scan), then each tile emits its rows in order.  immesh_lio_registered_cloud: a strided gather.
// Both transform with the state in LioCtrl when they run (the handle's current state) and read the scan through scan_load_dyn, so a
// scan whose count is device resident is published as it was localised.
// The scan feed (immesh_lio_feed_enable) runs the same three kernels and the gather inside the scan's launch sequence with `fd` set:
// the rows then go to the feed's row ring at the cursor k_feed_head placed (row r in slot r % ring), and nothing is written when the
// scan's rows were lost.  fd == null: the blocking publishers, rows from 0.
#define SPUB_THREADS 256   // one tile of the scan per block
static_assert(IMMESH_SCAN_PUB_COLS == 4, "scan publisher row width");
__global__ void __launch_bounds__(SPUB_THREADS) k_eff_count(ScanBuf sb_, int* tile_cnt) {
    pdl_wait();
    const ScanBuf sb = scan_load_dyn(sb_);
    const int i = blockIdx.x * SPUB_THREADS + threadIdx.x;
    const int c = __syncthreads_count(i < sb.n && sb.match_node[i] >= 0);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = c;
}
__global__ void __launch_bounds__(SPUB_THREADS) k_eff_emit(LioParams P, ScanBuf sb_, const LioCtrl* ctrl, const int* tile_off, float4* rows, int* scan_index,
                                                           const LioFeedDev* fd, long long ring) {
    __shared__ int s_warp[SPUB_THREADS / 32];
    __shared__ double s_state[12];
    pdl_wait();
    long long base = 0;
    if (fd) {
        if (fd->lost) return;   // block-uniform
        base = fd->eff_base;
    }
    const ScanBuf sb = scan_load_dyn(sb_);
    if (threadIdx.x < 12) s_state[threadIdx.x] = ctrl->state[threadIdx.x];
    const int i = blockIdx.x * SPUB_THREADS + threadIdx.x;
    const bool m = i < sb.n && sb.match_node[i] >= 0;
    const unsigned int b = __ballot_sync(0xffffffffu, m);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    if (!m) return;
    int off = tile_off[blockIdx.x] + __popc(b & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    float r[4];
    scan_pub_row(P, s_state, sb.body + (size_t)i * 3, sb.wsqrt[i], r);
    const long long pos = fd ? (base + off) % ring : off;
    rows[pos] = make_float4(r[0], r[1], r[2], r[3]);
    if (scan_index) scan_index[pos] = i;
}
// rows j = 0 .. ceil(n / skip) - 1 from point j * skip; pts == null: the localised scan.  inten != null: the intensity of point i is
// inten[i] (the front-end's clouds keep it beside the packed points) instead of column col.  fd != null: the source is the scan's
// FeedDyn (source 2: its full scan, stride 3, intensity inten or 0; source 1: the localised scan)
__global__ void __launch_bounds__(SPUB_THREADS) k_reg_gather(LioParams P, ScanBuf sb_, const LioCtrl* ctrl, const float* pts, int n, int stride, int col, int skip, float4* rows,
                                                             const float* __restrict__ inten, const LioFeedDev* fd, long long ring) {
    __shared__ double s_state[12];
    pdl_wait();
    long long base = 0;
    if (fd) {
        if (fd->lost || fd->dyn.src == 0) return;   // block-uniform
        base = fd->reg_base;
        pts = nullptr;
        if (fd->dyn.src == 2) { pts = fd->dyn.pts; n = feed_full_n(fd->dyn); inten = fd->dyn.inten; stride = 3; col = -1; }
    }
    if (threadIdx.x < 12) s_state[threadIdx.x] = ctrl->state[threadIdx.x];
    if (!pts) {
        const ScanBuf sb = scan_load_dyn(sb_);
        pts = sb.body; n = sb.n; stride = 3; col = -1;
    }
    __syncthreads();
    const int m = n > 0 ? (n - 1) / skip + 1 : 0;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const float* p = pts + (size_t)j * skip * stride;
        float r[4];
        scan_pub_row(P, s_state, p, inten ? inten[(size_t)j * skip] : col >= 0 ? p[col] : 0.0f, r);
        rows[fd ? (base + j) % ring : j] = make_float4(r[0], r[1], r[2], r[3]);
    }
}
__global__ void k_scan_n(ScanBuf sb_, int* out) { *out = scan_load_dyn(sb_).n; }

// ---- scan feed (immesh_lio_feed_enable): k_feed_head runs right behind the scan's last kernel (k_grow_finish, or the IMU chain's
// initialisation copies): the state, the header, and the row cursor (feed_append); k_feed_done, behind the row emitters, publishes the
// scan's number to the host word the reader polls.
#define FEED_THREADS 128
__global__ void __launch_bounds__(FEED_THREADS) k_feed_head(ScanBuf sb_, const LioCtrl* ctrl, const int* counters, LioFeedDev* fd, long long* hdr, double* states,
                                                            long long max_scans, long long max_rows, const int* eff_total, int skip) {
    pdl_wait();
    const FeedDyn d = fd->dyn;
    const long long slot = (d.scan - 1) % max_scans;
    if (threadIdx.x == 0) {
        fd->started = d.scan;   // before any byte of the slot changes (a reader checks it after its copy)
        __threadfence();
    }
    __syncthreads();
    for (int i = threadIdx.x; i < IM_STATE_DOUBLES; i += blockDim.x) states[slot * IM_STATE_DOUBLES + i] = ctrl->state[i];
    if (threadIdx.x == 0) {
        const int branch = d.branch_dev ? *d.branch_dev : d.branch;
        const bool lio = d.lio && (!d.branch_dev || branch == 3);
        const int iters = lio ? ctrl->iters_run : 0;
        long long ne = 0, nr = 0;
        if (lio) {
            if (eff_total) ne = *eff_total;
            const int n = d.src == 2 ? feed_full_n(d) : d.src == 1 ? scan_load_dyn(sb_).n : 0;
            nr = n > 0 ? (n - 1) / skip + 1 : 0;
        }
        long long* h = hdr + slot * IMMESH_LIO_FEED_HDR;
        feed_append(*fd, ne, nr, max_rows, h);
        h[IMMESH_FEED_KIND] = d.kind;
        h[IMMESH_FEED_BRANCH] = branch;
        h[IMMESH_FEED_ITERS] = iters;
        h[IMMESH_FEED_MATCHES] = iters > 0 ? (long long)ctrl->stats[iters - 1].n_match : 0;
        h[IMMESH_FEED_CONVERGED] = iters > 0 ? (long long)ctrl->stats[iters - 1].converged : 0;
        h[IMMESH_FEED_ERR] = counters[IM_LC_ERR];
        h[IMMESH_FEED_SOURCE] = lio ? d.src : 0;
        h[IMMESH_FEED_SCAN] = d.scan;
    }
    __syncthreads();
    pdl_trigger();
}
__global__ void k_feed_done(const LioFeedDev* fd, long long* done) {
    pdl_wait();
    if (threadIdx.x == 0) {
        __threadfence_system();
        *(volatile long long*)done = fd->dyn.scan;
    }
}

// ---- growth of the map pools (immesh_lio_reserve): rebuild of the root hash into a larger table, then the back-pointers to slots
#define GROW_THREADS 256
__global__ void __launch_bounds__(GROW_THREADS) k_rehash_roots(VoxelMapDev from, VoxelMapDev to, int* slot_map) {
    const unsigned int cap = from.cap_mask + 1u;   // at most 2^30 slots (IM_POOL_LIMIT)
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += gridDim.x * blockDim.x) rehash_root_slot(from, to, s, slot_map);
}
__global__ void __launch_bounds__(GROW_THREADS) k_remap_roots(VoxelMapDev to, int n_nodes, const int* from_pub_list, int n_pub, const int* slot_map) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_nodes; i += gridDim.x * blockDim.x) remap_node_root_slot(to, i, slot_map);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pub; i += gridDim.x * blockDim.x) remap_pub_entry(from_pub_list, to, i, slot_map);
}

// ---- local map (local_map.cuh).  k_local_map_box: one thread evaluates laser_map_fov_segment at the state the scan's IESKF starts
// from (automatic = 1, gated by LocalMapCtrl::on), after clamping the node free stack's top that the previous scan's pops may have
// left negative (before any push).  k_evict_roots: a grid-stride sweep over the hash slots against this scan's removal boxes (or
// the caller's, immesh_voxelmap_evict_boxes); it leaves at once when there are none.
__global__ void k_local_map_box(LioCtrl* ctrl, int* node_free_top, int automatic) {
    pdl_wait();
    if (threadIdx.x == 0) {
        if (*node_free_top < 0) *node_free_top = 0;
        LocalMapCtrl& L = ctrl->lm;
        L.n_rm = 0;
        if (automatic && L.on) local_map_rule(L, ctrl->state + 9);   // pos_end
    }
    pdl_trigger();
}
#define EVICT_THREADS 256
__global__ void __launch_bounds__(EVICT_THREADS) k_evict_roots(VoxelMapDev map, LioCtrl* ctrl, const float* boxes, int n_boxes) {
    pdl_wait();
    if (!boxes) { boxes = &ctrl->lm.rm[0][0]; n_boxes = ctrl->lm.n_rm; }
    if (n_boxes <= 0) return;
    const unsigned int cap = map.cap_mask + 1u;
    unsigned long long roots = 0, nodes = 0, chunks = 0;
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += gridDim.x * blockDim.x) {
        int nn, nc;
        roots += evict_root_slot(map, s, boxes, n_boxes, &nn, &nc);
        nodes += nn;
        chunks += nc;
    }
    if (roots) {
        atomicAdd(&ctrl->lm.roots, roots);
        atomicAdd(&ctrl->lm.nodes, nodes);
        atomicAdd(&ctrl->lm.chunks, chunks);
    }
    pdl_trigger();
}

// ------------------------------------------------------------------ host side

#include "nccl_api.hpp"
using immesh::nccl; using immesh::nccl_uid_t; using immesh::nccl_comm_t; using immesh::kNcclUint32; using immesh::kNcclUint64; using immesh::kNcclSum;

static void fill_params(const immesh_lio_config* c, LioParams& P) {
    P.voxel_size = c->voxel_size;
    P.voxel_size_f = (float)c->voxel_size;
    P.voxel_size_ins = (double)P.voxel_size_f;
    P.max_layer = c->max_layer;
    for (int i = 0; i < 5; ++i) P.layer_init[i] = c->layer_init_size[i];
    P.max_points = c->max_points_size;
    P.planer_threshold = (float)c->min_eigen_value;
    P.dept_err = (float)c->dept_err;
    // DEG2RAD is PCL's macro ((x)*0.017453293); the squared sine is a per-configuration constant
    const float be = (float)c->beam_err;
    const double s = std::sin((double)be * 0.017453293);
    P.dir_var = s * s;
    const double sc = std::sin((double)(float)0.01 * 0.017453293);  // CALIB_ANGLE_COV, include/common_lib.h:41
    P.dir_var_calib = sc * sc;
    P.calib_laser = c->calib_laser;
    P.max_iter = c->max_iteration;
    for (int i = 0; i < 9; ++i) P.extR[i] = c->ext_R[i];
    for (int i = 0; i < 3; ++i) P.extT[i] = c->ext_T[i];
}

// Grids are fixed per handle (sized for max_scan_points, at most 8 waves of blocks; every per-point kernel is a grid-stride
// loop over the n it reads from the device-resident ScanDyn), so that the captured launch sequence is identical for every scan.
static int grid_fixed(const immesh_lio* h, int threads, int max_waves = 8) {
    long long g = ((long long)h->max_scan + threads - 1) / threads;
    const long long cap = (long long)h->n_sm * max_waves;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// scan publishers (immesh_lio_effect_cloud / immesh_lio_registered_cloud): the validity of the per-scan rows
static int scan_rows_status(const immesh_lio* h, const char* what) {
    if (h->scan_rows >= 0) return IMMESH_OK;
    return im_fail(IMMESH_E_INVALID, (std::string(what) + ": the per-scan buffers were overwritten by " + h->scan_rows_overwritten_by +
                                      " after the last IESKF run (immesh_lio_estimate / immesh_lio_step*)").c_str());
}

#if defined(IM_DEBUG_STAMPS)
extern "C" int immesh_debug_stamps(long long* out64) {   // debug variant only (tools/debug/build_stamps.sh); not declared in include/
    return cudaMemcpyFromSymbol(out64, immesh::g_stamps, 64 * sizeof(long long)) == cudaSuccess ? 0 : -1;
}
#endif

extern "C" {

int immesh_lio_create(const immesh_lio_config* cfg, immesh_lio_t** out) {
    if (!cfg || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    if (cfg->max_iteration < 1 || cfg->max_iteration > IM_MAX_ITER) return im_fail(IMMESH_E_INVALID, "max_iteration must be in [1,8]");
    if (cfg->max_layer < 0 || cfg->max_layer > 4) return im_fail(IMMESH_E_INVALID, "max_layer must be in [0,4]");
    if (!(cfg->voxel_size > 0) || cfg->max_points_size < 1) return im_fail(IMMESH_E_INVALID, "voxel_size and max_points_size must be positive");
    for (int i = 0; i < 5; ++i)
        if (cfg->layer_init_size[i] < 0) return im_fail(IMMESH_E_INVALID, "layer_init_size must be non-negative");
    if (cfg->hash_capacity_log2 != 0 && (cfg->hash_capacity_log2 < 10 || cfg->hash_capacity_log2 > 30)) return im_fail(IMMESH_E_INVALID, "hash_capacity_log2 must be 0 (default) or in [10,30]");
    if (cfg->max_nodes < 0 || cfg->max_chunks < 0 || cfg->max_scan_points < 0) return im_fail(IMMESH_E_INVALID, "capacities must be non-negative (0 = default)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path");
    immesh::Building<immesh_lio> owner(new immesh_lio(), immesh_lio_destroy);   // every failure below releases what was created
    immesh_lio* h = owner.get();
    fill_params(cfg, h->P);
    h->use_graph = std::getenv("IMMESH_GRAPH") ? std::atoi(std::getenv("IMMESH_GRAPH")) : 1;
    const int caplog = cfg->hash_capacity_log2 ? cfg->hash_capacity_log2 : 22;
    h->cap = (size_t)1 << caplog;
    h->max_nodes = cfg->max_nodes ? cfg->max_nodes : (4 << 20);
    h->max_chunks = cfg->max_chunks ? cfg->max_chunks : (4 << 20);
    h->max_scan = cfg->max_scan_points ? cfg->max_scan_points : (2 << 20);
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& e : h->ev) IM_CUDA(cudaEventCreate(&e));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CUDA(cudaEventCreateWithFlags(&h->ev_slot[i], cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_pose, cudaEventDisableTiming));
    VoxelMapDev& m = h->map;
    IM_CUDA(h->dev.alloc(&m.keys, h->cap, 0xFF));
    IM_CUDA(h->dev.alloc(&m.root_node, h->cap, 0xFF));
    m.cap_mask = (unsigned)(h->cap - 1);
    IM_CUDA(h->dev.alloc(&m.nodes, (size_t)h->max_nodes));
    IM_CUDA(h->dev.alloc(&m.planes, (size_t)h->max_nodes));
    IM_CUDA(h->dev.alloc(&m.chunks, (size_t)h->max_chunks));
    IM_CUDA(h->dev.alloc(&m.avail, (size_t)h->max_chunks));
    IM_CUDA(h->dev.alloc(&m.pending, (size_t)h->max_chunks));
    IM_CUDA(h->dev.alloc(&h->d_counters, IM_LC_SIZE, 0));
    m.node_count = h->d_counters + IM_LC_NODES; m.chunk_bump = h->d_counters + IM_LC_CHUNK_BUMP; m.avail_top = h->d_counters + IM_LC_AVAIL_TOP;
    m.pending_n = h->d_counters + IM_LC_PENDING; m.err = h->d_counters + IM_LC_ERR; m.n_roots = h->d_counters + IM_LC_ROOTS;
    m.stat = h->d_counters + IM_LC_REFITS;   // [0] refits, [1] refit points
    m.max_nodes = h->max_nodes; m.max_chunks = h->max_chunks;
    IM_CUDA(h->dev.alloc(&m.pub, (size_t)h->max_nodes));
    IM_CUDA(h->dev.alloc(&m.pub_mark, h->cap, 0));
    IM_CUDA(h->dev.alloc(&m.pub_list, h->cap));
    m.pub_n = h->d_counters + IM_LC_PUB_N;
    m.node_free = nullptr;   // allocated by the first immesh_lio_local_map / immesh_voxelmap_evict_boxes
    m.node_free_top = h->d_counters + IM_LC_NODE_FREE; m.n_tombs = h->d_counters + IM_LC_TOMBS;
    ScanBuf& sb = h->sb;
    const size_t ms = (size_t)h->max_scan;
    float* d_body = nullptr;
    IM_CUDA(h->dev.alloc(&d_body, IM_SLOTS * ms * 3));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream_up, cudaStreamNonBlocking));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CUDA(cudaEventCreateWithFlags(&h->ev_up[i], cudaEventDisableTiming));
    sb.body = d_body;
    h->d_body_own = d_body;
    IM_CUDA(h->dev.alloc(&sb.body_cov, ms * 6));
    IM_CUDA(h->dev.alloc(&sb.p_imu, ms * 3));
    IM_CUDA(h->dev.alloc(&sb.bv_imu, ms * 6));
    IM_CUDA(h->dev.alloc(&sb.match_node, ms, 0xFF));
    IM_CUDA(h->dev.alloc(&sb.match_layer, ms, 0));
    IM_CUDA(h->dev.alloc(&sb.wsqrt, ms));
    IM_CUDA(h->dev.alloc(&sb.pw, ms * 3));
    IM_CUDA(h->dev.alloc(&sb.var, ms * 6));
    IM_CUDA(h->dev.alloc(&sb.sortkey, ms));
    IM_CUDA(h->dev.alloc(&sb.slot, ms));
    IM_CUDA(h->dev.alloc(&sb.seg, ms));
    IM_CUDA(h->dev.alloc(&h->d_sorted, ms));
    IM_CUDA(h->dev.alloc(&h->d_complex, ms));
    IM_CUDA(h->dev.alloc(&sb.touched, ms));
    IM_CUDA(h->dev.alloc(&sb.slot_count, h->cap, 0));
    IM_CUDA(h->dev.alloc(&sb.slot_offset, h->cap, 0));
    IM_CUDA(h->dev.alloc(&sb.slot_cursor, h->cap, 0));
    sb.n_touched = h->d_counters + IM_LC_TOUCHED; sb.seg_top = h->d_counters + IM_LC_SEG_TOP;
    sb.n = 0;
    IM_CUDA(h->dev.alloc(&h->d_ctrl, 1, 0));
    sb.dyn = &h->d_ctrl->dyn;
    IM_CUDA(h->pinned.alloc(&h->h_body, IM_SLOTS * ms * 3));
    IM_CUDA(h->pinned.alloc(&h->h_state, IM_STATE_DOUBLES + 64));
    IM_CUDA(h->pinned.alloc(&h->h_ints, IM_HINT_SIZE));
    IM_CUDA(h->pinned.alloc(&h->h_dyn, IM_SLOTS));
    IM_CUDA(h->pinned.alloc(&h->h_out, IM_SLOTS));
    std::memset(h->h_out, 0, IM_SLOTS * sizeof(LioOut));
    // StatesGroup(): identity rotation, cov = INIT_COV * I  (include/common_lib.h:201-211)
    std::memset(h->h_state, 0, IM_STATE_DOUBLES * sizeof(double));
    h->h_state[0] = h->h_state[4] = h->h_state[8] = 1.0;
    for (int i = 0; i < 18; ++i) h->h_state[24 + i * 18 + i] = 0.0000001;
    IM_CUDA(cudaMemcpy(h->d_ctrl->state, h->h_state, IM_STATE_DOUBLES * sizeof(double), cudaMemcpyHostToDevice));
    IM_CUDA(cudaDeviceSynchronize());
    *out = owner.release();
    return IMMESH_OK;
}

static void feed_free(immesh_lio* h);

int immesh_lio_destroy(immesh_lio_t* h) {
    if (!h) return IMMESH_OK;
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->graph.destroy();
    feed_free(h);
    if (h->win.local) immesh::peer_window_close(h->win);
    if (h->nccl_comm && nccl().CommDestroy) nccl().CommDestroy(h->nccl_comm);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    if (h->ev_pose) cudaEventDestroy(h->ev_pose);
    for (int i = 0; i < IM_SLOTS; ++i) if (h->ev_up[i]) cudaEventDestroy(h->ev_up[i]);
    if (h->stream_up) cudaStreamDestroy(h->stream_up);
    if (h->ev_mark) cudaEventDestroy(h->ev_mark);
    if (h->stream) cudaStreamDestroy(h->stream);
    for (int i = 0; i < IM_SLOTS; ++i) if (h->ev_slot[i]) cudaEventDestroy(h->ev_slot[i]);
    cudaGetLastError();
    delete h;
    return IMMESH_OK;
}

// ---- multi-GPU: shard the VoxelMap of this handle over `nranks` processes (one GPU each, NCCL over NVLink)
int immesh_comm_unique_id(char* out128) {
    if (!out128) return im_fail(IMMESH_E_INVALID, "null argument");
    if (!nccl().load()) return im_fail(IMMESH_E_CUDA, "libnccl.so.2 not found");
    nccl_uid_t id;
    if (nccl().GetUniqueId(&id)) return im_fail(IMMESH_E_CUDA, "ncclGetUniqueId failed");
    std::memcpy(out128, id.internal, 128);
    return IMMESH_OK;
}
int immesh_lio_shard(immesh_lio_t* h, int rank, int nranks, const char* unique_id128) {
    if (!h || !unique_id128 || nranks < 1 || rank < 0 || rank >= nranks) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (nranks > IM_MAX_RANKS) return im_fail(IMMESH_E_INVALID, "at most 8 ranks (one node)");
    if (nranks == 1) { h->P.shard_rank = 0; h->P.shard_n = 1; return IMMESH_OK; }
    if (h->grow_max_bytes > 0) return im_fail(IMMESH_E_INVALID, "a handle with automatic growth cannot be sharded (immesh_lio_set_growth(h, 0) first)");
    if (h->feed.on) return im_fail(IMMESH_E_INVALID, "a handle with the scan feed on cannot be sharded (immesh_lio_feed_enable(h, NULL) first)");
    if (h->lm_on || h->map.node_free)   // its tombstones would need a rebuild of the table, which a sharded handle cannot do
        return im_fail(IMMESH_E_INVALID, "a handle that used the local map (immesh_lio_local_map / immesh_voxelmap_evict_boxes) cannot be sharded");
    if (!nccl().load()) return im_fail(IMMESH_E_CUDA, "libnccl.so.2 not found");
    nccl_uid_t id;
    std::memcpy(id.internal, unique_id128, 128);
    nccl_comm_t comm = nullptr;
    const int rc = nccl().CommInitRank(&comm, nranks, id, rank);
    if (rc) return im_fail(IMMESH_E_CUDA, nccl().GetErrorString ? nccl().GetErrorString(rc) : "ncclCommInitRank failed");
    h->nccl_comm = comm;
    h->P.shard_rank = rank;
    h->P.shard_n = nranks;
    h->graph.destroy();   // the launch sequence changes
    h->words_cap = h->max_scan / 32 + 2;
    if (!h->d_bits) IM_CUDA(h->dev.alloc(&h->d_bits, (size_t)2 * h->words_cap, 0));
    // peer window over NVLink (CUDA IPC): the exchanges of the residual pass are then fused into its kernels.  IMMESH_SHARD_NCCL=1
    // keeps the NCCL all-reduce sequence (the baseline the fused path is measured against; same setting on every rank).  The
    // open is collective and its outcome is the same on every rank (peer_win.cuh).
    const char* force_nccl = std::getenv("IMMESH_SHARD_NCCL");
    if (!(force_nccl && force_nccl[0] == '1')) {
        const size_t bytes = IM_LIOWIN_BITS_OFF + (size_t)IM_MAX_RANKS * 2 * h->words_cap * sizeof(unsigned int);
        const cudaError_t e = immesh::peer_window_open(h->win, bytes, rank, nranks, comm, h->stream);
        if (e != cudaSuccess) {
            std::fprintf(stderr, "[immesh_b200] rank %d: peer window unavailable on some rank (%s here); all ranks use NCCL all-reduces for the sharded residual pass\n", rank, cudaGetErrorString(e));
            cudaGetLastError();
        }
    }
    return IMMESH_OK;
}
int immesh_lio_shard_transport(immesh_lio_t* h) {   // 0 = not sharded, 1 = NCCL all-reduces, 2 = fused peer-window exchange
    if (!h) return 0;
    if (h->P.shard_n <= 1) return 0;
    return h->win.ok ? 2 : 1;
}

int immesh_lio_set_state(immesh_lio_t* h, const double* s) {
    if (!h || !s) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(h->h_state, s, IM_STATE_DOUBLES * sizeof(double));
    IM_CUDA(cudaMemcpyAsync(h->d_ctrl->state, h->h_state, IM_STATE_DOUBLES * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    h->pose_pub_idx = -1;
    return IMMESH_OK;
}
int immesh_lio_get_state(immesh_lio_t* h, double* s) {
    if (!h || !s) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaMemcpyAsync(h->h_state, h->d_ctrl->state, IM_STATE_DOUBLES * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(s, h->h_state, IM_STATE_DOUBLES * sizeof(double));
    return IMMESH_OK;
}

static int push_dyn(immesh_lio* h, int n, int slot = 0, double dt = 0.0, double cov_gyr = 0.0, double cov_acc = 0.0);
// per-scan inputs: the scan itself (host: staged through pinned slot `slot` unless the caller's buffer is pinned already) and
// the ScanDyn block every kernel of the sequence reads; both in stream order, so the previous scan is never disturbed
static int upload_scan(immesh_lio* h, const float* body, int n, int on_device = 0, int slot = 0, double dt = 0.0, double cov_gyr = 0.0, double cov_acc = 0.0) {
    if ((!body && n > 0) || n < 0) return im_fail(IMMESH_E_INVALID, "bad scan");
    if (n > h->max_scan) return im_fail(IMMESH_E_CAPACITY, "scan larger than max_scan_points");
    if (on_device) {
        h->sb.body = body;  // caller-owned device buffer, must stay valid until the next call on this handle
    } else {
        float* dst = h->d_body_own + (size_t)slot * h->max_scan * 3;   // the slot's previous user has finished (ev_slot waited on by the caller)
        h->sb.body = dst;
        if (n > 0)
            IM_CUDA(immesh::upload_async(dst, body, (size_t)n * 3 * sizeof(float), h->h_body + (size_t)slot * h->max_scan * 3, h->stream_up, h->ev_up[slot], h->stream));
    }
    return push_dyn(h, n, slot, dt, cov_gyr, cov_acc);
}
static int push_dyn(immesh_lio* h, int n, int slot, double dt, double cov_gyr, double cov_acc) {
    ++h->uploads;
    h->sb.n = n;
    h->last_n = n;
    ScanDyn& d = h->h_dyn[slot];
    d.body = h->sb.body;
    d.n = n;
    d.scan_idx = h->scan_counter;
    d.dt = dt; d.cov_gyr = cov_gyr; d.cov_acc = cov_acc;
    d.epoch = h->win.epoch;
    d.mode = 0; d.pad_ = 0;
    d.n_dev = h->next_n_dev;
    h->next_n_dev = nullptr;
    h->dyn_last = d;
    h->dyn_last.dt = 0.0;
    IM_CUDA(cudaMemcpyAsync(&h->d_ctrl->dyn, &d, sizeof(ScanDyn), cudaMemcpyHostToDevice, h->stream));
    return IMMESH_OK;
}
static int lio_flags_status(int err) {
    if (err & (IM_ERR_NODE_POOL | IM_ERR_CHUNK_POOL | IM_ERR_HASH_FULL | IM_ERR_SEG_POOL)) return im_fail(IMMESH_E_CAPACITY, "device pool overflow (raise the capacities in immesh_lio_config)");
    if (err & IM_ERR_IMU_CARRY) return im_fail(IMMESH_E_CAPACITY, "immesh_lio_step_async_depth_imu: carried and new IMU samples exceeded max_imu (the frame's samples were dropped)");
    if (err & (IM_ERR_KEY_RANGE | IM_ERR_FX_RANGE)) return im_fail(IMMESH_E_RANGE, "coordinate / normal-equation term outside the representable range");
    if (err & IM_ERR_PEER_TIMEOUT) return im_fail(IMMESH_E_CUDA, "sharded mode: a peer rank did not publish its data in time (peer window epoch flag)");
    return IMMESH_OK;
}
// the calls that reuse the per-scan buffers for their own points: the effect / registered rows of the last run are gone
static void scan_rows_overwritten(immesh_lio* h, const char* by) {
    h->scan_rows = -1;
    h->scan_rows_overwritten_by = by;
}
// counters of map-growing step number `step`, finished: the use the growth check starts from, and the largest use of one step seen
// so far (an older block arriving late is skipped)
static void note_counters(immesh_lio* h, const int* c, long long step) {
    if (step <= h->known_step) return;
    // the difference to the last known step; over several steps (their blocks were not all seen) it bounds one step from above
    h->max_step_nodes = std::max(h->max_step_nodes, c[IM_LC_NODES] - h->known[IM_LC_NODES]);
    h->max_step_chunks = std::max(h->max_step_chunks, c[IM_LC_CHUNK_BUMP] - h->known[IM_LC_CHUNK_BUMP]);
    std::memcpy(h->known, c, sizeof(h->known));
    h->known_step = step;
}
// the result blocks of the finished steps still in the staging slots, in step order (consecutive steps: one step's use each)
static void note_slots(immesh_lio* h, bool only_finished) {
    int order[IM_SLOTS], n = 0;
    for (int s = 0; s < IM_SLOTS; ++s)
        if (h->slot_busy[s] && (!only_finished || cudaEventQuery(h->ev_slot[s]) == cudaSuccess)) order[n++] = s;
    cudaGetLastError();   // cudaErrorNotReady of the queries
    std::sort(order, order + n, [&](int a, int b) { return h->slot_step[a] < h->slot_step[b]; });
    for (int i = 0; i < n; ++i) note_counters(h, h->h_out[order[i]].counters, h->slot_step[order[i]]);
}
// the counter block into c (IM_LC_SIZE ints), blocking: the caller has drained what it needs
static cudaError_t lio_read_counters(const immesh_lio* h, int* c) {
    return cudaMemcpy(c, h->d_counters, IM_LC_SIZE * sizeof(int), cudaMemcpyDeviceToHost);
}
static int check_flags(immesh_lio* h) {
    IM_CUDA(cudaMemcpyAsync(h->h_ints, h->d_counters, IM_LC_SIZE * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    h->tombs_known = h->h_ints[IM_LC_TOMBS];
    if (h->grow_max_bytes > 0) note_counters(h, h->h_ints, h->map_steps);
    return lio_flags_status(h->h_ints[IM_LC_ERR]);
}

// ---- growth of the map pools.  Bytes per record: root slot 32 (key 8, root_node 4, pub_mark 4, pub_list 4, the per-scan
// slot_count / slot_offset / slot_cursor 12), node 944 (NodeRec 656, PlaneRec 256, PubRec 32), chunk 520 (Chunk 512, avail 4,
// pending 4).  Node, chunk and slot ids are 32-bit ints, and the allocating atomics may count past a full pool: every pool stops
// at 2^30 records.
#define IM_POOL_LIMIT (1LL << 30)
static const size_t kSlotBytes = 8 + 4 + 4 + 4 + 3 * 4;
static const size_t kNodeBytes = sizeof(NodeRec) + sizeof(PlaneRec) + sizeof(PubRec);
static const size_t kChunkBytes = sizeof(Chunk) + 2 * sizeof(int);

static size_t pool_bytes(long long cap, long long nodes, long long chunks) {
    return (size_t)cap * kSlotBytes + (size_t)nodes * kNodeBytes + (size_t)chunks * kChunkBytes;
}
// Enlarge the pools to (cap slots, nodes, chunks), each >= the current one.  Drains the handle's stream; allocates every new
// buffer before anything is touched, so that a failure (allocation, ceiling, id limits) leaves the handle as it was; migrates on
// the stream; frees the old buffers after the migration and drops the captured launch sequence (it holds the old pointers).
static int lio_grow(immesh_lio* h, long long cap, long long nodes, long long chunks, bool rehash = false) {
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    const long long cap0 = (long long)h->cap, nodes0 = h->max_nodes, chunks0 = h->max_chunks;
    if (cap > IM_POOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "root hash: more than 2^30 slots (32-bit slot ids)");
    if (nodes > IM_POOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "node pool: more than 2^30 node records (32-bit node ids)");
    if (chunks > IM_POOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "chunk pool: more than 2^30 chunks (32-bit chunk ids)");
    const bool g_cap = cap > cap0 || rehash, g_nodes = nodes > nodes0, g_chunks = chunks > chunks0;   // rehash: the table at its size
    if (!g_cap && !g_nodes && !g_chunks) return IMMESH_OK;
    size_t bytes = h->dev.bytes() - pool_bytes(cap0, nodes0, chunks0) + pool_bytes(cap, nodes, chunks);
    if (h->map.node_free) bytes += (size_t)(nodes - nodes0) * sizeof(int);   // the local map's node free stack follows the node pool
    if (h->grow_max_bytes > 0 && bytes > (size_t)h->grow_max_bytes) {
        const std::string pools = std::string(g_cap ? " root hash" : "") + (g_nodes ? " node pool" : "") + (g_chunks ? " chunk pool" : "");
        return im_fail(IMMESH_E_CAPACITY, ("growth of the" + pools + " to " + std::to_string(bytes) + " device bytes is above the ceiling of " +
                                           std::to_string(h->grow_max_bytes) + " (immesh_lio_set_growth)").c_str());
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));
    IM_CUDA(lio_read_counters(h, h->h_ints));
    const int* c = h->h_ints;
    const int n_nodes = std::min(c[IM_LC_NODES], h->max_nodes), n_chunks = std::min(c[IM_LC_CHUNK_BUMP], h->max_chunks);
    const int n_avail = std::max(0, std::min(c[IM_LC_AVAIL_TOP], h->max_chunks)), n_pending = std::min(c[IM_LC_PENDING], h->max_chunks);
    const int n_pub = std::min<long long>(c[IM_LC_PUB_N], cap0);
    const int n_free = std::max(0, std::min(c[IM_LC_NODE_FREE], h->max_nodes));
    const bool had_tombs = c[IM_LC_TOMBS] > 0;

    VoxelMapDev nm = h->map;   // the map after the growth
    ScanBuf nsb = h->sb;
    int* slot_map = nullptr;
    immesh::MemSet fresh, tmp;   // the new buffers (freed on every failure below); the slot map of the rehash (freed on return)
    const char* pool = "";
    cudaError_t e = cudaSuccess;
    if (g_nodes && e == cudaSuccess) {
        pool = "node pool";
        if ((e = fresh.alloc(&nm.nodes, nodes)) == cudaSuccess && (e = fresh.alloc(&nm.planes, nodes)) == cudaSuccess) e = fresh.alloc(&nm.pub, nodes);
        if (e == cudaSuccess && h->map.node_free) e = fresh.alloc(&nm.node_free, nodes);
    }
    if (g_chunks && e == cudaSuccess) {
        pool = "chunk pool";
        if ((e = fresh.alloc(&nm.chunks, chunks)) == cudaSuccess && (e = fresh.alloc(&nm.avail, chunks)) == cudaSuccess) e = fresh.alloc(&nm.pending, chunks);
    }
    if (g_cap && e == cudaSuccess) {
        pool = "root hash";
        if ((e = fresh.alloc(&nm.keys, cap)) == cudaSuccess && (e = fresh.alloc(&nm.root_node, cap)) == cudaSuccess && (e = fresh.alloc(&nm.pub_mark, cap)) == cudaSuccess &&
            (e = fresh.alloc(&nm.pub_list, cap)) == cudaSuccess && (e = fresh.alloc(&nsb.slot_count, cap)) == cudaSuccess &&
            (e = fresh.alloc(&nsb.slot_offset, cap)) == cudaSuccess && (e = fresh.alloc(&nsb.slot_cursor, cap)) == cudaSuccess)
            e = tmp.alloc(&slot_map, cap0);
    }
    if (e != cudaSuccess)
        return im_fail_alloc(e, (std::string(pool) + ": device allocation for the growth failed (" + cudaGetErrorString(e) + "); the handle is unchanged").c_str());
    cudaStream_t st = h->stream;
    auto migrate = [&]() -> cudaError_t {
        cudaError_t r = cudaSuccess;
#define MG(x) do { if ((r = (x)) != cudaSuccess) return r; } while (0)
        if (g_nodes && n_nodes > 0) {
            MG(cudaMemcpyAsync(nm.nodes, h->map.nodes, (size_t)n_nodes * sizeof(NodeRec), cudaMemcpyDeviceToDevice, st));
            MG(cudaMemcpyAsync(nm.planes, h->map.planes, (size_t)n_nodes * sizeof(PlaneRec), cudaMemcpyDeviceToDevice, st));
            MG(cudaMemcpyAsync(nm.pub, h->map.pub, (size_t)n_nodes * sizeof(PubRec), cudaMemcpyDeviceToDevice, st));
        }
        if (g_nodes && nm.node_free && n_free > 0) MG(cudaMemcpyAsync(nm.node_free, h->map.node_free, (size_t)n_free * sizeof(int), cudaMemcpyDeviceToDevice, st));
        if (g_chunks) {
            if (n_chunks > 0) MG(cudaMemcpyAsync(nm.chunks, h->map.chunks, (size_t)n_chunks * sizeof(Chunk), cudaMemcpyDeviceToDevice, st));
            if (n_avail > 0) MG(cudaMemcpyAsync(nm.avail, h->map.avail, (size_t)n_avail * sizeof(int), cudaMemcpyDeviceToDevice, st));
            if (n_pending > 0) MG(cudaMemcpyAsync(nm.pending, h->map.pending, (size_t)n_pending * sizeof(int), cudaMemcpyDeviceToDevice, st));
        }
        if (g_cap) {
            MG(cudaMemsetAsync(nm.keys, 0xFF, (size_t)cap * 8, st));
            MG(cudaMemsetAsync(nm.root_node, 0xFF, (size_t)cap * 4, st));
            MG(cudaMemsetAsync(nm.pub_mark, 0, (size_t)cap * 4, st));
            for (int* p : {nsb.slot_count, nsb.slot_offset, nsb.slot_cursor}) MG(cudaMemsetAsync(p, 0, (size_t)cap * 4, st));
            nm.cap_mask = (unsigned)(cap - 1);
            const int g = (int)std::min<long long>((cap0 + GROW_THREADS - 1) / GROW_THREADS, (long long)h->n_sm * 16);
            IM_LAUNCH(k_rehash_roots, g, GROW_THREADS, 0, st, h->map, nm, slot_map);
            // with the node pool kept, root_slot is rewritten in place: the last step of the migration, after every allocation succeeded
            const int gn = (int)std::min<long long>((std::max(n_nodes, n_pub) + GROW_THREADS - 1) / GROW_THREADS + 1, (long long)h->n_sm * 16);
            IM_LAUNCH(k_remap_roots, gn, GROW_THREADS, 0, st, nm, n_nodes, (const int*)h->map.pub_list, n_pub, (const int*)slot_map);
            MG(cudaMemsetAsync(nm.n_tombs, 0, sizeof(int), st));   // the rebuilt table holds no tombstone
        }
        MG(cudaGetLastError());
        MG(cudaStreamSynchronize(st));
        if (g_cap && had_tombs && n_pub > 0) {
            // pending plane-marker entries of evicted roots were remapped to -1: the list keeps the others, in order
            std::vector<int> lst(n_pub);
            MG(cudaMemcpy(lst.data(), nm.pub_list, (size_t)n_pub * sizeof(int), cudaMemcpyDeviceToHost));
            const int kept = (int)(std::remove(lst.begin(), lst.end(), -1) - lst.begin());
            if (kept > 0) MG(cudaMemcpy(nm.pub_list, lst.data(), (size_t)kept * sizeof(int), cudaMemcpyHostToDevice));
            MG(cudaMemcpy(nm.pub_n, &kept, sizeof(int), cudaMemcpyHostToDevice));
        }
#undef MG
        return r;
    };
    if ((e = migrate()) != cudaSuccess) {   // a sticky CUDA error: nothing new is kept
        cudaGetLastError();
        return immesh::im_fail_cuda(e, __FILE__, __LINE__);
    }
    // the replaced buffers go; the new ones join the handle's device memory
    if (g_nodes) { h->dev.free(h->map.nodes); h->dev.free(h->map.planes); h->dev.free(h->map.pub); if (h->map.node_free) h->dev.free(h->map.node_free); }
    if (g_chunks) { h->dev.free(h->map.chunks); h->dev.free(h->map.avail); h->dev.free(h->map.pending); }
    if (g_cap) {
        for (const void* p : {(const void*)h->map.keys, (const void*)h->map.root_node, (const void*)h->map.pub_mark, (const void*)h->map.pub_list,
                              (const void*)h->sb.slot_count, (const void*)h->sb.slot_offset, (const void*)h->sb.slot_cursor})
            h->dev.free(p);
    }
    h->dev.take(std::move(fresh));
    nm.max_nodes = (int)nodes;
    nm.max_chunks = (int)chunks;
    h->map = nm;
    h->sb = nsb;
    h->cap = (size_t)cap;
    h->max_nodes = (int)nodes;
    h->max_chunks = (int)chunks;
    if (cap > cap0 || g_nodes || g_chunks) h->growths++;
    if (g_cap) h->tombs_known = 0;
    h->graph.destroy();   // the next pipelined step captures the launch sequence again, with the new pointers
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}
// Automatic growth (immesh_lio_set_growth) before a step of n points is queued: growth_targets (pool_growth.cuh) on the use of the
// last step known to have finished, without waiting for the others.  Only when a pool is short is the handle drained; the decision
// is then taken again on its exact counters.
// Purge of the local map's tombstones before a step: when the last finished step left more than an eighth of the root hash's slots
// as tombstones, the handle is drained and the table rebuilt at its size through the growth's rehash, which drops them (hash_find
// walks a probe chain that tombstones only lengthen).  Independent of immesh_lio_set_growth.
static int lio_purge_check(immesh_lio* h) {
    if (!h->map.node_free) return IMMESH_OK;   // nothing was ever evicted
    long long newest = -1;
    for (int s = 0; s < IM_SLOTS; ++s)
        if (h->slot_busy[s] && h->slot_step[s] > newest && cudaEventQuery(h->ev_slot[s]) == cudaSuccess) {
            newest = h->slot_step[s];
            h->tombs_known = h->h_out[s].counters[IM_LC_TOMBS];
        }
    cudaGetLastError();   // cudaErrorNotReady of the queries
    if ((long long)h->tombs_known * 8 <= (long long)h->cap) return IMMESH_OK;
    IM_CUDA(cudaStreamSynchronize(h->stream));
    IM_CUDA(lio_read_counters(h, h->h_ints));
    h->tombs_known = h->h_ints[IM_LC_TOMBS];
    if ((long long)h->tombs_known * 8 <= (long long)h->cap) return IMMESH_OK;
    const int rc = lio_grow(h, (long long)h->cap, h->max_nodes, h->max_chunks, true);
    if (rc == IMMESH_OK) h->lm_purges++;
    return rc;
}
static int lio_growth_check(immesh_lio* h, long long n) {
    const int prc = lio_purge_check(h);
    if (prc) return prc;
    if (h->grow_max_bytes <= 0) return IMMESH_OK;
    long long steps = 1, n_max = n;
    note_slots(h, true);
    for (int s = 0; s < IM_SLOTS; ++s) {
        if (h->slot_busy[s] && h->slot_step[s] > h->known_step) {   // still in flight
            ++steps;
            n_max = std::max<long long>(n_max, h->h_dyn[s].n);
        }
    }
    for (int pass = 0; pass < 2; ++pass) {
        long long cap = (long long)h->cap, nodes = h->max_nodes, chunks = h->max_chunks;
        growth_targets(h->known, steps, n_max, h->max_step_nodes, h->max_step_chunks, &cap, &nodes, &chunks);
        const bool short_pool = cap > (long long)h->cap || nodes > h->max_nodes || chunks > h->max_chunks;
        if (!short_pool) return IMMESH_OK;
        if (pass == 1) return lio_grow(h, cap, nodes, chunks);
        IM_CUDA(cudaStreamSynchronize(h->stream));
        note_slots(h, false);
        IM_CUDA(lio_read_counters(h, h->h_ints));
        note_counters(h, h->h_ints, h->map_steps);
        steps = 1;
        n_max = n;
    }
    return IMMESH_OK;
}
// the local map's two launches: the box rule (boxes == null; gated on the device by LocalMapCtrl::on) or the caller's boxes, then the
// eviction sweep.  pdl as in launch_grow.
static void launch_local_map(immesh_lio* h, const float* boxes = nullptr, int n_boxes = 0, bool pdl = false) {
    IM_LAUNCH_PDL(pdl, k_local_map_box, 1, 32, 0, h->stream, h->d_ctrl, h->map.node_free_top, boxes ? 0 : 1);
    IM_LAUNCH_PDL(pdl, k_evict_roots, grid_fixed(h, EVICT_THREADS), EVICT_THREADS, 0, h->stream, h->map, h->d_ctrl, boxes, n_boxes);
}
// resident blocks per SM of the persistent per-voxel map update k_grow_voxel (headroom for the kernels on the other streams)
#define GROW_VOXEL_BPS 4
// map growth of the scan described by the device-resident ScanDyn.  pdl: every launch is a programmatic dependent launch (the
// sequence directly follows a kernel on h->stream, with no event or copy in between)
static void launch_grow(immesh_lio* h, int mode, bool pdl = false) {
    const int g = grid_fixed(h, 128);
    IM_LAUNCH_PDL(pdl, k_grow_point, g, 128, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, mode);
    IM_LAUNCH_PDL(pdl, k_grow_segment, grid_fixed(h, 128, 2), 128, 0, h->stream, h->sb);
    IM_LAUNCH_PDL(pdl, k_grow_scatter, g, 128, 0, h->stream, h->sb);
    int* n_complex = h->d_counters + IM_LC_COMPLEX;
    IM_LAUNCH_PDL(pdl, k_grow_simple, h->n_sm * 16, 128, 0, h->stream, h->map, h->P, h->sb, mode, h->d_complex, n_complex);
    IM_LAUNCH_PDL(pdl, k_grow_voxel, h->n_sm * GROW_VOXEL_BPS, 128, 0, h->stream, h->map, h->P, h->sb, mode, h->d_sorted, h->d_counters + IM_LC_WORK, (const int*)h->d_complex, (const int*)n_complex);
    IM_LAUNCH_PDL(pdl, k_grow_finish, 1, 256, 0, h->stream, h->map, h->sb, h->d_ctrl, h->d_counters);
}
// IESKF iterations.  One GPU: per iteration k_match then k_terms; the last block of k_terms runs the 6x6 IESKF update.
// Sharded over peer windows: pass1(+publish bits) -> pass2(wait bits, +publish sums) -> solve(wait sums), exchanges fused in.
// Sharded over NCCL (baseline): pass1 -> all-reduce(bit words) -> pass2 -> all-reduce(58 int64 sums) -> solve.
// pdl (one GPU only): every launch is a programmatic dependent launch, as in launch_grow.
static int launch_estimate(immesh_lio* h, bool pdl = false) {
    IM_LAUNCH_PDL(pdl, k_reset_scan, 2, 256, 0, h->stream, h->sb, h->d_ctrl, 1);
    IM_LAUNCH_PDL(pdl, k_prepare, grid_fixed(h, 128), 128, 0, h->stream, h->P, h->sb);
    const int g = grid_fixed(h, RES_THREADS, 4);
    if (h->P.shard_n > 1 && h->win.ok) {
        LioPeers pe;
        for (int r = 0; r < IM_MAX_RANKS; ++r) pe.w[r] = h->win.peer[r];
        pe.rank = h->win.rank; pe.n = h->win.n; pe.words_cap = h->words_cap; pe.pad = 0;
        for (int it = 0; it < h->P.max_iter; ++it) {
            // one epoch per iteration on top of the scan's base (ScanDyn::epoch, advanced once per scan); the two phases have separate flag rows
            IM_LAUNCH(k_shard_pass1_p2p, g, RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, pe, 1 + it);
            IM_LAUNCH(k_shard_pass2_p2p, g, RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, it, pe, 1 + it);
            IM_LAUNCH(k_solve_p2p, 1, SOLVE_THREADS, 0, h->stream, h->P, h->d_ctrl, it, pe, 1 + it, h->map.err);
        }
        return IMMESH_OK;
    }
    if (h->P.shard_n > 1) {
        const int words = h->words_cap;
        for (int it = 0; it < h->P.max_iter; ++it) {
            IM_CUDA(cudaMemsetAsync(h->d_bits, 0, (size_t)2 * words * sizeof(unsigned int), h->stream));
            IM_LAUNCH(k_shard_pass1, g, RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, h->d_bits, words);
            if (nccl().AllReduce(h->d_bits, h->d_bits, (size_t)2 * words, kNcclUint32, kNcclSum, h->nccl_comm, h->stream)) return im_fail(IMMESH_E_CUDA, "ncclAllReduce(bits) failed");
            IM_LAUNCH(k_shard_pass2, g, RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, it, (const unsigned int*)h->d_bits, words);
            if (nccl().AllReduce(&h->d_ctrl->acc[it][0], &h->d_ctrl->acc[it][0], (size_t)IM_NTERMS * 2, kNcclUint64, kNcclSum, h->nccl_comm, h->stream)) return im_fail(IMMESH_E_CUDA, "ncclAllReduce(acc) failed");
            IM_LAUNCH(k_solve, 1, SOLVE_THREADS, 0, h->stream, h->P, h->d_ctrl, it);
        }
        return IMMESH_OK;
    }
    const int gm = h->n_sm * 8;   // one resident wave of k_match blocks (__launch_bounds__(128, 8)); k_match picks the lanes per point from n
    for (int it = 0; it < h->P.max_iter; ++it) {
        IM_LAUNCH_PDL(pdl, k_match, gm, MATCH_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl);
        IM_LAUNCH_PDL(pdl, k_terms, g, RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, it, 1);
    }
    return IMMESH_OK;
}

// ---- scan feed.  feed_stage copies the scan's FeedDyn from the pinned ring (in stream order ahead of its kernels); launch_feed queues
// the record (lio: the scan ran the IESKF, so the effect count, the head and the two row emitters; otherwise the head alone), then
// k_feed_done; feed_commit numbers the scan as queued and marks it with the feed's event.  pdl as in launch_grow.
static int feed_stage(immesh_lio* h, const immesh_lio::FeedNext& nx, int kind, int branch, bool lio) {
    immesh_lio::Feed& f = h->feed;
    const long long k = f.queued + 1;
    // the ring entry was last used IM_FEED_DYN_RING scans ago; the staging slots keep far fewer scans in flight, so this never drains
    if (*(volatile long long*)f.h_done < k - IM_FEED_DYN_RING) IM_CUDA(cudaStreamSynchronize(h->stream));
    FeedDyn& d = f.h_dyn[k % IM_FEED_DYN_RING];
    d.scan = k;
    d.kind = nx.kind >= 0 ? nx.kind : kind;
    d.branch = nx.kind >= 0 ? nx.branch : branch;
    d.lio = lio ? 1 : 0;
    d.src = (!lio || f.registered == 0) ? 0 : (f.registered == 2 && nx.pts) ? 2 : 1;
    d.pts = d.src == 2 ? nx.pts : nullptr;
    d.inten = d.src == 2 ? nx.inten : nullptr;
    d.n = d.src == 2 ? nx.n : 0;
    d.n_dev = d.src == 2 ? nx.n_dev : nullptr;
    d.pad_ = 0;
    d.branch_dev = nx.kind >= 0 ? nx.branch_dev : nullptr;
    IM_CUDA(cudaMemcpyAsync(&f.dev->dyn, &d, sizeof(FeedDyn), cudaMemcpyHostToDevice, h->stream));
    return IMMESH_OK;
}
// The plane-map markers (f.mk_rows > 0), behind the scan's rows: walk = the scan ran a map update (not the IMU chain's branch 1).
// The grids are fixed, so that the cost follows the pending count rather than the hash capacity the scratch covers.
static void launch_markers(immesh_lio* h, bool walk, bool pdl) {
    immesh_lio::Feed& f = h->feed;
    cudaStream_t st = h->stream;
    LioMarkDev* md = f.mk_dev;
    if (walk) {
        const size_t cap = f.mk_cap;
        unsigned int* ku[2] = {f.mk_sort, f.mk_sort + cap};
        unsigned int* vu[2] = {f.mk_sort + 2 * cap, f.mk_sort + 3 * cap};
        const int* n_dev = &md->n;
        const int tiles = (int)((cap + VG_TILE - 1) / VG_TILE);
        const int g = h->n_sm * 4, gs = std::min(tiles, h->n_sm);
        IM_LAUNCH_PDL(pdl, k_mark_begin, 1, 32, 0, st, (const int*)h->map.pub_n, md);
        int cur = 0;
        for (int half = 0; half < 2; ++half) {
            IM_LAUNCH_PDL(pdl, k_pub_keys, g, PUB_THREADS, 0, st, h->map, 0, n_dev, half, half ? (const unsigned int*)vu[cur] : (const unsigned int*)nullptr,
                          ku[cur ^ half], vu[cur ^ half]);
            cur = rs_sort_passes(st, ku, vu, cur ^ half, (int)cap, 4, f.mk_hist, n_dev, gs);
        }
        int* slots = (int*)ku[0];   // the keys are spent: the sorted order is in vu[cur]
        int* cnt = (int*)ku[1];
        IM_LAUNCH_PDL(pdl, k_pub_count, g, PUB_THREADS, 0, st, h->map, 0, n_dev, (const unsigned int*)vu[cur], slots, cnt, md->misc + 1);
        IM_LAUNCH_PDL(pdl, k_pub_scan, 1, 1024, 0, st, cnt, (const LioMarkDev*)md, md->misc);
        IM_LAUNCH_PDL(pdl, k_mark_head, 1, 32, 0, st, (const LioFeedDev*)f.dev, md, h->map.pub_n, f.mk_hdr, f.max_scans, f.mk_rows, 1);
        IM_LAUNCH_PDL(pdl, k_pub_emit, g, PUB_THREADS, 0, st, h->map, 0, (const int*)slots, (const int*)cnt, f.mk_ring, (const LioMarkDev*)md, f.mk_rows);
    } else {
        IM_LAUNCH_PDL(pdl, k_mark_head, 1, 32, 0, st, (const LioFeedDev*)f.dev, md, h->map.pub_n, f.mk_hdr, f.max_scans, f.mk_rows, 0);
    }
}
// the markers' sort scratch covers the hash capacity; a growth of the hash (drained, its launch sequence dropped) enlarges it here,
// before the next scan's launch sequence is queued or captured
static int markers_fit(immesh_lio* h) {
    immesh_lio::Feed& f = h->feed;
    if (f.mk_rows == 0 || f.mk_cap >= h->cap) return IMMESH_OK;
    IM_CUDA(im_stage_reset(h, [&f] { f.mk_scratch = immesh::MemSet(); f.mk_sort = nullptr; f.mk_hist = nullptr; f.mk_cap = 0; }));
    const size_t tiles = (h->cap + VG_TILE - 1) / VG_TILE;
    IM_CUDA(f.mk_scratch.alloc(&f.mk_sort, 4 * h->cap));
    IM_CUDA(f.mk_scratch.alloc(&f.mk_hist, 256 * tiles));
    f.mk_cap = h->cap;
    return IMMESH_OK;
}
static void launch_feed(immesh_lio* h, bool lio, bool walk, bool pdl = false) {
    immesh_lio::Feed& f = h->feed;
    cudaStream_t st = h->stream;
    const bool eff = lio && f.effect;
    if (eff) {
        IM_LAUNCH_PDL(pdl, k_eff_count, f.nb, SPUB_THREADS, 0, st, h->sb, f.tiles);
        IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, f.tiles, f.nb, f.tiles + f.nb);
    }
    IM_LAUNCH_PDL(pdl, k_feed_head, 1, FEED_THREADS, 0, st, h->sb, (const LioCtrl*)h->d_ctrl, (const int*)h->d_counters, f.dev, f.hdr, f.states, f.max_scans, f.max_rows,
                  eff ? (const int*)(f.tiles + f.nb) : (const int*)nullptr, f.skip);
    if (eff)
        IM_LAUNCH_PDL(pdl, k_eff_emit, f.nb, SPUB_THREADS, 0, st, h->P, h->sb, (const LioCtrl*)h->d_ctrl, (const int*)f.tiles, f.rows, f.idx, (const LioFeedDev*)f.dev, f.max_rows);
    if (lio && f.registered)
        IM_LAUNCH_PDL(pdl, k_reg_gather, h->n_sm * 8, SPUB_THREADS, 0, st, h->P, h->sb, (const LioCtrl*)h->d_ctrl, (const float*)nullptr, 0, 3, -1, f.skip, f.rows,
                      (const float*)nullptr, (const LioFeedDev*)f.dev, f.max_rows);
    if (f.mk_rows) launch_markers(h, walk, pdl);
    IM_LAUNCH_PDL(pdl, k_feed_done, 1, 32, 0, st, (const LioFeedDev*)f.dev, f.d_done);
}
static int feed_commit(immesh_lio* h) {
    ++h->feed.queued;
    IM_CUDA(cudaEventRecord(h->feed.ev, h->stream));
    return IMMESH_OK;
}
static void markers_free(immesh_lio* h) {
    immesh_lio::Feed& f = h->feed;
    f.mk_mem = immesh::MemSet();
    f.mk_scratch = immesh::MemSet();
    f.mk_dev = nullptr; f.mk_hdr = nullptr; f.mk_ring = nullptr; f.mk_sort = nullptr; f.mk_hist = nullptr;
    f.mk_rows = 0; f.mk_cap = 0;
}
static void feed_free(immesh_lio* h) {
    immesh_lio::Feed& f = h->feed;
    if (f.ev) cudaEventDestroy(f.ev);
    if (f.stream) cudaStreamDestroy(f.stream);
    f.ev = nullptr; f.stream = nullptr;
    f.dev_mem = immesh::MemSet();
    f.pinned = immesh::MemSet(immesh::MemSet::Pinned);
    f.dev = nullptr; f.hdr = nullptr; f.states = nullptr; f.rows = nullptr; f.idx = nullptr; f.tiles = nullptr;
    f.h_dyn = nullptr; f.h_done = nullptr; f.d_done = nullptr;
    f.on = 0; f.queued = 0;
    markers_free(h);
}

int immesh_lio_predict(immesh_lio_t* h, double dt, double cov_gyr, double cov_acc) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    ScanDyn& d = h->h_dyn[0];   // the scan described by the block stays what it was; only the prediction inputs change
    d = h->dyn_last;
    d.dt = dt; d.cov_gyr = cov_gyr; d.cov_acc = cov_acc;
    IM_CUDA(cudaMemcpyAsync(&h->d_ctrl->dyn, &d, sizeof(ScanDyn), cudaMemcpyHostToDevice, h->stream));
    IM_LAUNCH(k_predict, 1, PREDICT_THREADS, 0, h->stream, h->d_ctrl);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaStreamSynchronize(h->stream));
    h->pose_pub_idx = -1;
    return IMMESH_OK;
}

int immesh_voxelmap_build(immesh_lio_t* h, const float* body, int n) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int rc = lio_growth_check(h, n);
    if (rc) return rc;
    rc = upload_scan(h, body, n);
    if (rc) return rc;
    h->scan_rows = 0;   // the reference publishes no effect cloud after voxel_map_init
    ++h->map_steps;
    if (h->lm_on) launch_local_map(h);   // places the box at the building scan's pose
    launch_grow(h, 1);
    IM_CUDA(cudaGetLastError());
    return check_flags(h);
}

int immesh_lio_estimate(immesh_lio_t* h, const float* body, int n, int* iters_run) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    h->win.epoch += IM_MAX_ITER + 1;   // epoch base of this scan (same sequence of calls on every rank)
    int rc = upload_scan(h, body, n);
    if (rc) return rc;
    if (h->lm_on) launch_local_map(h);
    rc = launch_estimate(h);
    if (rc) return rc;
    h->scan_rows = 1;
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_ints + IM_HINT_ITERS, &h->d_ctrl->iters_run, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    rc = check_flags(h);
    if (iters_run) *iters_run = h->h_ints[IM_HINT_ITERS];
    h->pose_pub_idx = -1;
    return rc;
}

int immesh_voxelmap_update(immesh_lio_t* h) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    const int rc = lio_growth_check(h, h->last_n);
    if (rc) return rc;
    ++h->map_steps;
    launch_grow(h, 0);
    IM_CUDA(cudaGetLastError());
    return check_flags(h);
}

// queue predict + estimate + update for one scan; no host synchronisation unless both staging slots are busy.  Host work per
// scan in the pipelined form: (memcpy into the pinned slot unless the caller's buffer is pinned) + H2D scan + H2D ScanDyn +
// ONE cudaGraphLaunch (no node is touched) + ONE D2H of the LioOut block + one event.
static int lio_enqueue(immesh_lio_t* h, const float* body, int n, int on_device, double dt, double cov_gyr, double cov_acc, bool allow_graph, int kind) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    const immesh_lio::FeedNext nx = h->feed_next;   // the front-end's or the IMU chain's scan, for this call only
    h->feed_next = immesh_lio::FeedNext();
    int grc = lio_growth_check(h, n);
    if (grc == IMMESH_OK) grc = markers_fit(h);
    if (grc) return grc;
    const int s = (++h->step_counter) & (IM_SLOTS - 1);
    if (h->slot_busy[s]) {
        const auto t0 = std::chrono::steady_clock::now();
        IM_CUDA(cudaEventSynchronize(h->ev_slot[s]));
        h->host_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        h->slot_busy[s] = 0;
    }
    h->win.epoch += IM_MAX_ITER + 1;   // epoch base of this scan: advanced exactly once per scan
    ++h->scan_counter;
    ++h->map_steps;   // (a replayed graph runs no host code of launch_grow: counted here)
    const bool timing = !(allow_graph && h->use_graph && !profiler().enabled && (h->P.shard_n <= 1 || h->win.ok));
    if (timing) IM_CUDA(cudaEventRecord(h->ev[0], h->stream));
    int rc = upload_scan(h, body, n, on_device, s, dt, cov_gyr, cov_acc);
    if (rc) return rc;
    if (h->feed.on) {
        rc = feed_stage(h, nx, kind, 0, true);
        if (rc) return rc;
    }
    // The pipelined entry points replay the scan's launch sequence as one CUDA graph, captured once: every per-scan value is
    // read from the device-resident ScanDyn, so a replay is a bare cudaGraphLaunch.  The blocking entry points launch
    // directly, with stage timing events in between.
    bool queued = false;
    int lrc = IMMESH_OK;
    if (!timing) {
        const unsigned sig = 1u | (h->feed.on ? 2u : 0u) | (h->lm_on ? 4u : 0u) | (h->win.ok ? 8u : 0u) | (h->feed.mk_rows ? 16u : 0u) | ((unsigned)h->P.max_iter << 8) |
                             ((unsigned)h->P.shard_n << 16);
        // one GPU: every kernel after k_predict is a programmatic dependent launch (the sharded paths wait on peers and NCCL)
        const bool pdl = h->P.shard_n <= 1;
        queued = immesh::run_graphed_static(h->graph, sig, h->stream, [&] {
            IM_LAUNCH(k_predict, 1, PREDICT_THREADS, 0, h->stream, h->d_ctrl);
            if (h->lm_on) launch_local_map(h, nullptr, 0, pdl);
            lrc = launch_estimate(h, pdl);
            launch_grow(h, 0, pdl);
            if (h->feed.on) launch_feed(h, true, true, pdl);
        }) == cudaSuccess;
        if (!queued) h->use_graph = 0;   // not expected; keep working through direct launches
    }
    if (!queued) {
        if (!timing) IM_CUDA(cudaEventRecord(h->ev[0], h->stream));
        IM_LAUNCH(k_predict, 1, PREDICT_THREADS, 0, h->stream, h->d_ctrl);
        if (h->lm_on) launch_local_map(h);
        IM_CUDA(cudaEventRecord(h->ev[1], h->stream));
        lrc = launch_estimate(h);
        IM_CUDA(cudaEventRecord(h->ev[2], h->stream));
        launch_grow(h, 0);
    }
    if (lrc) return lrc;
    h->scan_rows = 1;
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_out + s, &h->d_ctrl->out, sizeof(LioOut), cudaMemcpyDeviceToHost, h->stream));
    if (!queued) IM_CUDA(cudaEventRecord(h->ev[3], h->stream));
    if (h->feed.on) {
        if (!queued) launch_feed(h, true, true);   // behind ev[3]: immesh_lio_last_timing stays the step's own
        IM_CUDA(cudaGetLastError());
        rc = feed_commit(h);
        if (rc) return rc;
    }
    IM_CUDA(cudaEventRecord(h->ev_slot[s], h->stream));
    h->slot_busy[s] = 1;
    h->slot_step[s] = h->map_steps;
    h->timed_last = queued ? 0 : 1;
    h->pose_pub_idx = h->scan_counter;
    return IMMESH_OK;
}
static int lio_wait_impl(immesh_lio_t* h, double* state_out, int* iters_run, bool timings) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    const int s = h->step_counter & (IM_SLOTS - 1);
    IM_CUDA(cudaStreamSynchronize(h->stream));
    if (h->grow_max_bytes > 0) note_slots(h, false);
    for (int i = 0; i < IM_SLOTS; ++i) h->slot_busy[i] = 0;
    if (profiler().enabled) profiler().collect();
    const LioOut& o = h->h_out[s];
    h->tombs_known = o.counters[IM_LC_TOMBS];
    if (state_out) std::memcpy(state_out, o.state, IM_STATE_DOUBLES * sizeof(double));
    if (iters_run) *iters_run = o.iters_run;
    if (timings && h->timed_last) {
        float a = 0, b = 0, c = 0;
        cudaEventElapsedTime(&a, h->ev[0], h->ev[3]);
        cudaEventElapsedTime(&b, h->ev[1], h->ev[2]);
        cudaEventElapsedTime(&c, h->ev[2], h->ev[3]);
        h->last_ms[0] = a; h->last_ms[1] = b; h->last_ms[2] = c;
    }
    return lio_flags_status(o.counters[IM_LC_ERR]);
}

int immesh_lio_step(immesh_lio_t* h, const float* body, int n, double dt, double cov_gyr, double cov_acc, double* state_out, int* iters_run) {
    int rc = lio_enqueue(h, body, n, 0, dt, cov_gyr, cov_acc, false, IMMESH_FEED_KIND_STEP);
    return rc ? rc : lio_wait_impl(h, state_out, iters_run, true);
}
int immesh_lio_step_dev(immesh_lio_t* h, const float* d_body, int n, double dt, double cov_gyr, double cov_acc, double* state_out, int* iters_run) {
    int rc = lio_enqueue(h, d_body, n, 1, dt, cov_gyr, cov_acc, false, IMMESH_FEED_KIND_STEP_DEV);
    return rc ? rc : lio_wait_impl(h, state_out, iters_run, true);
}
int immesh_lio_step_async(immesh_lio_t* h, const float* body, int n, int on_device, double dt, double cov_gyr, double cov_acc) {
    return lio_enqueue(h, body, n, on_device, dt, cov_gyr, cov_acc, true, IMMESH_FEED_KIND_STEP_ASYNC);
}
// the scan AND its point count are device resident (e.g. produced by the device front-end): n is read at execution time
int immesh_lio_step_async_dev_n(immesh_lio_t* h, const float* d_body_xyz, int n_max, const int* d_n, double dt, double cov_gyr, double cov_acc) {
    if (!h || !d_n || n_max < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    h->next_n_dev = d_n;
    return lio_enqueue(h, d_body_xyz, n_max, 1, dt, cov_gyr, cov_acc, true, IMMESH_FEED_KIND_STEP_ASYNC_DEV_N);
}
// voxel_map_init queued like a pipelined step (internal: the first scan after the IMU initialisation, immesh_lio_step_async_imu): the
// build kernels of immesh_voxelmap_build on a device-resident full scan, behind the staging-slot protocol, without a host wait.
// d_n != null: the count is read on the device (n its upper bound; *d_n == 0 builds nothing), and the scan feed records nothing -- the
// depth IMU chain records its frame once, behind its step.
static int build_async_dev(immesh_lio_t* h, const float* d_body_xyz, int n, const int* d_n) {
    if (!h || !d_body_xyz || n < 1) return im_fail(IMMESH_E_INVALID, "bad argument");
    const immesh_lio::FeedNext nx = h->feed_next;   // the IMU chain's branch 2 (recorded with its header and state)
    h->feed_next = immesh_lio::FeedNext();
    if (n > h->max_scan) return im_fail(IMMESH_E_CAPACITY, "scan larger than max_scan_points");
    const bool record = h->feed.on && !d_n;
    int grc = lio_growth_check(h, n);
    if (grc == IMMESH_OK) grc = markers_fit(h);
    if (grc) return grc;
    const int s = (++h->step_counter) & (IM_SLOTS - 1);
    if (h->slot_busy[s]) {
        const auto t0 = std::chrono::steady_clock::now();
        IM_CUDA(cudaEventSynchronize(h->ev_slot[s]));
        h->host_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        h->slot_busy[s] = 0;
    }
    ++h->scan_counter;
    ++h->map_steps;
    h->next_n_dev = d_n;
    int rc = upload_scan(h, d_body_xyz, n, 1, s);
    // d_n: the depth IMU chain, whose step follows in the same call and takes this scan index again -- one pose-ring slot per call, so
    // that a mesh frame still reading the pose of up to 7 calls ago keeps it
    if (d_n) --h->scan_counter;
    if (rc) return rc;
    if (h->lm_on) launch_local_map(h);   // places the box at the building scan's pose
    launch_grow(h, 1);
    h->scan_rows = 0;   // the reference publishes no effect cloud after voxel_map_init
    if (record) {
        rc = feed_stage(h, nx, IMMESH_FEED_KIND_IMU, 2, false);
        if (rc) return rc;
        launch_feed(h, false, true);   // voxel_map_init is followed by pubPlaneMap (:1899-1900)
    }
    IM_CUDA(cudaGetLastError());
    if (record) {
        rc = feed_commit(h);
        if (rc) return rc;
    }
    IM_CUDA(cudaMemcpyAsync(h->h_out + s, &h->d_ctrl->out, sizeof(LioOut), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaEventRecord(h->ev_slot[s], h->stream));
    h->slot_busy[s] = 1;
    h->slot_step[s] = h->map_steps;
    h->timed_last = 0;
    if (!d_n) h->pose_pub_idx = h->scan_counter;
    return IMMESH_OK;
}
int immesh_voxelmap_build_async_dev(immesh_lio_t* h, const float* d_body_xyz, int n) { return build_async_dev(h, d_body_xyz, n, nullptr); }
int immesh_voxelmap_build_async_dev_n(immesh_lio_t* h, const float* d_body_xyz, int n_max, const int* d_n) {
    if (!d_n) return im_fail(IMMESH_E_INVALID, "bad argument");
    return build_async_dev(h, d_body_xyz, n_max, d_n);
}
int immesh_lio_wait(immesh_lio_t* h, double* state_out, int* iters_run) { return lio_wait_impl(h, state_out, iters_run, false); }
// internal (immesh_lio_step_async_imu, branch 1): record the scan in the feed, header and state only, behind the work queued for it
int immesh_lio_feed_record_state(immesh_lio_t* h, int kind, int branch) {
    if (!h || !h->feed.on) return IMMESH_OK;
    const int rc = feed_stage(h, immesh_lio::FeedNext(), kind, branch, false);
    if (rc) return rc;
    launch_feed(h, false, false);   // the reference continues before pubPlaneMap
    IM_CUDA(cudaGetLastError());
    return feed_commit(h);
}

int immesh_lio_feed_enable(immesh_lio_t* h, const immesh_lio_feed_config* c) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_enable: the scan feed runs on a single GPU: the handle is sharded");
    if (c && (c->max_scans < 1 || c->max_scans > (1LL << 24) || c->max_rows < 0 || c->max_rows > (1LL << 32) || (c->effect != 0 && c->effect != 1) ||
              c->registered < 0 || c->registered > 2 || c->point_skip < 1 || ((c->effect || c->registered) && c->max_rows < 1)))
        return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_enable: needs max_scans in [1, 2^24], max_rows in [0, 2^32] (>= 1 with rows), effect 0 or 1, "
                                         "registered 0, 1 or 2 and point_skip >= 1");
    IM_CUDA(im_stage_reset(h, [h] { feed_free(h); }));
    if (!c) return IMMESH_OK;
    immesh_lio::Feed& f = h->feed;
    f.max_scans = c->max_scans;
    f.max_rows = c->max_rows;
    f.effect = c->effect;
    f.registered = c->registered;
    f.skip = c->point_skip;
    f.nb = (h->max_scan + SPUB_THREADS - 1) / SPUB_THREADS;
    if (f.nb < 1) f.nb = 1;
    auto fail = [&](cudaError_t e) { feed_free(h); cudaGetLastError(); return immesh::im_fail_cuda(e, __FILE__, __LINE__); };
    cudaError_t e;
    if ((e = f.dev_mem.alloc(&f.dev, 1, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.hdr, (size_t)f.max_scans * IMMESH_LIO_FEED_HDR, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.states, (size_t)f.max_scans * IM_STATE_DOUBLES, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.rows, (size_t)std::max<long long>(f.max_rows, 1))) != cudaSuccess) return fail(e);
    if (f.effect && (e = f.dev_mem.alloc(&f.idx, (size_t)f.max_rows)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.tiles, (size_t)f.nb + 1, 0)) != cudaSuccess) return fail(e);
    if ((e = f.pinned.alloc(&f.h_dyn, IM_FEED_DYN_RING)) != cudaSuccess) return fail(e);
    if ((e = f.pinned.alloc(&f.h_done, 1)) != cudaSuccess) return fail(e);
    *f.h_done = 0;
    std::memset(f.h_dyn, 0, IM_FEED_DYN_RING * sizeof(FeedDyn));
    if ((e = cudaHostGetDevicePointer((void**)&f.d_done, f.h_done, 0)) != cudaSuccess) return fail(e);
    if ((e = cudaStreamCreateWithFlags(&f.stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e);
    if ((e = cudaEventCreateWithFlags(&f.ev, cudaEventDisableTiming)) != cudaSuccess) return fail(e);
    if ((e = cudaEventRecord(f.ev, h->stream)) != cudaSuccess) return fail(e);
    if ((e = cudaStreamSynchronize(h->stream)) != cudaSuccess) return fail(e);
    f.on = 1;
    return IMMESH_OK;
}

// the common part of the two reads: the wait, counts[2..3], then feed_read of `rings`, its copies and the marks at `started` on the
// feed's stream (never the handle's)
static int lio_feed_read(immesh_lio* h, const FeedRings& rings, const long long* started, int64_t since, int wait, int64_t* scans, double* states,
                         int cap_scans, void* rows, void* second, int64_t cap_rows, int64_t* counts) {
    immesh_lio::Feed& f = h->feed;
    if (wait) IM_CUDA(cudaEventSynchronize(f.ev));   // the newest queued scan's record, nothing else
    const long long fin = *(volatile long long*)f.h_done;
    counts[2] = fin;
    counts[3] = f.queued;
    auto copy = [&f](void* dst, const void* src, size_t bytes) {
        IM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, f.stream));
        return IMMESH_OK;
    };
    auto marks = [&](long long* m) {
        IM_CUDA(cudaMemcpyAsync(m, started, 2 * sizeof(long long), cudaMemcpyDeviceToHost, f.stream));
        IM_CUDA(cudaStreamSynchronize(f.stream));
        return IMMESH_OK;
    };
    return feed_read(rings, since, fin, scans, states, cap_scans, rows, second, cap_rows, counts, copy, marks);
}
int immesh_lio_feed(immesh_lio_t* h, int64_t since, int wait, int64_t* scans, double* states, int cap_scans, float* rows, int32_t* row_index, int64_t cap_rows,
                    int64_t* counts) {
    if (!h || !counts || cap_scans < 0 || cap_rows < 0 || (cap_scans > 0 && !scans)) return im_fail(IMMESH_E_INVALID, "bad argument");
    for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed: the handle is sharded");
    immesh_lio::Feed& f = h->feed;
    if (!f.on) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed: the scan feed is not enabled (immesh_lio_feed_enable)");
    if (since < 0 || since > f.queued) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed: since_scan must be in [0, newest queued scan]");
    const FeedRings rings{f.max_scans, f.max_rows, f.hdr, f.states, f.rows, f.idx};
    const int rc = lio_feed_read(h, rings, &f.dev->started, since, wait, scans, states, cap_scans, rows, row_index, cap_rows, counts);
    if (rc == IMMESH_E_RANGE) return im_fail(rc, "immesh_lio_feed: scans of the range left the rings or were overwritten while they were read; read on from counts[2]");
    if (rc == IMMESH_E_CAPACITY) return im_fail(rc, "immesh_lio_feed: more scans or rows than the caps (counts holds them)");
    return rc;
}
int immesh_lio_feed_markers_enable(immesh_lio_t* h, int64_t max_rows) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers_enable: the handle is sharded");
    immesh_lio::Feed& f = h->feed;
    if (!f.on) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers_enable: the scan feed is not enabled (immesh_lio_feed_enable)");
    if (max_rows < 0 || max_rows > (1LL << 32)) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers_enable: max_rows must be in [0, 2^32] (0: off)");
    IM_CUDA(im_stage_reset(h, [h] { markers_free(h); }));
    if (max_rows == 0) return IMMESH_OK;
    auto fail = [&](cudaError_t e) { markers_free(h); cudaGetLastError(); return immesh::im_fail_cuda(e, __FILE__, __LINE__); };
    cudaError_t e;
    if ((e = f.mk_mem.alloc(&f.mk_dev, 1, 0)) != cudaSuccess) return fail(e);
    if ((e = f.mk_mem.alloc(&f.mk_hdr, (size_t)f.max_scans * IMMESH_LIO_FEED_MARKER_HDR, 0)) != cudaSuccess) return fail(e);
    if ((e = f.mk_mem.alloc(&f.mk_ring, (size_t)max_rows * IMMESH_PLANE_MARKER_COLS)) != cudaSuccess) return fail(e);
    f.mk_rows = max_rows;
    const int rc = markers_fit(h);
    if (rc) { markers_free(h); return rc; }
    return IMMESH_OK;
}

int immesh_lio_feed_markers(immesh_lio_t* h, int64_t since, int wait, int64_t* scans, int cap_scans, double* rows, int64_t cap_rows, int64_t* counts) {
    if (!h || !counts || cap_scans < 0 || cap_rows < 0 || (cap_scans > 0 && !scans)) return im_fail(IMMESH_E_INVALID, "bad argument");
    for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers: the handle is sharded");
    immesh_lio::Feed& f = h->feed;
    if (!f.on || f.mk_rows == 0) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers: the plane-map markers are not enabled (immesh_lio_feed_markers_enable)");
    if (since < 0 || since > f.queued) return im_fail(IMMESH_E_INVALID, "immesh_lio_feed_markers: since_scan must be in [0, newest queued scan]");
    const FeedRings rings = marker_rings(f.max_scans, f.mk_rows, f.mk_hdr, f.mk_ring);
    const int rc = lio_feed_read(h, rings, &f.mk_dev->started, since, wait, scans, nullptr, cap_scans, rows, nullptr, cap_rows, counts);
    if (rc == IMMESH_E_RANGE)
        return im_fail(rc, "immesh_lio_feed_markers: records of the range left the rings, were overwritten while they were read, or predate the enable; read on from counts[2]");
    if (rc == IMMESH_E_CAPACITY) return im_fail(rc, "immesh_lio_feed_markers: more scans or rows than the caps (counts holds them)");
    return rc;
}
// queue a write of `bytes` bytes over a caller-provided device buffer on the localization stream (benchmark L2 flush)
int immesh_lio_enqueue_memset(immesh_lio_t* h, void* d_buf, size_t bytes) {
    if (!h || !d_buf) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaMemsetAsync(d_buf, 0, bytes, h->stream));
    return IMMESH_OK;
}

// work counters of the last step (roofline byte model): [n, touched root voxels are not kept, plane refits, points read by the refits]
int immesh_lio_work_stats(immesh_lio_t* h, int64_t* out /*[4]*/) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const LioOut& o = h->h_out[h->step_counter & (IM_SLOTS - 1)];
    out[0] = h->last_n; out[1] = o.counters[IM_LC_ROOTS]; out[2] = o.counters[IM_LC_REFITS]; out[3] = o.counters[IM_LC_REFIT_POINTS];
    return IMMESH_OK;
}
int immesh_lio_last_timing(immesh_lio_t* h, double* ms) {
    if (!h || !ms) return im_fail(IMMESH_E_INVALID, "null argument");
    ms[0] = h->last_ms[0]; ms[1] = h->last_ms[1]; ms[2] = h->last_ms[2];
    return IMMESH_OK;
}

int immesh_residual_build(immesh_lio_t* h, const float* body, int n, int* index_layer, double* ptpl, int cap, int* n_out) {
    if (!h || !n_out) return im_fail(IMMESH_E_INVALID, "null argument");
    int rc = upload_scan(h, body, n);
    if (rc) return rc;
    scan_rows_overwritten(h, "immesh_residual_build");
    if (!h->d_ptpl) IM_CUDA(h->dev.alloc(&h->d_ptpl, (size_t)h->max_scan * 31));
    IM_LAUNCH(k_reset_scan, 2, 256, 0, h->stream, h->sb, h->d_ctrl, 0);
    *n_out = 0;
    if (n == 0) return IMMESH_OK;
    IM_LAUNCH(k_prepare, grid_fixed(h, 128), 128, 0, h->stream, h->P, h->sb);
    IM_LAUNCH(k_residual, grid_fixed(h, RES_THREADS, 4), RES_THREADS, 0, h->stream, h->map, h->P, h->sb, h->d_ctrl, 0, 0);
    IM_LAUNCH(k_gather_ptpl, grid_fixed(h, 128), 128, 0, h->stream, h->map, h->sb, n, h->d_ptpl);
    IM_CUDA(cudaGetLastError());
    std::vector<int> node(n), layer(n);
    std::vector<double> vals((size_t)n * 31);
    IM_CUDA(cudaMemcpyAsync(node.data(), h->sb.match_node, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(layer.data(), h->sb.match_layer, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(vals.data(), h->d_ptpl, (size_t)n * 31 * 8, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int m = 0;
    for (int i = 0; i < n; ++i) {
        if (node[i] < 0) continue;
        if (m < cap) {
            if (index_layer) { index_layer[2 * m] = i; index_layer[2 * m + 1] = layer[i]; }
            if (ptpl) std::memcpy(ptpl + (size_t)m * 31, vals.data() + (size_t)i * 31, 31 * 8);
        }
        ++m;
    }
    *n_out = m;
    return check_flags(h);
}

static void var9_to_6(const double* v9, double* v6) {  // upper triangle of the caller's (symmetric) 3x3
    v6[0] = v9[0]; v6[1] = v9[1]; v6[2] = v9[2]; v6[3] = v9[4]; v6[4] = v9[5]; v6[5] = v9[8];
}
static int upload_pv(immesh_lio* h, const double* pts_world, const double* var9, int n) {
    if ((!pts_world || !var9) && n > 0) return im_fail(IMMESH_E_INVALID, "null argument");
    if (n < 0 || n > h->max_scan) return im_fail(IMMESH_E_CAPACITY, "too many points");
    std::vector<float> pw((size_t)n * 3);
    std::vector<double> v6((size_t)n * 6);
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < 3; ++j) pw[(size_t)i * 3 + j] = (float)pts_world[(size_t)i * 3 + j];  // already float-valued in the reference
        var9_to_6(var9 + (size_t)i * 9, v6.data() + (size_t)i * 6);
    }
    IM_CUDA(cudaMemcpyAsync(h->sb.pw, pw.data(), pw.size() * 4, cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaMemcpyAsync(h->sb.var, v6.data(), v6.size() * 8, cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    return push_dyn(h, n);
}
int immesh_voxelmap_build_pv(immesh_lio_t* h, const double* pts_world, const double* var9, int n) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    int rc = lio_growth_check(h, n);
    if (rc) return rc;
    rc = upload_pv(h, pts_world, var9, n);
    if (rc) return rc;
    scan_rows_overwritten(h, "immesh_voxelmap_build_pv");
    ++h->map_steps;
    launch_grow(h, 3);
    IM_CUDA(cudaGetLastError());
    return check_flags(h);
}
int immesh_voxelmap_update_pv(immesh_lio_t* h, const double* pts_world, const double* var9, int n) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    int rc = lio_growth_check(h, n);
    if (rc) return rc;
    rc = upload_pv(h, pts_world, var9, n);
    if (rc) return rc;
    scan_rows_overwritten(h, "immesh_voxelmap_update_pv");
    ++h->map_steps;
    launch_grow(h, 2);
    IM_CUDA(cudaGetLastError());
    return check_flags(h);
}
int immesh_residual_build_pv(immesh_lio_t* h, const double* pts_body, const double* pts_world, const double* var9, int n, int* index_layer,
                             double* ptpl, int cap, int* n_out) {
    if (!h || !n_out || ((!pts_body || !pts_world || !var9) && n > 0)) return im_fail(IMMESH_E_INVALID, "null argument");
    if (n < 0 || n > h->max_scan) return im_fail(IMMESH_E_CAPACITY, "too many points");
    *n_out = 0;
    if (n == 0) return IMMESH_OK;
    scan_rows_overwritten(h, "immesh_residual_build_pv");
    std::vector<double> v6((size_t)n * 6);
    for (int i = 0; i < n; ++i) var9_to_6(var9 + (size_t)i * 9, v6.data() + (size_t)i * 6);
    IM_CUDA(cudaMemcpyAsync(h->sb.var, v6.data(), v6.size() * 8, cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaMemcpyAsync(h->sb.p_imu, pts_world, (size_t)n * 24, cudaMemcpyHostToDevice, h->stream));  // p_imu doubles as scratch for the world points
    IM_LAUNCH(k_match_pv, grid_fixed(h, 128), 128, 0, h->stream, h->map, h->P, h->sb, h->sb.p_imu, n);
    IM_CUDA(cudaGetLastError());
    std::vector<int> node(n), layer(n);
    IM_CUDA(cudaMemcpyAsync(node.data(), h->sb.match_node, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(layer.data(), h->sb.match_layer, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int m = 0, nn = 0;
    for (int i = 0; i < n; ++i) nn = node[i] > nn ? node[i] : nn;
    std::vector<PlaneRec> planes;
    // fetch only the matched plane records
    std::vector<int> uniq;
    for (int i = 0; i < n; ++i) if (node[i] >= 0) uniq.push_back(node[i]);
    std::sort(uniq.begin(), uniq.end());
    uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
    planes.resize(uniq.size());
    for (size_t u = 0; u < uniq.size(); ++u)
        IM_CUDA(cudaMemcpyAsync(&planes[u], h->map.planes + uniq[u], sizeof(PlaneRec), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        if (node[i] < 0) continue;
        if (m < cap) {
            const PlaneRec& pl = planes[std::lower_bound(uniq.begin(), uniq.end(), node[i]) - uniq.begin()];
            if (index_layer) { index_layer[2 * m] = i; index_layer[2 * m + 1] = layer[i]; }
            if (ptpl) {
                double* o = ptpl + (size_t)m * 31;
                for (int j = 0; j < 3; ++j) { o[j] = pts_body[(size_t)i * 3 + j]; o[3 + j] = pl.normal[j]; o[6 + j] = pl.center[j]; }
                o[9] = (double)pl.d;
                for (int j = 0; j < 21; ++j) o[10 + j] = pl.pv[j];
            }
        }
        ++m;
    }
    *n_out = m;
    return check_flags(h);
}

int immesh_lio_iter_stats(immesh_lio_t* h, int it, double* out) {
    if (!h || !out || it < 0 || it >= IM_MAX_ITER) return im_fail(IMMESH_E_INVALID, "bad argument");
    IterStats s;
    IM_CUDA(cudaMemcpyAsync(&s, &h->d_ctrl->stats[it], sizeof(IterStats), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(out, s.HTH, 36 * 8);
    std::memcpy(out + 36, s.HTz, 6 * 8);
    out[42] = s.n_match; out[43] = s.total_residual;
    std::memcpy(out + 44, s.solution, 18 * 8);
    out[62] = s.converged;
    return IMMESH_OK;
}

int immesh_lio_matches(immesh_lio_t* h, int* plane_layer, int n) {
    if (!h || !plane_layer || n > h->max_scan) return im_fail(IMMESH_E_INVALID, "bad argument");
    std::vector<int> node(n), layer(n);
    IM_CUDA(cudaMemcpyAsync(node.data(), h->sb.match_node, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(layer.data(), h->sb.match_layer, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) plane_layer[i] = node[i] >= 0 ? layer[i] : -1;
    return IMMESH_OK;
}

int immesh_lio_match_nodes(immesh_lio_t* h, int* node, int n) {
    if (!h || !node || n > h->max_scan) return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaMemcpyAsync(node, h->sb.match_node, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    return IMMESH_OK;
}

int64_t immesh_voxelmap_dump(immesh_lio_t* h, double* rows, int64_t cap_rows) {
    if (!h) return -1;
    int c[IM_LC_SIZE];
    if (lio_read_counters(h, c) != cudaSuccess) return -1;
    const int nn = c[IM_LC_NODES] < h->max_nodes ? c[IM_LC_NODES] : h->max_nodes;
    std::vector<unsigned long long> keys(h->cap);
    std::vector<int> roots(h->cap);
    std::vector<NodeRec> nodes(nn > 0 ? nn : 1);
    std::vector<PlaneRec> planes(nn > 0 ? nn : 1);
    cudaMemcpy(keys.data(), h->map.keys, h->cap * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(roots.data(), h->map.root_node, h->cap * 4, cudaMemcpyDeviceToHost);
    if (nn > 0) {
        cudaMemcpy(nodes.data(), h->map.nodes, (size_t)nn * sizeof(NodeRec), cudaMemcpyDeviceToHost);
        cudaMemcpy(planes.data(), h->map.planes, (size_t)nn * sizeof(PlaneRec), cudaMemcpyDeviceToHost);
    }
    return dump_voxelmap(keys.data(), roots.data(), h->cap, nodes.data(), planes.data(), rows, cap_rows);
}

int immesh_voxelmap_plane_markers(immesh_lio_t* h, double* rows, int cap, int* n_out, int64_t* counts) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows)) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    if (counts) for (int k = 0; k < 5; ++k) counts[k] = 0;
    IM_CUDA(cudaStreamSynchronize(h->stream));   // everything queued on the handle, the pipelined steps included
    IM_CUDA(cudaMemcpyAsync(h->h_ints + IM_HINT_PUB, h->map.pub_n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    const int n = h->h_ints[IM_HINT_PUB];
    if (counts) counts[4] = n;
    if (n == 0) return IMMESH_OK;
    const int nb = (n + VG_TILE - 1) / VG_TILE;
    const size_t need = (size_t)6 * n + (size_t)256 * nb + 8;
    IM_CUDA(h->scratch.regrow(&h->d_pub_scratch, &h->pub_scratch_ints, need));
    unsigned int* ku[2] = {(unsigned int*)h->d_pub_scratch, (unsigned int*)h->d_pub_scratch + n};
    unsigned int* vu[2] = {(unsigned int*)h->d_pub_scratch + 2 * (size_t)n, (unsigned int*)h->d_pub_scratch + 3 * (size_t)n};
    int* slots = h->d_pub_scratch + 4 * (size_t)n;
    int* cnt = h->d_pub_scratch + 5 * (size_t)n;
    int* hist = h->d_pub_scratch + 6 * (size_t)n;
    int* misc = hist + (size_t)256 * nb;   // [0] rows in all, [1..4] the reference's counters
    cudaStream_t st = h->stream;
    const int g = std::min((n + PUB_THREADS - 1) / PUB_THREADS, h->n_sm * 16);
    IM_CUDA(cudaMemsetAsync(misc, 0, 8 * sizeof(int), st));
    int cur = 0;
    for (int half = 0; half < 2; ++half) {
        IM_LAUNCH(k_pub_keys, g, PUB_THREADS, 0, st, h->map, n, (const int*)nullptr, half, half ? (const unsigned int*)vu[cur] : (const unsigned int*)nullptr,
                  ku[cur ^ half], vu[cur ^ half]);
        cur = rs_sort_passes(st, ku, vu, cur ^ half, n, 4, hist);
    }
    IM_LAUNCH(k_pub_count, g, PUB_THREADS, 0, st, h->map, n, (const int*)nullptr, (const unsigned int*)vu[cur], slots, cnt, misc + 1);
    IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, cnt, n, misc);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_ints + IM_HINT_PUB, misc, 5 * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int total = h->h_ints[IM_HINT_PUB];
    *n_out = total;
    if (counts) for (int k = 0; k < 4; ++k) counts[k] = h->h_ints[IM_HINT_PUB + 1 + k];
    if (total > cap) return im_fail(IMMESH_E_CAPACITY, "plane markers: more rows than cap (*n_out holds the number needed; nothing was consumed)");
    // at least one row, so that k_pub_emit never gets a null pointer
    IM_CUDA(h->scratch.regrow(&h->d_pub_rows, &h->pub_rows_doubles, std::max<size_t>((size_t)total, 1) * IM_PUB_COLS, (size_t)1024 * IM_PUB_COLS));
    IM_CUDA(cudaMemsetAsync(h->map.pub_n, 0, sizeof(int), st));
    IM_LAUNCH(k_pub_emit, g, PUB_THREADS, 0, st, h->map, n, (const int*)slots, (const int*)cnt, h->d_pub_rows, (const LioMarkDev*)nullptr, 0LL);
    IM_CUDA(cudaGetLastError());
    if (total > 0) IM_CUDA(cudaMemcpyAsync(rows, h->d_pub_rows, (size_t)total * IM_PUB_COLS * sizeof(double), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    return IMMESH_OK;
}

int immesh_lio_effect_cloud(immesh_lio_t* h, float* rows, int32_t* scan_index, int cap, int* n_out) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows)) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    int rc = scan_rows_status(h, "immesh_lio_effect_cloud");
    if (rc) return rc;
    IM_CUDA(cudaStreamSynchronize(h->stream));   // everything queued on the handle, the pipelined steps included
    const int n_max = h->dyn_last.n;              // the scan's count, or its bound when the count is device resident
    if (h->scan_rows == 0 || n_max <= 0) return IMMESH_OK;
    const int nb = (n_max + SPUB_THREADS - 1) / SPUB_THREADS;
    IM_CUDA(h->scratch.regrow(&h->d_spub_tiles, &h->spub_tiles_cap, (size_t)nb + 1, 1024));
    int* tiles = h->d_spub_tiles;
    cudaStream_t st = h->stream;
    IM_LAUNCH(k_eff_count, nb, SPUB_THREADS, 0, st, h->sb, tiles);
    IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, tiles, nb, tiles + nb);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_ints + IM_HINT_PUB, tiles + nb, sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int total = h->h_ints[IM_HINT_PUB];
    *n_out = total;
    if (total > cap) return im_fail(IMMESH_E_CAPACITY, "effect cloud: more rows than cap (*n_out holds the number needed)");
    if (total == 0) return IMMESH_OK;
    IM_CUDA(h->scratch.regrow(&h->d_spub_rows, &h->spub_rows_cap, (size_t)total, 1024));
    if (scan_index) IM_CUDA(h->scratch.regrow(&h->d_spub_idx, &h->spub_idx_cap, (size_t)total, 1024));
    IM_LAUNCH(k_eff_emit, nb, SPUB_THREADS, 0, st, h->P, h->sb, (const LioCtrl*)h->d_ctrl, (const int*)tiles, h->d_spub_rows, scan_index ? h->d_spub_idx : (int*)nullptr,
              (const LioFeedDev*)nullptr, 0LL);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(rows, h->d_spub_rows, (size_t)total * sizeof(float4), cudaMemcpyDeviceToHost, st));
    if (scan_index) IM_CUDA(cudaMemcpyAsync(scan_index, h->d_spub_idx, (size_t)total * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    return IMMESH_OK;
}

// inten (device, or null): the points' intensity as a separate array (immesh_lio_frontend_cloud)
static int registered_rows(immesh_lio_t* h, const float* pts, const float* inten, int n, int stride, int intensity_col, int on_device, int point_skip, float* rows,
                           int cap, int* n_out) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (point_skip <= 0) return im_fail(IMMESH_E_INVALID, "registered cloud: point_skip must be positive");
    if (pts && (n < 0 || stride < 3 || intensity_col >= stride)) return im_fail(IMMESH_E_INVALID, "registered cloud: needs n >= 0, stride >= 3 and intensity_col < stride");
    *n_out = 0;
    cudaStream_t st = h->stream;
    if (!pts) {
        const int rc = scan_rows_status(h, "immesh_lio_registered_cloud");
        if (rc) return rc;
        if (h->scan_rows == 0) return im_fail(IMMESH_E_INVALID, "immesh_lio_registered_cloud: pts == NULL publishes the scan of the last IESKF run, and there is none");
    }
    IM_CUDA(cudaStreamSynchronize(st));
    if (!pts) {
        IM_CUDA(h->scratch.regrow(&h->d_spub_tiles, &h->spub_tiles_cap, 1, 1024));
        IM_LAUNCH(k_scan_n, 1, 1, 0, st, h->sb, h->d_spub_tiles);
        IM_CUDA(cudaGetLastError());
        IM_CUDA(cudaMemcpyAsync(h->h_ints + IM_HINT_PUB, h->d_spub_tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
        n = h->h_ints[IM_HINT_PUB];
    }
    const int m = n > 0 ? (n - 1) / point_skip + 1 : 0;
    *n_out = m;
    if (m > cap) return im_fail(IMMESH_E_CAPACITY, "registered cloud: more rows than cap (*n_out holds the number needed)");
    if (m == 0) return IMMESH_OK;
    const float* src = pts;
    if (pts && !on_device) {
        const size_t floats = ((size_t)(m - 1) * point_skip + 1) * stride;   // up to the last point published
        IM_CUDA(h->scratch.regrow(&h->d_spub_in, &h->spub_in_cap, floats, 1024));
        IM_CUDA(cudaMemcpyAsync(h->d_spub_in, pts, floats * sizeof(float), cudaMemcpyHostToDevice, st));
        src = h->d_spub_in;
    }
    IM_CUDA(h->scratch.regrow(&h->d_spub_rows, &h->spub_rows_cap, (size_t)m, 1024));
    const int g = std::min((m + SPUB_THREADS - 1) / SPUB_THREADS, h->n_sm * 16);
    IM_LAUNCH(k_reg_gather, g, SPUB_THREADS, 0, st, h->P, h->sb, (const LioCtrl*)h->d_ctrl, src, n, stride, intensity_col, point_skip, h->d_spub_rows, inten,
              (const LioFeedDev*)nullptr, 0LL);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(rows, h->d_spub_rows, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    return IMMESH_OK;
}
int immesh_lio_registered_cloud(immesh_lio_t* h, const float* pts, int n, int stride, int intensity_col, int on_device, int point_skip, float* rows, int cap, int* n_out) {
    return registered_rows(h, pts, nullptr, n, stride, intensity_col, on_device, point_skip, rows, cap, n_out);
}
// internal (immesh_lio_frontend_cloud): rows of the packed device cloud d_xyz ([n][3]; null: the localised scan) with intensity d_inten
int immesh_lio_registered_cloud_sep(immesh_lio_t* h, const float* d_xyz, const float* d_inten, int n, int point_skip, float* rows, int cap, int* n_out) {
    return registered_rows(h, d_xyz, d_inten, n, 3, -1, 1, point_skip, rows, cap, n_out);
}

int immesh_voxelmap_counts(immesh_lio_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    int c[IM_LC_SIZE];
    IM_CUDA(lio_read_counters(h, c));
    out[0] = c[IM_LC_ROOTS]; out[1] = c[IM_LC_NODES]; out[2] = c[IM_LC_CHUNK_BUMP]; out[3] = c[IM_LC_ERR];
    return IMMESH_OK;
}

int immesh_lio_capacity(immesh_lio_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    IM_CUDA(lio_read_counters(h, h->h_ints));
    const int* c = h->h_ints;
    out[0] = (int64_t)h->cap; out[1] = c[IM_LC_ROOTS];
    out[2] = h->max_nodes; out[3] = c[IM_LC_NODES];
    out[4] = h->max_chunks; out[5] = (int64_t)c[IM_LC_CHUNK_BUMP] - std::max(c[IM_LC_AVAIL_TOP], 0);
    out[6] = (int64_t)h->dev.bytes(); out[7] = h->growths;
    return IMMESH_OK;
}
int immesh_lio_reserve(immesh_lio_t* h, int64_t root_slots, int64_t nodes, int64_t chunks) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_reserve: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    long long cap = (long long)h->cap;
    if (root_slots > IM_POOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "root hash: more than 2^30 slots (32-bit slot ids)");
    while (cap < root_slots) cap *= 2;
    const int rc = lio_grow(h, cap, std::max<long long>(nodes, h->max_nodes), std::max<long long>(chunks, h->max_chunks));
    if (rc == IMMESH_OK) return rc;
    return im_fail(rc, (std::string("immesh_lio_reserve: ") + immesh::last_error_storage()).c_str());
}
int immesh_lio_set_growth(immesh_lio_t* h, int64_t max_bytes) {
    if (!h || max_bytes < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (max_bytes > 0 && h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_set_growth: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    if (max_bytes > 0 && h->grow_max_bytes <= 0) {   // growth starts from the map as it is now
        IM_CUDA(cudaStreamSynchronize(h->stream));
        IM_CUDA(lio_read_counters(h, h->h_ints));
        note_counters(h, h->h_ints, ++h->map_steps);   // the map as it is now, under a step number of its own
    }
    h->grow_max_bytes = max_bytes;
    return IMMESH_OK;
}

// ---- local map (local_map.cuh)
// the node free stack, allocated once: from then on alloc_node pops it first (the captured launch sequence holds the map: dropped)
static int lio_node_free_alloc(immesh_lio* h) {
    if (h->map.node_free) return IMMESH_OK;
    IM_CUDA(h->dev.alloc(&h->map.node_free, (size_t)h->max_nodes));
    h->graph.destroy();
    return IMMESH_OK;
}
int immesh_lio_local_map(immesh_lio_t* h, double cube_len, float det_range, float mov_threshold) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_local_map: the local map runs on a single GPU: the handle is sharded");
    const bool on = cube_len != 0.0;
    if (on && !(std::isfinite(cube_len) && cube_len > 0 && std::isfinite(det_range) && det_range > 0 && std::isfinite(mov_threshold) && mov_threshold > 0))
        return im_fail(IMMESH_E_INVALID, "immesh_lio_local_map: cube_len, det_range and mov_threshold must be finite and positive (cube_len = 0 turns the local map off)");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    if (on) {
        const int rc = lio_node_free_alloc(h);
        if (rc) return rc;
    }
    LocalMapCtrl L;
    IM_CUDA(cudaMemcpy(&L, &h->d_ctrl->lm, sizeof(L), cudaMemcpyDeviceToHost));
    L.cube_len = on ? cube_len : 0.0;
    L.det_range = on ? det_range : 0.f;
    L.mov_threshold = on ? mov_threshold : 0.f;
    L.on = on ? 1 : 0;
    L.placed = 0;   // the box is placed at the next evaluation
    L.n_rm = 0;
    IM_CUDA(cudaMemcpy(&h->d_ctrl->lm, &L, sizeof(L), cudaMemcpyHostToDevice));
    if (h->lm_on != (on ? 1 : 0)) h->graph.destroy();   // the launch sequence changes
    h->lm_on = on ? 1 : 0;
    return IMMESH_OK;
}
int immesh_voxelmap_evict_boxes(immesh_lio_t* h, const float* boxes, int n) {
    if (!h || n < 0 || (n > 0 && !boxes)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (h->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_voxelmap_evict_boxes: the handle is sharded");
    for (int i = 0; i < 6 * n; ++i)
        if (std::isnan(boxes[i])) return im_fail(IMMESH_E_INVALID, "immesh_voxelmap_evict_boxes: a box edge is NaN");
    if (n == 0) return IMMESH_OK;
    if (!h->map.node_free) {
        IM_CUDA(cudaStreamSynchronize(h->stream));
        const int rc = lio_node_free_alloc(h);
        if (rc) return rc;
    }
    // the device copy of the boxes is reused by every call: a queued sweep must not see it freed by a regrow (drain first)
    if ((size_t)n * 6 > h->lm_boxes_cap) IM_CUDA(cudaStreamSynchronize(h->stream));
    IM_CUDA(h->scratch.regrow(&h->d_lm_boxes, &h->lm_boxes_cap, (size_t)n * 6, 64));
    // staged through a host copy of the library's own (pageable) memory: the copy from pageable memory has read its source when it
    // returns, so the caller may reuse `boxes` at once whatever memory they are in (a pinned source would still be read later)
    const std::vector<float> staged(boxes, boxes + (size_t)n * 6);
    IM_CUDA(cudaMemcpyAsync(h->d_lm_boxes, staged.data(), staged.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    launch_local_map(h, h->d_lm_boxes, n);   // queued behind the handle's steps
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}
int immesh_lio_local_map_state(immesh_lio_t* h, float* box, int64_t* stats) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    LocalMapCtrl L;
    IM_CUDA(cudaMemcpy(&L, &h->d_ctrl->lm, sizeof(L), cudaMemcpyDeviceToHost));
    int c[IM_LC_SIZE];
    IM_CUDA(lio_read_counters(h, c));
    if (box) for (int k = 0; k < 6; ++k) box[k] = L.box[k];
    if (stats) {
        stats[0] = L.placed; stats[1] = (int64_t)L.moves; stats[2] = (int64_t)L.roots; stats[3] = (int64_t)L.nodes; stats[4] = (int64_t)L.chunks;
        stats[5] = c[IM_LC_TOMBS]; stats[6] = h->lm_purges; stats[7] = std::max(c[IM_LC_NODE_FREE], 0);
    }
    return IMMESH_OK;
}

}  // extern "C"
