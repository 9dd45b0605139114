// immesh_b200 -- IMU step in front of the hot path (SURVEY 8f-2) on the device: ImuProcess::UndistortPcl
// (/root/reference/src/IMU_Processing.cpp:755-958), and the IMU-enabled scan loop of Voxel_mapping::service_LiDAR_update
// (ImuProcess::Process2 :960-1006 + src/voxel_mapping.cpp:1820-1905) as one queued call per scan.  The state and its covariance
// stay in the localization handle's HBM (LioCtrl::state), the time stamps the scans carry over in ImuTime; the host decides
// nothing from device data.
//   k_imu_forward   one block: thread 0 seeds the running quantities from the state (IMUpose[0]) and works out the interval plan
//                   (imu_plan) from the staged samples; then all live IMU intervals in sequence (18x18 F P F^T + Q each) and the
//                   scan-end prediction
//   k_imu_intake    (the _i entry) point records of `stride` floats -> [n][4] x y z t + [n] intensity
//   k_imu_keys      time-stamp keys (ordered-uint image of the float curvature) for the stable radix sort (radix_sort.cuh)
//   k_imu_gather    points in time order
//   k_imu_undistort thread per point: interval lookup + rigid transform into the scan-end frame (16 B in, 16 B out per point)
// The depth IMU chain (immesh_lio_step_async_depth_imu) decides its branch on the device, from the depth cloud's device count:
//   k_dimu_branch   one block: sync_packages' drop rule and carry (src/voxel_mapping_common.cpp:393-400), the batch carried + own,
//                   the branch of Process2 / service_LiDAR_update, and the counts every later kernel of the frame reads
//   k_dimu_init     branch 1: IMU_init (imu_init_batch, the host chain's code) and the init-end test, on the device
//   k_dimu_expand   the cloud as x y z t, t = 0 (l515_handler's curvature, src/preprocess.cpp:270): the stable time sort of all-equal
//                   stamps is the identity, so this is the sorted cloud
//   k_imu_forward_dn / k_imu_undistort_dn   k_imu_forward / k_imu_undistort with the counts and mean_acc_norm read on the device
// There is no CPU path.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdio>
#include <cstring>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"
#include "imu_core.cuh"

using immesh::im_fail; using immesh::ImuParams; using immesh::ImuStep; using immesh::ImuTime; using immesh::ImuInit; using immesh::DepthImu;

namespace {

#include "radix_sort.cuh"

#define IMU_FWD_THREADS 352

// pts: the scan as given (unsorted), read for its last point's stamp only
__device__ __forceinline__ void imu_forward_block(const ImuParams& P, LioCtrl* ctrl, double* run, ImuTime* tm, const double* imu, int n_imu, const float* pts, int n,
                                                  double lidar_beg_time, ImuStep* steps, double* poses) {
    __shared__ double Fx[324], T[324];
    __shared__ double s_note, s_dt;
    __shared__ int s_steps;
    if (threadIdx.x == 0) {
        const double* st = ctrl->state;
        for (int i = 0; i < 3; ++i) { run[6 + i] = st[12 + i]; run[9 + i] = st[9 + i]; }
        for (int i = 0; i < 9; ++i) run[12 + i] = st[i];
        immesh::imu_write_pose(poses, 0.0, run);   // IMUpose[0] = (0, acc_s_last, angvel_last, vel_end, pos_end, rot_end), :800
        s_steps = immesh::imu_plan(*tm, imu, n_imu, pts[4 * (size_t)(n - 1) + 3], lidar_beg_time, steps, &s_note, &s_dt);
    }
    __syncthreads();
    const int n_steps = s_steps;
    for (int k = 0; k < n_steps; ++k)
        immesh::imu_forward_step(P, ctrl->state, run, steps[k], poses + (size_t)(k + 1) * IM_POSE_DOUBLES, Fx, T, threadIdx.x, blockDim.x);
    if (threadIdx.x == 0) immesh::imu_predict_end(ctrl->state, run, s_note, s_dt);
}
__global__ void __launch_bounds__(IMU_FWD_THREADS) k_imu_forward(ImuParams P, LioCtrl* ctrl, double* run, ImuTime* tm, const double* imu, int n_imu, const float* pts, int n,
                                                                  double lidar_beg_time, ImuStep* steps, double* poses) {
    imu_forward_block(P, ctrl, run, tm, imu, n_imu, pts, n, lidar_beg_time, steps, poses);
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_keys(const float* __restrict__ pts, int n, unsigned int* keys, unsigned int* vals) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        unsigned int b = __float_as_uint(pts[4 * (size_t)i + 3]);
        if (b == 0x80000000u) b = 0u;                              // -0.0 and +0.0 compare equal in time_list
        keys[i] = (b & 0x80000000u) ? ~b : (b | 0x80000000u);     // order-preserving image of the float (time_list: x.curvature < y.curvature)
        vals[i] = (unsigned int)i;
    }
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_intake(const float* __restrict__ rec, int n, int stride, int tcol, int icol, float4* out, float* out_i) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float* r = rec + (size_t)i * stride;
        out[i] = make_float4(r[0], r[1], r[2], r[tcol]);
        out_i[i] = r[icol];
    }
}
// in_i != nullptr: the intensity follows its point through the same permutation
__global__ void __launch_bounds__(VG_THREADS) k_imu_gather(const float4* __restrict__ in, const unsigned int* __restrict__ vals, int n, float4* out,
                                                            const float* __restrict__ in_i, float* out_i) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vals[i];
        out[i] = in[v];
        if (in_i) out_i[i] = in_i[v];
    }
}
// the IMUpose count comes from the plan (ImuTime::n_pose); the dynamic shared memory is sized for the batch's upper bound
__device__ __forceinline__ void imu_undistort_block(const ImuParams& P, const LioCtrl* ctrl, const double* __restrict__ poses, const ImuTime* tm, float* pts, int n) {
    extern __shared__ double s_pose[];
    __shared__ double s_end[12];
    const int n_pose = tm->n_pose;
    for (int i = threadIdx.x; i < n_pose * IM_POSE_DOUBLES; i += blockDim.x) s_pose[i] = poses[i];
    if (threadIdx.x < 12) s_end[threadIdx.x] = ctrl->state[threadIdx.x];
    __syncthreads();
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) immesh::imu_undistort_point(P, s_end, s_pose, n_pose, pts, s);
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_undistort(ImuParams P, const LioCtrl* ctrl, const double* __restrict__ poses, const ImuTime* tm, float* pts, int n) {
    imu_undistort_block(P, ctrl, poses, tm, pts, n);
}

// ---- the depth IMU chain: the decision of imu_core.cuh (dimu_decide, dimu_init, dimu_begin) on one thread, in stream order
static_assert(IM_DIMU_DROPPED == IMMESH_FEED_BRANCH_DROPPED, "the dropped branch is the feed's");
__global__ void k_dimu_branch(DepthImu* D, const int* d_n, const double* __restrict__ own, int n_own, double* batch, int max_imu, int* err) {
    __shared__ int s_base;
    if (threadIdx.x == 0) {
        int overflow = 0;
        s_base = immesh::dimu_decide(*D, *d_n, n_own, max_imu, &overflow);
        if (overflow) atomicOr(err, immesh::IM_ERR_IMU_CARRY);
    }
    __syncthreads();
    const int base = s_base;
    if (base >= 0)
        for (int i = threadIdx.x; i < 7 * n_own; i += blockDim.x) batch[7 * (size_t)base + i] = own[i];
}
__global__ void k_dimu_init(DepthImu* D, const double* __restrict__ batch, double* state, ImuTime* tm, double frame_time) {
    if (threadIdx.x == 0) immesh::dimu_init(*D, batch, state, *tm, frame_time);
}
__global__ void k_dimu_begin(DepthImu* D, int fresh, int max_ini) {
    if (threadIdx.x == 0) immesh::dimu_begin(*D, fresh, max_ini);
}
__global__ void __launch_bounds__(VG_THREADS) k_dimu_expand(const DepthImu* D, const float* __restrict__ xyz, float4* out) {
    const int n = D->n_und;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        out[i] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], 0.0f);
}
__global__ void __launch_bounds__(IMU_FWD_THREADS) k_imu_forward_dn(ImuParams P, const DepthImu* D, LioCtrl* ctrl, double* run, ImuTime* tm, const double* imu,
                                                                     const float* pts, double lidar_beg_time, ImuStep* steps, double* poses) {
    const int n = D->n_und;
    if (n <= 0) return;   // block-uniform: branches 2 and 3 only
    P.mean_acc_norm = D->mean_acc_norm;
    imu_forward_block(P, ctrl, run, tm, imu, D->n_imu, pts, n, lidar_beg_time, steps, poses);
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_undistort_dn(ImuParams P, const DepthImu* D, const LioCtrl* ctrl, const double* __restrict__ poses, const ImuTime* tm,
                                                                  float* pts) {
    const int n = D->n_und;
    if (n <= 0) return;
    imu_undistort_block(P, ctrl, poses, tm, pts, n);
}

}  // namespace

struct immesh_imu {
    ImuParams P;
    int max_points = 0, max_imu = 0, nblocks_max = 0, n_sm = 132;
    // ImuProcess members on the device: ImuTime (time stamps) and run = [acc_s_last 3 | angvel_last 3 | vel 3 | pos 3 | R 9]
    ImuTime* d_time = nullptr;
    double* d_run = nullptr;
    double* d_poses = nullptr;      // [max_imu + 2][22]
    ImuStep* d_steps = nullptr;     // [max_imu] the plan of the last scan
    double* d_imu = nullptr;        // [max_imu][7] the scan's IMU batch
    float* d_in = nullptr;          // [max_points][4] the scan, when given in host memory
    float* d_out = nullptr;         // [max_points][4] time-sorted, compensated
    unsigned int *d_k[2] = {nullptr, nullptr}, *d_v[2] = {nullptr, nullptr};
    int* d_hist = nullptr;
    // pinned staging ring, IM_SLOTS deep: slot s holds a scan's IMU batch and the host words of its copies (h_imu) and a host scan
    // (h_pts); it is reused only after the event recorded behind its copies (ev_stage)
    double* h_imu = nullptr;
    float* h_pts = nullptr;
    size_t slot_doubles = 0;
    cudaEvent_t ev_stage[IM_SLOTS] = {};
    int stage_busy[IM_SLOTS] = {};
    int stage_idx = 0;
    // initialisation phase of immesh_lio_step_async_imu (imu_need_init_ ... MAX_INI_COUNT)
    ImuInit ini = {{0, 0, -1.0}, {0, 0, 0}, 1, 1};
    int init_phase = 0;     // imu_need_init_ (only after immesh_imu_init_begin)
    int max_ini = 3;        // MAX_INI_COUNT (mapping/imu_int_frame)
    int began = 0;          // immesh_imu_init_begin has been called on the handle
    int pending_reset = 0;  // device members still to be reset in stream order: 1 Reset(), 2 a fresh ImuProcess
    int map_built = 0;      // m_init_map: the chain has built the VoxelMap
    // immesh_lio_step_async_imu_i, allocated by its first call: the caller's point records and the intensity beside d_in / d_out
    int rec_stride = 0;     // floats per record that d_rec / h_rec hold
    float* d_rec = nullptr; // [max_points][rec_stride] the scan's records, when given in host memory
    float* h_rec = nullptr; // pinned, IM_SLOTS slots of [max_points][rec_stride]
    float* d_in_i = nullptr;   // [max_points] intensity in scan order
    float* d_out_i = nullptr;  // [max_points] intensity in time order (beside d_out)
    // which chain runs on the handle: 0 none yet, 1 immesh_lio_step_async_imu[_i] (phase on the host), 2 immesh_lio_step_async_depth_imu
    // (phase on the device, in d_dimu; allocated by its first call with d_own)
    int chain = 0;
    DepthImu* d_dimu = nullptr;
    DepthImu* h_dimu = nullptr;   // pinned: the first call's upload, the state query's read
    double* d_own = nullptr;      // [max_imu][7] the frame's own samples (d_imu holds the batch)
    int dimu_begin = 0;           // immesh_imu_init_begin since the last depth call: k_dimu_begin is due
    int dimu_fresh = 0;           //   and it was the handle's first (a fresh ImuProcess)
    immesh::MemSet dev, pinned{immesh::MemSet::Pinned};   // every buffer above
};

// internal entry points of frontend_capi.cu / lio_capi.cu
extern "C" int immesh_voxelgrid_max_points(immesh_voxelgrid_t* h);
extern "C" int immesh_frontend_build_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* d_pts, int n, int stride, int calib_laser, const float* d_inten);
extern "C" int immesh_frontend_step_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float leaf,
                                          double dt, double cov_gyr, double cov_acc, int icol, const float* isep);
extern "C" int immesh_lio_feed_record_state(immesh_lio_t* lio, int kind, int branch);

// the next staging slot; blocks (back-pressure, counted in the localization handle's host wait) while its last copies are in flight
static int imu_stage_slot(immesh_imu* h, immesh_lio* lio) {
    const int s = (++h->stage_idx) & (IM_SLOTS - 1);
    if (h->stage_busy[s]) {
        const auto t0 = std::chrono::steady_clock::now();
        IM_CUDA(cudaEventSynchronize(h->ev_stage[s]));
        lio->host_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        h->stage_busy[s] = 0;
    }
    return s;
}
static int imu_stage_release(immesh_imu* h, int s, cudaStream_t st) {
    IM_CUDA(cudaEventRecord(h->ev_stage[s], st));
    h->stage_busy[s] = 1;
    return IMMESH_OK;
}

// the buffers of the _i entry: intensity beside d_in / d_out, and record staging of `stride` floats per point (grown for wider
// records).  Each of the two steps is all or nothing: after a failure the handle is as it was.
static int imu_records_alloc(immesh_imu* h, int stride) {
    const size_t n = (size_t)h->max_points;
    if (!h->d_in_i) {
        immesh::MemSet dev;
        float *d_in_i, *d_out_i;
        IM_CUDA(dev.alloc(&d_in_i, n));
        IM_CUDA(dev.alloc(&d_out_i, n));
        h->d_in_i = d_in_i;
        h->d_out_i = d_out_i;
        h->dev.take(std::move(dev));
    }
    if (stride > h->rec_stride) {
        immesh::MemSet dev, pinned(immesh::MemSet::Pinned);
        float *d_rec, *h_rec;
        IM_CUDA(dev.alloc(&d_rec, n * stride));
        IM_CUDA(pinned.alloc(&h_rec, IM_SLOTS * n * stride));
        IM_CUDA(cudaDeviceSynchronize());   // no queued copy still reads the narrower staging
        h->dev.free(h->d_rec); h->pinned.free(h->h_rec);
        h->d_rec = d_rec; h->h_rec = h_rec; h->rec_stride = stride;
        h->dev.take(std::move(dev));
        h->pinned.take(std::move(pinned));
    }
    return IMMESH_OK;
}

// UndistortPcl queued on the localization stream through staging slot s: batch (+ host scan) upload, plan + forward propagation,
// stable time sort, compensation into d_out.  No host synchronisation.  icol >= 0: pts holds records of `stride` floats (time stamp in
// column tcol, intensity in icol), taken apart into d_in / d_in_i, and the intensity is sorted with the points into d_out_i.
static int imu_enqueue_undistort(immesh_imu* h, immesh_lio* lio, const double* imu, int n_imu, const float* pts_xyzt, int n, int on_device, double lidar_beg_time, int s,
                                 int stride = 4, int tcol = 3, int icol = -1) {
    cudaStream_t st = lio->stream;
    if (n_imu > 0) {
        double* hi = h->h_imu + (size_t)s * h->slot_doubles;
        std::memcpy(hi, imu, (size_t)n_imu * 7 * sizeof(double));
        IM_CUDA(cudaMemcpyAsync(h->d_imu, hi, (size_t)n_imu * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    const float* d_pts = pts_xyzt;
    if (icol >= 0) {
        const float* d_rec = pts_xyzt;
        if (!on_device) {
            float* hr = h->h_rec + (size_t)s * h->max_points * h->rec_stride;
            std::memcpy(hr, pts_xyzt, (size_t)n * stride * sizeof(float));
            IM_CUDA(cudaMemcpyAsync(h->d_rec, hr, (size_t)n * stride * sizeof(float), cudaMemcpyHostToDevice, st));
            d_rec = h->d_rec;
        }
        IM_LAUNCH(k_imu_intake, std::min((n + VG_THREADS - 1) / VG_THREADS, h->n_sm * 8), VG_THREADS, 0, st, d_rec, n, stride, tcol, icol, (float4*)h->d_in, h->d_in_i);
        d_pts = h->d_in;
    } else if (!on_device) {
        float* hp = h->h_pts + (size_t)s * h->max_points * 4;
        std::memcpy(hp, pts_xyzt, (size_t)n * 4 * sizeof(float));
        IM_CUDA(cudaMemcpyAsync(h->d_in, hp, (size_t)n * 4 * sizeof(float), cudaMemcpyHostToDevice, st));
        d_pts = h->d_in;
    }
    IM_LAUNCH(k_imu_forward, 1, IMU_FWD_THREADS, 0, st, h->P, lio->d_ctrl, h->d_run, h->d_time, (const double*)h->d_imu, n_imu, d_pts, n, lidar_beg_time, h->d_steps, h->d_poses);
    const int nb = (n + VG_TILE - 1) / VG_TILE;
    const int gs = std::min(nb * (VG_TILE / VG_THREADS), h->n_sm * 8);
    IM_LAUNCH(k_imu_keys, gs, VG_THREADS, 0, st, d_pts, n, h->d_k[0], h->d_v[0]);
    const int cur = rs_sort_passes(st, h->d_k, h->d_v, 0, n, 4, h->d_hist);
    IM_LAUNCH(k_imu_gather, gs, VG_THREADS, 0, st, (const float4*)d_pts, (const unsigned int*)h->d_v[cur], n, (float4*)h->d_out,
              icol >= 0 ? (const float*)h->d_in_i : (const float*)nullptr, icol >= 0 ? h->d_out_i : (float*)nullptr);
    const size_t smem = (size_t)(n_imu + 1) * IM_POSE_DOUBLES * sizeof(double);   // IMUpose holds at most n_imu + 1 entries
    IM_LAUNCH(k_imu_undistort, gs, VG_THREADS, smem, st, h->P, (const LioCtrl*)lio->d_ctrl, (const double*)h->d_poses, (const ImuTime*)h->d_time, h->d_out, n);
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}

extern "C" {

int immesh_imu_create(const immesh_imu_config* c, immesh_imu_t** out) {
    if (!c || !out || c->max_points < 1 || c->max_imu < 1 || c->max_imu > 256) return im_fail(IMMESH_E_INVALID, "bad argument (max_imu must be in [1, 256])");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path"); }
    immesh::Building<immesh_imu> owner(new immesh_imu(), immesh_imu_destroy);   // every failure below releases what was created
    immesh_imu* h = owner.get();
    for (int i = 0; i < 3; ++i) { h->P.cov_gyr[i] = c->cov_gyr[i]; h->P.cov_acc[i] = c->cov_acc[i]; h->P.cov_bias_gyr[i] = c->cov_bias_gyr[i]; h->P.cov_bias_acc[i] = c->cov_bias_acc[i]; h->P.lid_T[i] = c->lid_T[i]; }
    for (int i = 0; i < 9; ++i) h->P.lid_R[i] = c->lid_R[i];
    h->P.mean_acc_norm = c->mean_acc_norm;
    h->max_points = c->max_points; h->max_imu = c->max_imu;
    h->nblocks_max = (c->max_points + VG_TILE - 1) / VG_TILE;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    const size_t n = (size_t)c->max_points;
    // the time stamps a handle starts from (immesh_imu_reset sets them; a fresh ImuProcess is immesh_imu_init_begin's)
    ImuTime t0;
    std::memset(&t0, 0, sizeof(t0));
    t0.last_lidar_end_time = -1.0;
    t0.n_pose = 1;
    IM_CUDA(h->dev.alloc(&h->d_time, 1));
    IM_CUDA(cudaMemcpy(h->d_time, &t0, sizeof(ImuTime), cudaMemcpyHostToDevice));
    IM_CUDA(h->dev.alloc(&h->d_run, IM_IMU_RUN, 0));
    IM_CUDA(h->dev.alloc(&h->d_poses, ((size_t)c->max_imu + 2) * IM_POSE_DOUBLES));
    IM_CUDA(h->dev.alloc(&h->d_steps, (size_t)c->max_imu + 1));
    IM_CUDA(h->dev.alloc(&h->d_imu, (size_t)c->max_imu * 7));
    IM_CUDA(h->dev.alloc(&h->d_in, n * 4));
    IM_CUDA(h->dev.alloc(&h->d_out, n * 4));
    for (int i = 0; i < 2; ++i) {
        IM_CUDA(h->dev.alloc(&h->d_k[i], n));
        IM_CUDA(h->dev.alloc(&h->d_v[i], n));
    }
    IM_CUDA(h->dev.alloc(&h->d_hist, (size_t)256 * h->nblocks_max));
    h->slot_doubles = (size_t)c->max_imu * 7 + 32;   // the batch + the host words of an initialising scan
    IM_CUDA(h->pinned.alloc(&h->h_imu, IM_SLOTS * h->slot_doubles));
    IM_CUDA(h->pinned.alloc(&h->h_pts, IM_SLOTS * n * 4));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CUDA(cudaEventCreateWithFlags(&h->ev_stage[i], cudaEventDisableTiming));
    *out = owner.release();
    return IMMESH_OK;
}
int immesh_imu_destroy(immesh_imu_t* h) {
    if (!h) return IMMESH_OK;
    cudaDeviceSynchronize();
    for (int i = 0; i < IM_SLOTS; ++i) if (h->ev_stage[i]) cudaEventDestroy(h->ev_stage[i]);
    delete h;
    return IMMESH_OK;
}
int immesh_imu_reset(immesh_imu_t* h, const double* last_imu7, double last_lidar_end_time, double last_update_time, const double* acc_s_last, const double* angvel_last) {
    if (!h || !last_imu7) return im_fail(IMMESH_E_INVALID, "null argument");
    ImuTime t;
    std::memset(&t, 0, sizeof(t));
    std::memcpy(t.last_imu, last_imu7, 7 * sizeof(double));
    t.last_lidar_end_time = last_lidar_end_time;
    t.upd_beg = last_update_time;   // + 0.0f / 1000: exactly last_update_time
    t.n_pose = 1;
    double run6[6] = {0, 0, 0, 0, 0, 0};
    if (acc_s_last) std::memcpy(run6, acc_s_last, 24);
    if (angvel_last) std::memcpy(run6 + 3, angvel_last, 24);
    IM_CUDA(cudaDeviceSynchronize());   // nothing queued earlier still reads the members
    IM_CUDA(cudaMemcpy(h->d_time, &t, sizeof(t), cudaMemcpyHostToDevice));
    IM_CUDA(cudaMemcpy(h->d_run, run6, sizeof(run6), cudaMemcpyHostToDevice));
    return IMMESH_OK;
}

int immesh_imu_undistort(immesh_imu_t* h, immesh_lio_t* lio, const double* imu, int n_imu, const float* pts_xyzt, int n, int on_device, double lidar_beg_time, float* out_xyzt) {
    if (!h || !lio || (!imu && n_imu > 0) || n_imu < 0 || (!pts_xyzt && n > 0) || n < 1) return im_fail(IMMESH_E_INVALID, "bad argument (the scan must hold at least one point)");
    if (n > h->max_points || n_imu > h->max_imu) return im_fail(IMMESH_E_CAPACITY, "scan / IMU batch larger than the configured capacity");
    const int s = imu_stage_slot(h, lio);
    int rc = imu_enqueue_undistort(h, lio, imu, n_imu, pts_xyzt, n, on_device, lidar_beg_time, s);
    if (rc) return rc;
    rc = imu_stage_release(h, s, lio->stream);
    if (rc) return rc;
    lio->pose_pub_idx = -1;   // the state moved
    if (out_xyzt) {
        float* hp = h->h_pts + (size_t)s * h->max_points * 4;
        IM_CUDA(cudaMemcpyAsync(hp, h->d_out, (size_t)n * 4 * sizeof(float), cudaMemcpyDeviceToHost, lio->stream));
        IM_CUDA(cudaStreamSynchronize(lio->stream));
        std::memcpy(out_xyzt, hp, (size_t)n * 4 * sizeof(float));
    }
    return IMMESH_OK;
}
const float* immesh_imu_device_points(immesh_imu_t* h) { return h ? h->d_out : nullptr; }
int immesh_imu_get_poses(immesh_imu_t* h, double* out, int cap_poses) {   // IMUpose of the last call, 22 doubles each; returns their number
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaDeviceSynchronize());
    int n_pose = 0;
    IM_CUDA(cudaMemcpy(&n_pose, &h->d_time->n_pose, sizeof(int), cudaMemcpyDeviceToHost));
    const int m = std::min(cap_poses, n_pose);
    if (m > 0) IM_CUDA(cudaMemcpy(out, h->d_poses, (size_t)m * IM_POSE_DOUBLES * sizeof(double), cudaMemcpyDeviceToHost));
    return n_pose;
}

int immesh_imu_init_begin(immesh_imu_t* h, int max_ini_count) {
    if (!h || max_ini_count < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    h->init_phase = 1;
    h->max_ini = max_ini_count;
    h->dimu_begin = 1;
    immesh::imu_init_reset(h->ini);
    if (!h->began) {   // a fresh ImuProcess: b_first_frame_, zero members
        h->began = 1;
        h->ini.first_frame = 1;
        h->dimu_fresh = 1;
        h->pending_reset = 2;
    } else {           // the loop's reset (m_flg_reset -> Reset()): b_first_frame_ stays false
        h->pending_reset = std::max(h->pending_reset, 1);
    }
    return IMMESH_OK;
}

}  // extern "C"

// the members immesh_imu_init_begin resets, in stream order ahead of the next scan
static int imu_pending_reset(immesh_imu* h, cudaStream_t st) {
    if (h->pending_reset) {
        if (h->pending_reset == 2) {   // a fresh ImuProcess (last_lidar_end_time_ = 0.0, see the header)
            IM_CUDA(cudaMemsetAsync(h->d_time, 0, sizeof(ImuTime), st));
            IM_CUDA(cudaMemsetAsync(h->d_run, 0, 6 * sizeof(double), st));
        } else {                       // Reset(): last_imu_ and angvel_last; acc_s_last and last_lidar_end_time_ are kept
            IM_CUDA(cudaMemsetAsync(h->d_time->last_imu, 0, 7 * sizeof(double), st));
            IM_CUDA(cudaMemsetAsync(h->d_run + 3, 0, 3 * sizeof(double), st));
        }
        h->pending_reset = 0;
    }
    return IMMESH_OK;
}

// the loop of immesh_lio_step_async_imu (icol < 0: [n][4] x y z t) and immesh_lio_step_async_imu_i (records of `stride` floats, the time
// stamp in column tcol, the intensity in icol, carried through the sort, the calibration and the VoxelGrid)
static int imu_chain(immesh_lio_t* lio, immesh_imu_t* h, immesh_voxelgrid_t* vg, const double* imu, int n_imu, const float* pts_xyzt, int n, int stride, int tcol,
                     int icol, int on_device, double lidar_beg_time, int calib_laser, float leaf, int* branch_out) {
    if (branch_out) *branch_out = 0;
    if (!lio || !h || !vg || (!imu && n_imu > 0) || n_imu < 0 || !pts_xyzt || n < 1 || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument (the scan must hold at least one point)");
    if (lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_imu runs on a single GPU: the localization handle is sharded");
    if (n_imu > h->max_imu) return im_fail(IMMESH_E_CAPACITY, "IMU batch larger than the IMU handle's max_imu");
    if (n > h->max_points || n > immesh_voxelgrid_max_points(vg)) return im_fail(IMMESH_E_CAPACITY, "scan larger than the IMU / VoxelGrid handle's max_points");
    if (n > lio->max_scan) return im_fail(IMMESH_E_CAPACITY, "scan larger than the localization handle's max_scan_points (the map is built from the whole scan, and a scan the VoxelGrid passes through reaches the step whole)");
    if (h->chain == 2) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_imu: the IMU handle runs immesh_lio_step_async_depth_imu (its phase is on the device)");
    cudaStream_t st = lio->stream;
    lio->fe_vg = nullptr;   // branches 1 and 2 publish nothing (voxel_mapping.cpp:1879, :1903)
    const int feed_kind = icol >= 0 ? IMMESH_FEED_KIND_IMU_I : IMMESH_FEED_KIND_IMU;   // how the scan feed records this scan
    if (icol >= 0) {
        const int rc = imu_records_alloc(h, on_device ? 0 : stride);
        if (rc) return rc;
    }
    h->chain = 1;
    int prc = imu_pending_reset(h, st);
    if (prc) return prc;
    const int s = imu_stage_slot(h, lio);
    if (h->init_phase) {
        // branch 1 (Process2 :973-1003): lidar_meas.last_update_time = pcl_end_time; IMU_init on a non-empty batch
        double* hw = h->h_imu + (size_t)s * h->slot_doubles + (size_t)h->max_imu * 7;   // host words: [upd_beg, curv | rot 9, bg 3, grav 3 | last_imu 7]
        hw[0] = lidar_beg_time;
        IM_CUDA(cudaMemcpyAsync((char*)h->d_time + offsetof(ImuTime, upd_beg), hw, sizeof(double), cudaMemcpyHostToDevice, st));
        float* curv_dst = (float*)((char*)h->d_time + offsetof(ImuTime, upd_curv));
        if (on_device) {
            IM_CUDA(cudaMemcpyAsync(curv_dst, pts_xyzt + (size_t)stride * (n - 1) + tcol, sizeof(float), cudaMemcpyDeviceToDevice, st));
        } else {
            std::memcpy(hw + 1, pts_xyzt + (size_t)stride * (n - 1) + tcol, sizeof(float));
            IM_CUDA(cudaMemcpyAsync(curv_dst, hw + 1, sizeof(float), cudaMemcpyHostToDevice, st));
        }
        if (n_imu > 0) {
            double* sw = hw + 2;
            double grav[3];
            const double norm = immesh::imu_init_batch(h->ini, imu, n_imu, grav);
            for (int i = 0; i < 9; ++i) sw[i] = (i % 4 == 0) ? 1.0 : 0.0;   // rot_end = Eye3d
            for (int i = 0; i < 3; ++i) { sw[9 + i] = 0.0; sw[12 + i] = grav[i]; }   // bias_g = Zero3d, gravity
            std::memcpy(sw + 15, imu + 7 * (size_t)(n_imu - 1), 7 * sizeof(double));   // last_imu_ = meas.imu.back()
            double* dst = lio->d_ctrl->state;
            IM_CUDA(cudaMemcpyAsync(dst, sw, 9 * sizeof(double), cudaMemcpyHostToDevice, st));
            IM_CUDA(cudaMemcpyAsync(dst + 15, sw + 9, 3 * sizeof(double), cudaMemcpyHostToDevice, st));
            IM_CUDA(cudaMemcpyAsync(dst + 21, sw + 12, 3 * sizeof(double), cudaMemcpyHostToDevice, st));
            IM_CUDA(cudaMemcpyAsync(h->d_time->last_imu, sw + 15, 7 * sizeof(double), cudaMemcpyHostToDevice, st));
            lio->pose_pub_idx = -1;
            if (h->ini.N > h->max_ini) {   // init_iter_num > MAX_INI_COUNT: imu_need_init_ = false; UndistortPcl scales by |mean_acc| from now on
                h->init_phase = 0;
                h->P.mean_acc_norm = norm;
            }
        }
        int rc = imu_stage_release(h, s, st);
        if (rc) return rc;
        rc = immesh_lio_feed_record_state(lio, feed_kind, 1);
        if (rc) return rc;
        if (branch_out) *branch_out = 1;
        return IMMESH_OK;
    }
    int rc = imu_enqueue_undistort(h, lio, imu, n_imu, pts_xyzt, n, on_device, lidar_beg_time, s, stride, tcol, icol);
    if (rc) return rc;
    rc = imu_stage_release(h, s, st);
    if (rc) return rc;
    lio->pose_pub_idx = -1;
    const float* d_out_i = icol >= 0 ? h->d_out_i : nullptr;
    if (!h->map_built) {
        // branch 2: voxel_map_init from the full-resolution, undistorted, calibrated scan (voxel_mapping.cpp:1844-1859, :1894-1904)
        lio->feed_next.kind = feed_kind;
        lio->feed_next.branch = 2;
        rc = immesh_frontend_build_async(lio, vg, h->d_out, n, 4, calib_laser, d_out_i);
        lio->feed_next = immesh_lio::FeedNext();
        if (rc) return rc;
        h->map_built = 1;
        if (branch_out) *branch_out = 2;
        return IMMESH_OK;
    }
    // branch 3: calibration -> VoxelGrid -> IESKF on the propagated state (no Forward_without_imu) -> map_incremental_grow
    lio->feed_next.kind = feed_kind;
    lio->feed_next.branch = 3;
    rc = immesh_frontend_step_async(lio, vg, h->d_out, n, 4, 1, calib_laser, leaf, 0.0, 0.0, 0.0, -1, d_out_i);
    lio->feed_next = immesh_lio::FeedNext();
    if (rc) return rc;
    if (branch_out) *branch_out = 3;
    return IMMESH_OK;
}

extern "C" {

int immesh_lio_step_async_imu(immesh_lio_t* lio, immesh_imu_t* h, immesh_voxelgrid_t* vg, const double* imu, int n_imu, const float* pts_xyzt, int n, int on_device,
                              double lidar_beg_time, int calib_laser, float leaf, int* branch_out) {
    return imu_chain(lio, h, vg, imu, n_imu, pts_xyzt, n, 4, 3, -1, on_device, lidar_beg_time, calib_laser, leaf, branch_out);
}
int immesh_lio_step_async_imu_i(immesh_lio_t* lio, immesh_imu_t* h, immesh_voxelgrid_t* vg, const double* imu, int n_imu, const float* pts, int n, int stride,
                                int time_col, int intensity_col, int on_device, double lidar_beg_time, int calib_laser, float leaf, int* branch_out) {
    if (branch_out) *branch_out = 0;
    if (stride < 4 || stride > 16 || time_col < 3 || time_col >= stride || intensity_col < 3 || intensity_col >= stride || time_col == intensity_col)
        return im_fail(IMMESH_E_INVALID, "bad records (stride <= 16; time_col and intensity_col distinct, >= 3 and < stride)");
    if (lio && lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_imu_i runs on a single GPU: the localization handle is sharded");
    return imu_chain(lio, h, vg, imu, n_imu, pts, n, stride, time_col, intensity_col, on_device, lidar_beg_time, calib_laser, leaf, branch_out);
}

// internal entry points of frontend_capi.cu (the depth frame's cloud, and the chain behind UndistortPcl)
int immesh_frontend_depth_check(immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int point_filter_num, double blind, int* n_sampled);
int immesh_frontend_depth_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num,
                                double blind, const float** d_xyz, const int** d_n);
int immesh_frontend_depth_imu_tail(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* d_xyzt, int n_max, const int* d_und, const int* d_b2, const int* d_b3,
                                   const int* d_branch, float leaf);

// The IMU-enabled loop on depth frames: one queued call per frame, every branch decided on the device (see the header).  The host
// queues the same launches whatever the frame holds; each kernel returns early unless its branch is the one the device took.
int immesh_lio_step_async_depth_imu(immesh_lio_t* lio, immesh_imu_t* h, immesh_voxelgrid_t* vg, const double* imu, int n_imu, const immesh_depth_frame* f,
                                    const void* depth, int on_device, int point_filter_num, double blind, double frame_time, float leaf) {
    if (!lio || !h || !vg || (!imu && n_imu > 0) || n_imu < 0 || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_depth_imu runs on a single GPU: the localization handle is sharded");
    if (h->chain == 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_depth_imu: the IMU handle runs immesh_lio_step_async_imu (its phase is on the host)");
    int ns = 0;
    int rc = immesh_frontend_depth_check(vg, f, depth, point_filter_num, blind, &ns);
    if (rc) return rc;
    if (n_imu > h->max_imu) return im_fail(IMMESH_E_CAPACITY, "IMU batch larger than the IMU handle's max_imu");
    if (ns > h->max_points) return im_fail(IMMESH_E_CAPACITY, "depth frame: more sampled pixels than the IMU handle's max_points");
    if (ns > lio->max_scan) return im_fail(IMMESH_E_CAPACITY, "depth frame: more sampled pixels than the localization handle's max_scan_points (the map is built from the whole cloud)");
    cudaStream_t st = lio->stream;
    if (!h->d_dimu) {   // all or nothing; the device phase starts from the host's (immesh_imu_init_begin before the first call, or none)
        immesh::MemSet dev, pinned(immesh::MemSet::Pinned);
        DepthImu *d_dimu, *h_dimu;
        double* d_own;
        IM_CUDA(dev.alloc(&d_dimu, 1));
        IM_CUDA(pinned.alloc(&h_dimu, 1));
        IM_CUDA(dev.alloc(&d_own, (size_t)h->max_imu * 7));
        std::memset(h_dimu, 0, sizeof(DepthImu));
        h_dimu->ini = h->ini;
        h_dimu->mean_acc_norm = h->P.mean_acc_norm;
        h_dimu->init_phase = h->init_phase;
        h_dimu->max_ini = h->max_ini;
        h_dimu->map_built = h->map_built;
        IM_CUDA(cudaMemcpyAsync(d_dimu, h_dimu, sizeof(DepthImu), cudaMemcpyHostToDevice, st));
        h->d_dimu = d_dimu; h->h_dimu = h_dimu; h->d_own = d_own;
        h->dev.take(std::move(dev));
        h->pinned.take(std::move(pinned));
        h->dimu_begin = 0;   // the upload carries the host's phase, b_first_frame_ included
        h->dimu_fresh = 0;
    }
    h->chain = 2;
    rc = imu_pending_reset(h, st);
    if (rc) return rc;
    if (h->dimu_begin) {
        IM_LAUNCH(k_dimu_begin, 1, 32, 0, st, h->d_dimu, h->dimu_fresh, h->max_ini);
        h->dimu_begin = 0;
        h->dimu_fresh = 0;
    }
    const float* d_xyz = nullptr;
    const int* d_n = nullptr;
    rc = immesh_frontend_depth_async(lio, vg, f, depth, on_device, point_filter_num, blind, &d_xyz, &d_n);
    if (rc) return rc;
    const int s = imu_stage_slot(h, lio);
    if (n_imu > 0) {
        double* hi = h->h_imu + (size_t)s * h->slot_doubles;
        std::memcpy(hi, imu, (size_t)n_imu * 7 * sizeof(double));
        IM_CUDA(cudaMemcpyAsync(h->d_own, hi, (size_t)n_imu * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    rc = imu_stage_release(h, s, st);
    if (rc) return rc;
    DepthImu* D = h->d_dimu;
    const int gs = std::min((ns + VG_THREADS - 1) / VG_THREADS, h->n_sm * 8);
    IM_LAUNCH(k_dimu_branch, 1, 128, 0, st, D, d_n, (const double*)h->d_own, n_imu, h->d_imu, h->max_imu, lio->d_counters + immesh::IM_LC_ERR);
    IM_LAUNCH(k_dimu_init, 1, 32, 0, st, D, (const double*)h->d_imu, lio->d_ctrl->state, h->d_time, frame_time);
    IM_LAUNCH(k_dimu_expand, gs, VG_THREADS, 0, st, (const DepthImu*)D, d_xyz, (float4*)h->d_out);
    IM_LAUNCH(k_imu_forward_dn, 1, IMU_FWD_THREADS, 0, st, h->P, (const DepthImu*)D, lio->d_ctrl, h->d_run, h->d_time, (const double*)h->d_imu, (const float*)h->d_out,
              frame_time, h->d_steps, h->d_poses);
    const size_t smem = (size_t)(h->max_imu + 1) * IM_POSE_DOUBLES * sizeof(double);   // IMUpose holds at most (carried + own) + 1 entries
    IM_LAUNCH(k_imu_undistort_dn, gs, VG_THREADS, smem, st, h->P, (const DepthImu*)D, (const LioCtrl*)lio->d_ctrl, (const double*)h->d_poses, (const ImuTime*)h->d_time,
              h->d_out);
    IM_CUDA(cudaGetLastError());
    lio->pose_pub_idx = -1;
    return immesh_frontend_depth_imu_tail(lio, vg, h->d_out, ns, &D->n_und, &D->n_b2, &D->n_b3, &D->branch, leaf);
}

int immesh_imu_depth_chain_state(immesh_imu_t* h, int64_t out[8]) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 8; ++i) out[i] = 0;
    if (!h->d_dimu) {
        out[7] = h->init_phase ? 0 : 1;
        return IMMESH_OK;
    }
    IM_CUDA(cudaDeviceSynchronize());
    IM_CUDA(cudaMemcpy(h->h_dimu, h->d_dimu, sizeof(DepthImu), cudaMemcpyDeviceToHost));
    for (int i = 0; i < 7; ++i) out[i] = h->h_dimu->cnt[i];
    out[7] = h->h_dimu->init_phase ? 0 : 1;
    return IMMESH_OK;
}

}  // extern "C"
