// immesh_b200 -- IMU step in front of the hot path (SURVEY 8f-2) on the device: ImuProcess::UndistortPcl
// (/root/reference/src/IMU_Processing.cpp:755-958), LiDAR-only flow.  The state and its covariance stay in the localization
// handle's HBM (LioCtrl::state); nothing but time stamps is decided on the host.
//   k_imu_begin     running quantities (vel, pos, R) <- state, IMUpose[0]
//   k_imu_forward   one block: all live IMU intervals in sequence (18x18 F P F^T + Q each), scan-end prediction
//   k_imu_keys      time-stamp keys (ordered-uint image of the float curvature) for the stable radix sort (radix_sort.cuh)
//   k_imu_gather    points in time order
//   k_imu_undistort thread per point: interval lookup + rigid transform into the scan-end frame (16 B in, 16 B out per point)
// There is no CPU path.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"
#include "imu_core.cuh"

using immesh::im_fail; using immesh::ImuParams; using immesh::ImuStep;

namespace {

#include "radix_sort.cuh"

#define IMU_FWD_THREADS 352

__global__ void k_imu_begin(const LioCtrl* ctrl, double* run, double* poses) {
    if (threadIdx.x == 0) {
        const double* st = ctrl->state;
        for (int i = 0; i < 3; ++i) { run[6 + i] = st[12 + i]; run[9 + i] = st[9 + i]; }
        for (int i = 0; i < 9; ++i) run[12 + i] = st[i];
        immesh::imu_write_pose(poses, 0.0, run);   // IMUpose[0] = (0, acc_s_last, angvel_last, vel_end, pos_end, rot_end), :800
    }
}
__global__ void __launch_bounds__(IMU_FWD_THREADS) k_imu_forward(ImuParams P, LioCtrl* ctrl, double* run, const ImuStep* steps, int n_steps, double* poses, double note, double dt_end) {
    __shared__ double Fx[324], T[324];
    for (int k = 0; k < n_steps; ++k)
        immesh::imu_forward_step(P, ctrl->state, run, steps[k], poses + (size_t)(k + 1) * IM_POSE_DOUBLES, Fx, T, threadIdx.x, blockDim.x);
    if (threadIdx.x == 0) immesh::imu_predict_end(ctrl->state, run, note, dt_end);
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_keys(const float* __restrict__ pts, int n, unsigned int* keys, unsigned int* vals) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        unsigned int b = __float_as_uint(pts[4 * (size_t)i + 3]);
        if (b == 0x80000000u) b = 0u;                              // -0.0 and +0.0 compare equal in time_list
        keys[i] = (b & 0x80000000u) ? ~b : (b | 0x80000000u);     // order-preserving image of the float (time_list: x.curvature < y.curvature)
        vals[i] = (unsigned int)i;
    }
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_gather(const float4* __restrict__ in, const unsigned int* __restrict__ vals, int n, float4* out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[vals[i]];
}
__global__ void __launch_bounds__(VG_THREADS) k_imu_undistort(ImuParams P, const LioCtrl* ctrl, const double* __restrict__ poses, int n_pose, float* pts, int n) {
    extern __shared__ double s_pose[];
    __shared__ double s_end[12];
    for (int i = threadIdx.x; i < n_pose * IM_POSE_DOUBLES; i += blockDim.x) s_pose[i] = poses[i];
    if (threadIdx.x < 12) s_end[threadIdx.x] = ctrl->state[threadIdx.x];
    __syncthreads();
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) immesh::imu_undistort_point(P, s_end, s_pose, n_pose, pts, s);
}

}  // namespace

struct immesh_imu {
    ImuParams P;
    int max_points = 0, max_imu = 0, nblocks_max = 0, n_sm = 132;
    // ImuProcess members that live on the host (time stamps) ...
    double last_imu[7] = {0, 0, 0, 0, 0, 0, 0};
    double last_lidar_end_time = -1.0, last_update_time = 0.0;
    // ... and on the device: run = [acc_s_last 3 | angvel_last 3 | vel 3 | pos 3 | R 9]
    double* d_run = nullptr;
    double* d_poses = nullptr;      // [max_imu + 2][22]
    ImuStep* d_steps = nullptr;
    ImuStep* h_steps = nullptr;     // pinned
    float* d_in = nullptr;          // [max_points][4] staging of host input
    float* d_out = nullptr;         // [max_points][4] time-sorted, compensated
    unsigned int *d_k[2] = {nullptr, nullptr}, *d_v[2] = {nullptr, nullptr};
    int* d_hist = nullptr;
    float* h_pts = nullptr;         // pinned
    int last_n = 0, last_poses = 0;
};

extern "C" {

int immesh_imu_create(const immesh_imu_config* c, immesh_imu_t** out) {
    if (!c || !out || c->max_points < 1 || c->max_imu < 1 || c->max_imu > 256) return im_fail(IMMESH_E_INVALID, "bad argument (max_imu must be in [1, 256])");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path"); }
    immesh_imu* h = new immesh_imu();
    for (int i = 0; i < 3; ++i) { h->P.cov_gyr[i] = c->cov_gyr[i]; h->P.cov_acc[i] = c->cov_acc[i]; h->P.cov_bias_gyr[i] = c->cov_bias_gyr[i]; h->P.cov_bias_acc[i] = c->cov_bias_acc[i]; h->P.lid_T[i] = c->lid_T[i]; }
    for (int i = 0; i < 9; ++i) h->P.lid_R[i] = c->lid_R[i];
    h->P.mean_acc_norm = c->mean_acc_norm;
    h->max_points = c->max_points; h->max_imu = c->max_imu;
    h->nblocks_max = (c->max_points + VG_TILE - 1) / VG_TILE;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    const size_t n = (size_t)c->max_points;
    IM_CUDA(cudaMalloc((void**)&h->d_run, IM_IMU_RUN * sizeof(double)));
    IM_CUDA(cudaMemset(h->d_run, 0, IM_IMU_RUN * sizeof(double)));
    IM_CUDA(cudaMalloc((void**)&h->d_poses, ((size_t)c->max_imu + 2) * IM_POSE_DOUBLES * sizeof(double)));
    IM_CUDA(cudaMalloc((void**)&h->d_steps, ((size_t)c->max_imu + 1) * sizeof(ImuStep)));
    IM_CUDA(cudaMallocHost((void**)&h->h_steps, ((size_t)c->max_imu + 1) * sizeof(ImuStep)));
    IM_CUDA(cudaMalloc((void**)&h->d_in, n * 4 * sizeof(float)));
    IM_CUDA(cudaMalloc((void**)&h->d_out, n * 4 * sizeof(float)));
    for (int i = 0; i < 2; ++i) {
        IM_CUDA(cudaMalloc((void**)&h->d_k[i], n * sizeof(unsigned int)));
        IM_CUDA(cudaMalloc((void**)&h->d_v[i], n * sizeof(unsigned int)));
    }
    IM_CUDA(cudaMalloc((void**)&h->d_hist, (size_t)256 * h->nblocks_max * sizeof(int)));
    IM_CUDA(cudaMallocHost((void**)&h->h_pts, n * 4 * sizeof(float)));
    *out = h;
    return IMMESH_OK;
}
int immesh_imu_destroy(immesh_imu_t* h) {
    if (!h) return IMMESH_OK;
    cudaDeviceSynchronize();
    cudaFree(h->d_run); cudaFree(h->d_poses); cudaFree(h->d_steps); cudaFreeHost(h->h_steps); cudaFree(h->d_in); cudaFree(h->d_out);
    for (int i = 0; i < 2; ++i) { cudaFree(h->d_k[i]); cudaFree(h->d_v[i]); }
    cudaFree(h->d_hist); cudaFreeHost(h->h_pts);
    delete h;
    return IMMESH_OK;
}
int immesh_imu_reset(immesh_imu_t* h, const double* last_imu7, double last_lidar_end_time, double last_update_time, const double* acc_s_last, const double* angvel_last) {
    if (!h || !last_imu7) return im_fail(IMMESH_E_INVALID, "null argument");
    std::memcpy(h->last_imu, last_imu7, 7 * sizeof(double));
    h->last_lidar_end_time = last_lidar_end_time;
    h->last_update_time = last_update_time;
    double run6[6] = {0, 0, 0, 0, 0, 0};
    if (acc_s_last) std::memcpy(run6, acc_s_last, 24);
    if (angvel_last) std::memcpy(run6 + 3, angvel_last, 24);
    IM_CUDA(cudaMemcpy(h->d_run, run6, sizeof(run6), cudaMemcpyHostToDevice));
    return IMMESH_OK;
}

int immesh_imu_undistort(immesh_imu_t* h, immesh_lio_t* lio, const double* imu, int n_imu, const float* pts_xyzt, int n, int on_device, double lidar_beg_time, float* out_xyzt) {
    if (!h || !lio || (!imu && n_imu > 0) || n_imu < 0 || (!pts_xyzt && n > 0) || n < 1) return im_fail(IMMESH_E_INVALID, "bad argument (the scan must hold at least one point)");
    if (n > h->max_points || n_imu > h->max_imu) return im_fail(IMMESH_E_CAPACITY, "scan / IMU batch larger than the configured capacity");
    cudaStream_t st = lio->stream;
    // ---- host: time stamps only (v_imu = last_imu_ + meas.imu, :759-764)
    std::vector<const double*> v;
    v.push_back(h->last_imu);
    for (int i = 0; i < n_imu; ++i) v.push_back(imu + 7 * (size_t)i);
    const double imu_end_time = v.back()[0];
    const double pcl_beg_time = std::max(lidar_beg_time, h->last_update_time);
    float last_curv = 0.f;
    if (on_device) IM_CUDA(cudaMemcpy(&last_curv, pts_xyzt + 4 * (size_t)(n - 1) + 3, sizeof(float), cudaMemcpyDeviceToHost));
    else last_curv = pts_xyzt[4 * (size_t)(n - 1) + 3];
    const double pcl_end_time = lidar_beg_time + (double)last_curv / double(1000);
    h->last_update_time = pcl_end_time;
    int n_steps = 0;
    for (size_t k = 0; k + 1 < v.size(); ++k) {
        const double *head = v[k], *tail = v[k + 1];
        if (tail[0] < h->last_lidar_end_time) continue;
        ImuStep& s = h->h_steps[n_steps++];
        for (int i = 0; i < 3; ++i) { s.gyr_avg[i] = 0.5 * (head[1 + i] + tail[1 + i]); s.acc_avg[i] = 0.5 * (head[4 + i] + tail[4 + i]); }
        s.dt = (head[0] < h->last_lidar_end_time) ? tail[0] - h->last_lidar_end_time : tail[0] - head[0];
        s.offs_t = tail[0] - pcl_beg_time;
    }
    double note, dt_end;
    if (imu_end_time > pcl_beg_time) { note = pcl_end_time > imu_end_time ? 1.0 : -1.0; dt_end = note * (pcl_end_time - imu_end_time); }
    else { note = pcl_end_time > pcl_beg_time ? 1.0 : -1.0; dt_end = note * (pcl_end_time - pcl_beg_time); }
    std::memcpy(h->last_imu, v.back(), 7 * sizeof(double));
    h->last_lidar_end_time = pcl_end_time;
    // ---- device
    const float* d_pts = pts_xyzt;
    if (!on_device) {
        std::memcpy(h->h_pts, pts_xyzt, (size_t)n * 4 * sizeof(float));
        IM_CUDA(cudaMemcpyAsync(h->d_in, h->h_pts, (size_t)n * 4 * sizeof(float), cudaMemcpyHostToDevice, st));
        d_pts = h->d_in;
    }
    if (n_steps > 0) IM_CUDA(cudaMemcpyAsync(h->d_steps, h->h_steps, (size_t)n_steps * sizeof(ImuStep), cudaMemcpyHostToDevice, st));
    IM_LAUNCH(k_imu_begin, 1, 32, 0, st, (const LioCtrl*)lio->d_ctrl, h->d_run, h->d_poses);
    IM_LAUNCH(k_imu_forward, 1, IMU_FWD_THREADS, 0, st, h->P, lio->d_ctrl, h->d_run, (const ImuStep*)h->d_steps, n_steps, h->d_poses, note, dt_end);
    const int nb = (n + VG_TILE - 1) / VG_TILE;
    const int gs = std::min(nb * (VG_TILE / VG_THREADS), h->n_sm * 8);
    IM_LAUNCH(k_imu_keys, gs, VG_THREADS, 0, st, d_pts, n, h->d_k[0], h->d_v[0]);
    int cur = 0;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 8 * pass;
        IM_LAUNCH(k_rs_hist, nb, VG_THREADS, 0, st, (const unsigned int*)h->d_k[cur], n, shift, h->d_hist, nb);
        IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, h->d_hist, 256 * nb, (int*)nullptr);
        IM_LAUNCH(k_rs_scatter, nb, VG_THREADS, 0, st, (const unsigned int*)h->d_k[cur], (const unsigned int*)h->d_v[cur], h->d_k[cur ^ 1], h->d_v[cur ^ 1], n, shift,
                  (const int*)h->d_hist, nb);
        cur ^= 1;
    }
    IM_LAUNCH(k_imu_gather, gs, VG_THREADS, 0, st, (const float4*)d_pts, (const unsigned int*)h->d_v[cur], n, (float4*)h->d_out);
    const int n_pose = n_steps + 1;
    IM_LAUNCH(k_imu_undistort, gs, VG_THREADS, (size_t)n_pose * IM_POSE_DOUBLES * sizeof(double), st, h->P, (const LioCtrl*)lio->d_ctrl, (const double*)h->d_poses, n_pose, h->d_out, n);
    IM_CUDA(cudaGetLastError());
    h->last_n = n; h->last_poses = n_pose;
    if (out_xyzt) {
        IM_CUDA(cudaMemcpyAsync(h->h_pts, h->d_out, (size_t)n * 4 * sizeof(float), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
        std::memcpy(out_xyzt, h->h_pts, (size_t)n * 4 * sizeof(float));
    }
    return IMMESH_OK;
}
const float* immesh_imu_device_points(immesh_imu_t* h) { return h ? h->d_out : nullptr; }
int immesh_imu_get_poses(immesh_imu_t* h, double* out, int cap_poses) {   // IMUpose of the last call, 22 doubles each; returns their number
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int m = std::min(cap_poses, h->last_poses);
    IM_CUDA(cudaDeviceSynchronize());
    IM_CUDA(cudaMemcpy(out, h->d_poses, (size_t)m * IM_POSE_DOUBLES * sizeof(double), cudaMemcpyDeviceToHost));
    return h->last_poses;
}

}  // extern "C"
