// immesh_b200 -- IMU step in front of the hot path (SURVEY 8f-2): the device bodies of ImuProcess::UndistortPcl
// (/root/reference/src/IMU_Processing.cpp:755-958) and the host part of IMU_init (:188-232).  Split of the work:
//   imu_plan                : time stamps only -- which IMU intervals are live, their dt / offset, the scan-end dt and sign (one thread
//                             of k_imu_forward, on the members carried in ImuTime)
//   imu_init_batch          : IMU_init's running means: on the host for immesh_lio_step_async_imu (the samples are host data), on the
//                             device for immesh_lio_step_async_depth_imu (the batch is assembled there); one implementation for both
//   imu_forward_step        : one IMU interval: bias / gravity-scale correction, 18x18 covariance propagation F P F^T + Q,
//                             attitude / velocity / position integration, IMUpose record (block-cooperative, tid / nthreads)
//   imu_predict_end         : state at the scan end (:881-896)
//   imu_compensate          : one point moved into the scan-end frame (:930-950), thread per point
// Same arithmetic order as oracle/orc_imu.hpp (left to right, no FMA): bit-identical results.
#pragma once
#include "hd_math.cuh"

namespace immesh {

#define IM_POSE_DOUBLES 22   // offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]  (Pose6D, common_lib.h)

struct ImuParams {
    double cov_gyr[3], cov_acc[3], cov_bias_gyr[3], cov_bias_acc[3];
    double mean_acc_norm;
    double lid_R[9], lid_T[3];
};
struct ImuStep {          // one live interval (head, tail) of v_imu
    double gyr_avg[3];    // 0.5 * (head + tail), raw
    double acc_avg[3];
    double dt;            // tail - head, or tail - last_lidar_end_time for the first live interval
    double offs_t;        // tail.stamp - pcl_beg_time
};
// running quantities of the propagation that are not part of the 348-double state: [acc_imu 3 | angvel_avr 3 | vel 3 | pos 3 | R 9]
#define IM_IMU_RUN 21

// The ImuProcess members UndistortPcl reads and writes from scan to scan, kept in device memory so that the interval plan of a scan
// is worked out on the device, in stream order, without reading the scan back.
struct ImuTime {
    double last_imu[7];          // last_imu_: stamp, angular_velocity, linear_acceleration
    double last_lidar_end_time;  // last_lidar_end_time_
    double upd_beg;              // lidar_meas.last_update_time = upd_beg + (double)upd_curv / 1000, the pcl_end_time of the last scan kept as
    float upd_curv;              //   its two inputs (lidar_beg_time, last point's curvature), so that a queued copy of the stamp can set it
    int n_pose;                  // IMUpose entries of the last plan
};

// The time-stamp logic of UndistortPcl (IMU_Processing.cpp:759-787, :810-836, :881-896): the live intervals of v_imu = last_imu_ +
// meas.imu with their dt and offset, the scan-end dt and sign, and the members carried to the next scan.  imu: [n_imu][7];
// last_curv: curvature of the LAST point of the unsorted scan (:786).  Returns the number of live intervals.
IM_HDN inline int imu_plan(ImuTime& tm, const double* imu, int n_imu, float last_curv, double lidar_beg_time, ImuStep* steps, double* note, double* dt_end) {
    const double* back = n_imu > 0 ? imu + 7 * (size_t)(n_imu - 1) : tm.last_imu;
    const double imu_end_time = back[0];
    const double last_update_time = tm.upd_beg + (double)tm.upd_curv / double(1000);
    const double pcl_beg_time = (lidar_beg_time < last_update_time) ? last_update_time : lidar_beg_time;   // MAX
    const double pcl_end_time = lidar_beg_time + (double)last_curv / double(1000);
    tm.upd_beg = lidar_beg_time;
    tm.upd_curv = last_curv;
    int n_steps = 0;
    for (int k = 0; k < n_imu; ++k) {
        const double* head = k == 0 ? tm.last_imu : imu + 7 * (size_t)(k - 1);
        const double* tail = imu + 7 * (size_t)k;
        if (tail[0] < tm.last_lidar_end_time) continue;
        ImuStep& s = steps[n_steps++];
        for (int i = 0; i < 3; ++i) { s.gyr_avg[i] = 0.5 * (head[1 + i] + tail[1 + i]); s.acc_avg[i] = 0.5 * (head[4 + i] + tail[4 + i]); }
        s.dt = (head[0] < tm.last_lidar_end_time) ? tail[0] - tm.last_lidar_end_time : tail[0] - head[0];
        s.offs_t = tail[0] - pcl_beg_time;
    }
    if (imu_end_time > pcl_beg_time) { *note = pcl_end_time > imu_end_time ? 1.0 : -1.0; *dt_end = *note * (pcl_end_time - imu_end_time); }
    else { *note = pcl_end_time > pcl_beg_time ? 1.0 : -1.0; *dt_end = *note * (pcl_end_time - pcl_beg_time); }
    if (back != tm.last_imu)
        for (int i = 0; i < 7; ++i) tm.last_imu[i] = back[i];
    tm.last_lidar_end_time = pcl_end_time;
    tm.n_pose = n_steps + 1;
    return n_steps;
}

// IMU_init, StatesGroup version (IMU_Processing.cpp:188-232): the samples in the reference's order, nothing else read.
// The covariance lines are commented out in the reference and absent here.
struct ImuInit {
    double mean_acc[3], mean_gyr[3];
    int N;             // init_iter_num (counts samples)
    int first_frame;   // b_first_frame_
};
// ImuProcess::Reset() as far as IMU_init's members go (:73-86)
IM_HDN inline void imu_init_reset(ImuInit& s) {
    s.mean_acc[0] = 0.0; s.mean_acc[1] = 0.0; s.mean_acc[2] = -1.0;
    s.mean_gyr[0] = s.mean_gyr[1] = s.mean_gyr[2] = 0.0;
    s.N = 1;
}
// one non-empty batch; returns |mean_acc| and gravity = -mean_acc / |mean_acc| * G_m_s2 (rot_end = I, bias_g = 0 are the caller's)
IM_HDN inline double imu_init_batch(ImuInit& s, const double* imu, int n_imu, double* gravity) {
    if (s.first_frame) {
        imu_init_reset(s);
        s.first_frame = 0;
        for (int i = 0; i < 3; ++i) { s.mean_acc[i] = imu[4 + i]; s.mean_gyr[i] = imu[1 + i]; }
    }
    for (int k = 0; k < n_imu; ++k) {
        const double* m = imu + 7 * (size_t)k;
        const double N = (double)s.N;
        for (int i = 0; i < 3; ++i) { s.mean_acc[i] = s.mean_acc[i] + (m[4 + i] - s.mean_acc[i]) / N; s.mean_gyr[i] = s.mean_gyr[i] + (m[1 + i] - s.mean_gyr[i]) / N; }
        s.N++;
    }
    const double norm = sqrt((s.mean_acc[0] * s.mean_acc[0] + s.mean_acc[1] * s.mean_acc[1]) + s.mean_acc[2] * s.mean_acc[2]);
    for (int i = 0; i < 3; ++i) gravity[i] = -s.mean_acc[i] / norm * 9.81;
    return norm;
}

// ---- the depth IMU chain (immesh_lio_step_async_depth_imu): the device-resident phase of ImuProcess and of the loop around it, and the
// decision of a frame, which one thread takes on the device (k_dimu_branch, k_dimu_init) and the host emulation restates.
#define IM_DIMU_DROPPED 4   // IMMESH_FEED_BRANCH_DROPPED
struct DepthImu {
    ImuInit ini;           // IMU_init's running means (init_iter_num, b_first_frame_)
    double mean_acc_norm;  // UndistortPcl's scale: the configured value until IMU_init ends, then |mean_acc|
    int init_phase;        // imu_need_init_
    int max_ini;           // MAX_INI_COUNT
    int map_built;         // m_init_map
    int carry;             // IMU samples of dropped frames, at the front of the batch buffer
    int branch;            // this frame's: 1, 2, 3 or IM_DIMU_DROPPED
    int n;                 // this frame's cloud
    int n_imu;             // this frame's batch: carried + own samples
    int n_und, n_b2, n_b3; // the cloud in branches 2 and 3 / 2 / 3, else 0: the counts the later kernels read
    long long cnt[8];      // calls, dropped, branch-1, -2, -3 frames, carried samples, carry overflows (immesh_imu_depth_chain_state)
};
// sync_packages (src/voxel_mapping_common.cpp:393-400): a cloud of <= 1 point is dropped and its IMU samples stay buffered for the next
// frame, whose meas.imu is then carried + own samples in arrival order.  More than max_imu of them: the frame is dropped and its own
// samples discarded (*overflow = 1).  Otherwise the branch of Process2 (IMU_Processing.cpp:973-1003) and service_LiDAR_update
// (voxel_mapping.cpp:1894-1905).  Returns the batch index the frame's own samples go to, or -1 when they are discarded.
IM_HDN inline int dimu_decide(DepthImu& D, int n, int n_own, int max_imu, int* overflow) {
    const int carry = D.carry, total = carry + n_own;
    int br = IM_DIMU_DROPPED, base = carry;
    *overflow = 0;
    if (total > max_imu) {
        *overflow = 1;
        base = -1;
        D.cnt[6] += 1;
    } else if (n <= 1) {
        D.carry = total;
    } else {
        D.carry = 0;
        D.n_imu = total;
        br = D.init_phase ? 1 : D.map_built ? 3 : 2;
        if (br == 2) D.map_built = 1;
    }
    D.cnt[0] += 1;
    D.cnt[br == IM_DIMU_DROPPED ? 1 : 1 + br] += 1;
    D.cnt[5] = D.carry;
    D.branch = br;
    D.n = n;
    D.n_und = br == 2 || br == 3 ? n : 0;
    D.n_b2 = br == 2 ? n : 0;
    D.n_b3 = br == 3 ? n : 0;
    return base;
}
// branch 1 (Process2 :973-1003): lidar_meas.last_update_time = pcl_end_time (frame_time + 0 / 1000: the depth points' curvature is 0);
// on a non-empty batch IMU_init, rot_end = I, bias_g = 0, gravity, last_imu_ = the batch's last sample, and the init-end test
// init_iter_num > MAX_INI_COUNT.  state: the 348-double state.  Other branches: nothing.
IM_HDN inline void dimu_init(DepthImu& D, const double* batch, double* state, ImuTime& tm, double frame_time) {
    if (D.branch != 1) return;
    tm.upd_beg = frame_time;
    tm.upd_curv = 0.0f;
    const int n_imu = D.n_imu;
    if (n_imu == 0) return;
    double grav[3];
    const double norm = imu_init_batch(D.ini, batch, n_imu, grav);
    for (int i = 0; i < 9; ++i) state[i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 3; ++i) { state[15 + i] = 0.0; state[21 + i] = grav[i]; }
    for (int i = 0; i < 7; ++i) tm.last_imu[i] = batch[7 * (size_t)(n_imu - 1) + i];
    if (D.ini.N > D.max_ini) {
        D.init_phase = 0;
        D.mean_acc_norm = norm;
    }
}
// immesh_imu_init_begin on a handle whose phase is on the device: Reset() of IMU_init's members (IMU_Processing.cpp:73-86) --
// b_first_frame_ kept, unless fresh (the handle's first immesh_imu_init_begin: a new ImuProcess, b_first_frame_ = true) -- the carry
// discarded (its samples belong before the reset); the first-map flag, mean_acc_norm and the counters are kept
IM_HDN inline void dimu_begin(DepthImu& D, int fresh, int max_ini) {
    imu_init_reset(D.ini);
    if (fresh) D.ini.first_frame = 1;
    D.init_phase = 1;
    D.max_ini = max_ini;
    D.carry = 0;
    D.cnt[5] = 0;
}

IM_HDN inline void imu_write_pose(double* pose, double t, const double* run) {
    pose[0] = t;
    for (int i = 0; i < 3; ++i) { pose[1 + i] = run[i]; pose[4 + i] = run[3 + i]; pose[7 + i] = run[6 + i]; pose[10 + i] = run[9 + i]; }
    for (int i = 0; i < 9; ++i) pose[13 + i] = run[12 + i];
}
// state: the 348-double StatesGroup image (rot 0, pos 9, vel 12, bg 15, ba 18, grav 21, cov 24).  Fx, T: 324-double scratch.
IM_HDN inline void imu_forward_step(const ImuParams& P, double* state, double* run, const ImuStep& s, double* pose_out, double* Fx, double* T, int tid, int nthreads) {
    double* cov = state + 24;
    const double dt = s.dt;
    if (tid == 0) {
        double angvel[3], acc_avr[3];
        for (int i = 0; i < 3; ++i) { angvel[i] = s.gyr_avg[i] - state[15 + i]; acc_avr[i] = s.acc_avg[i] * 9.81 / P.mean_acc_norm - state[18 + i]; }
        double En[9], Ask[9], RA[9];
        const double* R = run + 12;
        so3_exp_dt(angvel, -dt, En);
        skew3(acc_avr, Ask);
        m3_mul(R, Ask, RA);
        for (int i = 0; i < 324; ++i) Fx[i] = 0.0;
        for (int i = 0; i < 18; ++i) Fx[i * 18 + i] = 1.0;
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) {
                Fx[a * 18 + b] = En[a * 3 + b];
                Fx[a * 18 + 9 + b] = (a == b) ? -1.0 * dt : -0.0 * dt;
                Fx[(3 + a) * 18 + 6 + b] = (a == b) ? 1.0 * dt : 0.0 * dt;
                Fx[(6 + a) * 18 + b] = -RA[a * 3 + b] * dt;
                Fx[(6 + a) * 18 + 12 + b] = -R[a * 3 + b] * dt;
                Fx[(6 + a) * 18 + 15 + b] = (a == b) ? 1.0 * dt : 0.0 * dt;
            }
        for (int i = 0; i < 3; ++i) { run[3 + i] = angvel[i]; T[i] = acc_avr[i]; }   // T[0..2]: acc_avr handed to the last phase (T is rewritten below only after the barrier)
    }
    IM_SYNCBLOCK();
    double acc_keep[3] = {T[0], T[1], T[2]};
    IM_SYNCBLOCK();
    for (int idx = tid; idx < 324; idx += nthreads) {
        const int i = idx / 18, j = idx % 18;
        double sum = 0.0;
        for (int k = 0; k < 18; ++k) sum = sum + Fx[i * 18 + k] * cov[k * 18 + j];
        T[idx] = sum;
    }
    IM_SYNCBLOCK();
    {
        // cov_w: diag(cov_gyr) dt^2 at (0,0), R diag(cov_acc) R^T dt^2 at (6,6), diag(cov_bias_gyr) dt^2 at (9,9), diag(cov_bias_acc) dt^2 at (12,12)
        const double* R = run + 12;
        for (int idx = tid; idx < 324; idx += nthreads) {
            const int i = idx / 18, j = idx % 18;
            double sum = 0.0;
            for (int k = 0; k < 18; ++k) sum = sum + T[i * 18 + k] * Fx[j * 18 + k];
            double cw = 0.0;
            if (i < 3 && i == j) cw = P.cov_gyr[i] * dt * dt;
            else if (i >= 6 && i < 9 && j >= 6 && j < 9) {
                const int a = i - 6, b = j - 6;
                // ((R D) R^T)(a,b), products with the zero entries of D included as in the dense evaluation
                double rc[3];
                for (int q = 0; q < 3; ++q) rc[q] = (R[a * 3 + 0] * (q == 0 ? P.cov_acc[0] : 0.0) + R[a * 3 + 1] * (q == 1 ? P.cov_acc[1] : 0.0)) + R[a * 3 + 2] * (q == 2 ? P.cov_acc[2] : 0.0);
                cw = ((rc[0] * R[b * 3 + 0] + rc[1] * R[b * 3 + 1]) + rc[2] * R[b * 3 + 2]) * dt * dt;
            } else if (i >= 9 && i < 12 && i == j) cw = P.cov_bias_gyr[i - 9] * dt * dt;
            else if (i >= 12 && i < 15 && i == j) cw = P.cov_bias_acc[i - 12] * dt * dt;
            cov[idx] = sum + cw;
        }
    }
    IM_SYNCBLOCK();
    if (tid == 0) {
        double* acc_imu = run; double* angvel = run + 3; double* vel = run + 6; double* pos = run + 9; double* R = run + 12;
        double Ef[9], Rn[9], Ra[3];
        so3_exp_dt(angvel, dt, Ef);
        m3_mul(R, Ef, Rn);
        for (int i = 0; i < 9; ++i) R[i] = Rn[i];
        m3_vec(R, acc_keep, Ra);
        for (int i = 0; i < 3; ++i) acc_imu[i] = Ra[i] + state[21 + i];
        for (int i = 0; i < 3; ++i) pos[i] = (pos[i] + vel[i] * dt) + 0.5 * acc_imu[i] * dt * dt;
        for (int i = 0; i < 3; ++i) vel[i] = vel[i] + acc_imu[i] * dt;
        imu_write_pose(pose_out, s.offs_t, run);
    }
    IM_SYNCBLOCK();
}
// state at the scan end: vel_end, rot_end, pos_end  (note = +-1, dt already multiplied by note on the host, :881-896)
IM_HDN inline void imu_predict_end(double* state, const double* run, double note, double dt) {
    const double* acc_imu = run; const double* angvel = run + 3; const double* vel = run + 6; const double* pos = run + 9; const double* R = run + 12;
    const double w[3] = {note * angvel[0], note * angvel[1], note * angvel[2]};
    double E[9], Rn[9];
    for (int i = 0; i < 3; ++i) state[12 + i] = vel[i] + note * acc_imu[i] * dt;
    so3_exp_dt(w, dt, E);
    m3_mul(R, E, Rn);
    for (int i = 0; i < 9; ++i) state[i] = Rn[i];
    for (int i = 0; i < 3; ++i) state[9 + i] = (pos[i] + note * vel[i] * dt) + note * 0.5 * acc_imu[i] * dt * dt;
}
// one application of the backward compensation to point p = (x, y, z, curvature ms) with IMUpose `head`
IM_HDN inline void imu_compensate(const ImuParams& P, const double* state_end, const double* head, float* p) {
    const double dt = (double)p[3] / double(1000) - head[0];
    const double* acc = head + 1; const double* gyr = head + 4; const double* vel = head + 7; const double* pos = head + 10; const double* rot = head + 13;
    double E[9], R_i[9], T_ei[3];
    so3_exp_dt(gyr, dt, E);
    m3_mul(rot, E, R_i);
    for (int i = 0; i < 3; ++i) T_ei[i] = ((pos[i] + vel[i] * dt) + 0.5 * acc[i] * dt * dt) - state_end[9 + i];
    const double P_i[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double a[3], b[3], c[3], d[3];
    m3_vec(P.lid_R, P_i, a);
    for (int i = 0; i < 3; ++i) a[i] = a[i] + P.lid_T[i];
    m3_vec(R_i, a, b);
    for (int i = 0; i < 3; ++i) b[i] = b[i] + T_ei[i];
    for (int i = 0; i < 3; ++i) c[i] = ((state_end[0 * 3 + i] * b[0] + state_end[1 * 3 + i] * b[1]) + state_end[2 * 3 + i] * b[2]) - P.lid_T[i];
    for (int i = 0; i < 3; ++i) d[i] = (P.lid_R[0 * 3 + i] * c[0] + P.lid_R[1 * 3 + i] * c[1]) + P.lid_R[2 * 3 + i] * c[2];
    p[0] = (float)d[0]; p[1] = (float)d[1]; p[2] = (float)d[2];
}
// the point of sorted index s: interval = last head whose offset is < its time; sorted index 0 is re-compensated by every earlier
// head the reference's backward walk still visits (see oracle/orc_imu.hpp)
IM_HDN inline void imu_undistort_point(const ImuParams& P, const double* state_end, const double* poses, int n_pose, float* pts, int s) {
    float* p = pts + 4 * (size_t)s;
    const double t = (double)p[3] / double(1000);
    int j = n_pose - 2;
    while (j >= 0 && !(t > poses[(size_t)j * IM_POSE_DOUBLES])) --j;
    if (j < 0) return;
    imu_compensate(P, state_end, poses + (size_t)j * IM_POSE_DOUBLES, p);
    if (s == 0) {
        for (int q = j - 1; q >= 0; --q)
            if (t > poses[(size_t)q * IM_POSE_DOUBLES]) imu_compensate(P, state_end, poses + (size_t)q * IM_POSE_DOUBLES, p);
    }
}

}  // namespace immesh
