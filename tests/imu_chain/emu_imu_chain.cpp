// Host emulation of the IMU chain's two host-independent bodies (immesh_b200/csrc/imu_core.cuh), built with the emulation's flags:
// the interval plan k_imu_forward works out on the device (imu_plan) and IMU_init's running means (imu_init_batch, imu_init_reset).
// TEST INFRASTRUCTURE: tests/test_imu_chain_emu.py compares them with restatements of the reference.
#include <cstring>

#include "../../immesh_b200/csrc/lio_core.cuh"   // IM_SYNCBLOCK for the host (one thread)
#include "../../immesh_b200/csrc/imu_core.cuh"

using namespace immesh;

extern "C" {

// tm: [last_imu 7, last_lidar_end_time, upd_beg, upd_curv, n_pose] in/out; steps_out: [n_imu][8] (gyr_avg, acc_avg, dt, offs_t);
// out: [note, dt_end].  Returns the number of live intervals.
int emu_imu_plan(double* tm, const double* imu, int n_imu, float last_curv, double lidar_beg_time, double* steps_out, double* out) {
    ImuTime t;
    std::memset(&t, 0, sizeof(t));
    std::memcpy(t.last_imu, tm, 7 * sizeof(double));
    t.last_lidar_end_time = tm[7];
    t.upd_beg = tm[8];
    t.upd_curv = (float)tm[9];
    ImuStep steps[257];
    const int m = imu_plan(t, imu, n_imu, last_curv, lidar_beg_time, steps, out, out + 1);
    for (int k = 0; k < m; ++k) {
        for (int i = 0; i < 3; ++i) { steps_out[8 * k + i] = steps[k].gyr_avg[i]; steps_out[8 * k + 3 + i] = steps[k].acc_avg[i]; }
        steps_out[8 * k + 6] = steps[k].dt;
        steps_out[8 * k + 7] = steps[k].offs_t;
    }
    std::memcpy(tm, t.last_imu, 7 * sizeof(double));
    tm[7] = t.last_lidar_end_time; tm[8] = t.upd_beg; tm[9] = (double)t.upd_curv; tm[10] = t.n_pose;
    return m;
}

// st: [mean_acc 3, mean_gyr 3, N, first_frame] in/out.  reset != 0: ImuProcess::Reset() first.  n_imu > 0: one IMU_init batch,
// gravity -> grav, returns |mean_acc|.
double emu_imu_init(double* st, int reset, const double* imu, int n_imu, double* grav) {
    ImuInit s;
    for (int i = 0; i < 3; ++i) { s.mean_acc[i] = st[i]; s.mean_gyr[i] = st[3 + i]; }
    s.N = (int)st[6];
    s.first_frame = (int)st[7];
    if (reset) imu_init_reset(s);
    double norm = 0.0;
    if (n_imu > 0) norm = imu_init_batch(s, imu, n_imu, grav);
    for (int i = 0; i < 3; ++i) { st[i] = s.mean_acc[i]; st[3 + i] = s.mean_gyr[i]; }
    st[6] = s.N;
    st[7] = s.first_frame;
    return norm;
}

}  // extern "C"
