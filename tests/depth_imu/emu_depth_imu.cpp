// Host emulation of the depth IMU chain's decision (immesh_b200/csrc/imu_core.cuh: dimu_decide, dimu_init, dimu_begin), the code
// k_dimu_branch, k_dimu_init and k_dimu_begin run on one device thread, built with the emulation's flags.
// TEST INFRASTRUCTURE: tests/test_depth_imu_emu.py runs it against restatements of sync_packages, Process2 and IMU_init.
#include <cstring>

#include "../../immesh_b200/csrc/lio_core.cuh"   // IM_SYNCBLOCK for the host (one thread)
#include "../../immesh_b200/csrc/imu_core.cuh"

using namespace immesh;

extern "C" {

int emu_dimu_size() { return (int)sizeof(DepthImu); }
int emu_dimu_dropped() { return IM_DIMU_DROPPED; }

// a handle's device phase as the chain's first call sets it up from the host's
void emu_dimu_setup(DepthImu* D, double mean_acc_norm, int init_phase, int max_ini, int first_frame) {
    std::memset(D, 0, sizeof(DepthImu));
    imu_init_reset(D->ini);
    D->ini.first_frame = first_frame;
    D->mean_acc_norm = mean_acc_norm;
    D->init_phase = init_phase;
    D->max_ini = max_ini;
}
// immesh_imu_init_begin on a running handle, with the arguments immesh_lio_step_async_depth_imu passes k_dimu_begin (fresh = 0: the
// loop's reset, b_first_frame_ stays false)
void emu_dimu_begin(DepthImu* D, int fresh, int max_ini) { dimu_begin(*D, fresh, max_ini); }
// one frame: the cloud's count n and the frame's own samples; batch [max_imu][7] carries across calls.  state: [348] in/out;
// tm: [last_imu 7, upd_beg, upd_curv] in/out.  *overflow as dimu_decide.  Returns the branch.
int emu_dimu_frame(DepthImu* D, int n, const double* own, int n_own, double* batch, int max_imu, double* state, double* tm, double frame_time, int* overflow) {
    const int base = dimu_decide(*D, n, n_own, max_imu, overflow);
    if (base >= 0) std::memcpy(batch + 7 * (size_t)base, own, (size_t)n_own * 7 * sizeof(double));
    ImuTime t;
    std::memset(&t, 0, sizeof(t));
    std::memcpy(t.last_imu, tm, 7 * sizeof(double));
    t.upd_beg = tm[7];
    t.upd_curv = (float)tm[8];
    dimu_init(*D, batch, state, t, frame_time);
    std::memcpy(tm, t.last_imu, 7 * sizeof(double));
    tm[7] = t.upd_beg;
    tm[8] = (double)t.upd_curv;
    return D->branch;
}
// [mean_acc 3, mean_gyr 3, N, first_frame, mean_acc_norm, init_phase, map_built, carry, n_imu, n_und, n_b2, n_b3]
void emu_dimu_read(const DepthImu* D, double* out, long long* cnt) {
    for (int i = 0; i < 3; ++i) { out[i] = D->ini.mean_acc[i]; out[3 + i] = D->ini.mean_gyr[i]; }
    out[6] = D->ini.N; out[7] = D->ini.first_frame; out[8] = D->mean_acc_norm; out[9] = D->init_phase; out[10] = D->map_built;
    out[11] = D->carry; out[12] = D->n_imu; out[13] = D->n_und; out[14] = D->n_b2; out[15] = D->n_b3;
    for (int i = 0; i < 8; ++i) cnt[i] = D->cnt[i];
}

}  // extern "C"
