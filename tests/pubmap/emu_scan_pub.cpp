// TEST INFRASTRUCTURE (not product code): the host emulation of the localization kernels (tests/emu/emu_lio.cpp) with the IESKF
// weight buffer ScanBuf::wsqrt attached, and the two scan publishers -- immesh_lio_effect_cloud (publish_effect_world) and
// immesh_lio_registered_cloud (publish_frame_world) -- on the emulated buffers, with the CUDA library's contract: the same
// __host__ __device__ row function (lio_core.cuh: scan_pub_row), scan order, capacity and validity rules.  Built as its own library:
// the handles it creates keep the weights from the start.
#define immesh_lio_create emu_base_lio_create
#define immesh_lio_destroy emu_base_lio_destroy
#define immesh_lio_estimate emu_base_lio_estimate
#define immesh_voxelmap_build emu_base_voxelmap_build
#define emu_shard_begin emu_base_shard_begin
#include "../emu/emu_lio.cpp"
#undef immesh_lio_create
#undef immesh_lio_destroy
#undef immesh_lio_estimate
#undef immesh_voxelmap_build
#undef emu_shard_begin

#include <unordered_map>

namespace {
struct ScanPub {
    std::vector<float> wsqrt;
    int scan_rows = 0;   // 0: no IESKF run since create / map build, 1: the last run's buffers
};
std::unordered_map<immesh_lio*, ScanPub*> g_spub;
}  // namespace

extern "C" {
int immesh_lio_create(const immesh_lio_config* cfg, immesh_lio_t** out) {
    const int rc = emu_base_lio_create(cfg, out);
    if (rc) return rc;
    immesh_lio* h = *out;
    ScanPub* s = new ScanPub();
    s->wsqrt.assign(h->max_scan, 0.0f);
    g_spub[h] = s;
    h->sb.wsqrt = s->wsqrt.data();
    return 0;
}
int immesh_lio_destroy(immesh_lio_t* h) {
    auto it = g_spub.find(h);
    if (it != g_spub.end()) { delete it->second; g_spub.erase(it); }
    return emu_base_lio_destroy(h);
}
int immesh_voxelmap_build(immesh_lio_t* h, const float* body, int n) {
    g_spub[h]->scan_rows = 0;
    return emu_base_voxelmap_build(h, body, n);
}
int immesh_lio_estimate(immesh_lio_t* h, const float* body, int n, int* iters_run) {
    g_spub[h]->scan_rows = 1;
    return emu_base_lio_estimate(h, body, n, iters_run);
}
int emu_shard_begin(immesh_lio_t* h, const float* body, int n) {
    g_spub[h]->scan_rows = 1;
    return emu_base_shard_begin(h, body, n);
}
int immesh_lio_effect_cloud(immesh_lio_t* h, float* rows, int32_t* scan_index, int cap, int* n_out) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows)) return IMMESH_E_INVALID;
    *n_out = 0;
    if (g_spub[h]->scan_rows == 0) return 0;
    const ScanBuf& sb = h->sb;
    int m = 0;
    for (int i = 0; i < sb.n; ++i) m += sb.match_node[i] >= 0;
    *n_out = m;
    if (m > cap) return IMMESH_E_CAPACITY;
    int k = 0;
    for (int i = 0; i < sb.n; ++i) {
        if (sb.match_node[i] < 0) continue;
        scan_pub_row(h->P, h->ctrl.state, sb.body + (size_t)i * 3, sb.wsqrt[i], rows + (size_t)k * 4);
        if (scan_index) scan_index[k] = i;
        ++k;
    }
    return 0;
}
int immesh_lio_registered_cloud(immesh_lio_t* h, const float* pts, int n, int stride, int intensity_col, int on_device, int point_skip, float* rows, int cap, int* n_out) {
    (void)on_device;   // host memory only
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows) || point_skip <= 0) return IMMESH_E_INVALID;
    if (pts && (n < 0 || stride < 3 || intensity_col >= stride)) return IMMESH_E_INVALID;
    *n_out = 0;
    if (!pts) {
        if (g_spub[h]->scan_rows == 0) return IMMESH_E_INVALID;
        pts = h->sb.body; n = h->sb.n; stride = 3; intensity_col = -1;
    }
    const int m = n > 0 ? (n - 1) / point_skip + 1 : 0;
    *n_out = m;
    if (m > cap) return IMMESH_E_CAPACITY;
    for (int j = 0; j < m; ++j) {
        const float* p = pts + (size_t)j * point_skip * stride;
        scan_pub_row(h->P, h->ctrl.state, p, intensity_col >= 0 ? p[intensity_col] : 0.0f, rows + (size_t)j * 4);
    }
    return 0;
}
}  // extern "C"
