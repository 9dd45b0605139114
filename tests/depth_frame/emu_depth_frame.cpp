// TEST INFRASTRUCTURE (not product code): the depth frame's __host__ __device__ bodies (immesh_b200/csrc/depth_frame.cuh) run on the CPU
// with the device chain's orchestration -- k_depth_count's valid samples per block of DF_BLOCK sampled pixels, k_rf_scan's offsets, then
// k_depth_emit's points at block offset + rank in the block, and the frame's n, step, m and cmask.  The shipped library never links or
// calls this.
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/depth_frame.cuh"

using namespace immesh;

#define DF_BLOCK 1024   // depth_kernels.cuh

extern "C" {
// img: the device image as the caller passes it (pitch bytes per row); cam = fx fy cx cy z_min z_max depth_scale R[9] t[3].  Writes the
// valid samples' points [n][3] and their pixel indices (v * width + u); dims = n, step, m, cmask.  Returns n.
int emu_depth_frame(const void* img, long long pitch, int width, int height, int format, int kind, int stride, const double* cam, int append_target,
                    float* pts, int* pix, long long* dims) {
    DepthFrame D;
    std::memset(&D, 0, sizeof(D));
    const int bpp = depth_bytes_per_pixel(format);
    D.img = static_cast<const unsigned char*>(img);
    D.row_bytes = (long long)stride * pitch;
    D.col_bytes = (long long)stride * bpp;
    D.sw = depth_sampled(width, stride);
    D.sh = depth_sampled(height, stride);
    D.stride = stride; D.format = format; D.kind = kind;
    D.fx = cam[0]; D.fy = cam[1]; D.cx = cam[2]; D.cy = cam[3]; D.z_min = cam[4]; D.z_max = cam[5]; D.depth_scale = cam[6];
    std::memcpy(D.R, cam + 7, sizeof(D.R));
    std::memcpy(D.t, cam + 16, sizeof(D.t));
    const int ns = D.sw * D.sh, nb = (ns + DF_BLOCK - 1) / DF_BLOCK;
    std::vector<int> blk(nb, 0), off(nb + 1, 0);
    float p[3];
    for (int k = 0; k < ns; ++k) blk[k / DF_BLOCK] += depth_point(D, k, p) ? 1 : 0;   // k_depth_count
    for (int b = 0; b < nb; ++b) off[b + 1] = off[b] + blk[b];                       // k_rf_scan
    for (int b = 0; b < nb; ++b) {                                                   // k_depth_emit
        int rank = 0;
        for (int k = b * DF_BLOCK; k < ns && k < (b + 1) * DF_BLOCK; ++k) {
            if (!depth_point(D, k, p)) continue;
            const int i = off[b] + rank++;
            std::memcpy(pts + (size_t)i * 3, p, sizeof(p));
            pix[i] = (k / D.sw) * stride * width + (k % D.sw) * stride;
        }
    }
    const int n = off[nb];
    int step, m;
    unsigned int cmask;
    frame_append_dims(n, append_target, &step, &m, &cmask);
    dims[0] = n; dims[1] = step; dims[2] = m; dims[3] = cmask;
    return n;
}
// frame_append_dims and frame_append_max_m: out = step, m, cmask, max_m
void emu_append_dims(int n, int append_target, long long* out) {
    int step, m;
    unsigned int cmask;
    frame_append_dims(n, append_target, &step, &m, &cmask);
    out[0] = step; out[1] = m; out[2] = cmask; out[3] = frame_append_max_m(n, append_target);
}
}
