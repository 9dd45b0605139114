// TEST INFRASTRUCTURE (not product code): the localization's depth filter -- depth_frame.cuh's depth_point and depth_keep, the bodies the
// front-end kernels run -- with the kernels' multi-pass block compaction restated on the CPU (depth_kernels.cuh): k_depth_count's valid
// samples per block of `block` sampled pixels, their offsets, k_depth_keep's kept samples per block from each valid sample's global index
// (block offset + rank in the block), their offsets, then k_depth_emit's points at kept offset + rank in the block.  The shipped library
// never links or calls this.
#include <cstring>
#include <vector>

#include "../../immesh_b200/csrc/depth_frame.cuh"

using namespace immesh;

extern "C" {
// img: the device image as the caller passes it (pitch bytes per row); cam = fx fy cx cy z_min z_max depth_scale R[9] t[3] (camera to
// sensor frame).  block: sampled pixels per block (the kernels' DF_BLOCK = 1024; any block gives the same cloud).  Writes the kept
// points [n][3] and their pixel indices (v * width + u).  Returns n.
int emu_depth_lio(const void* img, long long pitch, int width, int height, int format, int kind, int stride, const double* cam, int point_filter_num,
                  double blind, int block, float* pts, int* pix) {
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
    const int ns = D.sw * D.sh, nb = (ns + block - 1) / block;
    std::vector<int> voff(nb + 1, 0), koff(nb + 1, 0);
    float p[3];
    for (int k = 0; k < ns; ++k) voff[k / block + 1] += depth_point(D, k, p) ? 1 : 0;   // k_depth_count
    for (int b = 0; b < nb; ++b) voff[b + 1] += voff[b];                                // scan
    for (int b = 0; b < nb; ++b) {                                                      // k_depth_keep
        int rank = 0;
        for (int k = b * block; k < ns && k < (b + 1) * block; ++k) {
            if (!depth_point(D, k, p)) continue;
            koff[b + 1] += depth_keep(voff[b] + rank++, p, point_filter_num, blind) ? 1 : 0;
        }
    }
    for (int b = 0; b < nb; ++b) koff[b + 1] += koff[b];                                // scan
    for (int b = 0; b < nb; ++b) {                                                      // k_depth_emit
        int vrank = 0, krank = 0;
        for (int k = b * block; k < ns && k < (b + 1) * block; ++k) {
            if (!depth_point(D, k, p)) continue;
            if (!depth_keep(voff[b] + vrank++, p, point_filter_num, blind)) continue;
            const int j = koff[b] + krank++;
            std::memcpy(pts + (size_t)j * 3, p, sizeof(p));
            pix[j] = (k / D.sw) * stride * width + (k % D.sw) * stride;
        }
    }
    return koff[nb];
}
}
