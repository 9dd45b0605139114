// immesh_b200 -- the textured mesh (immesh_mesh_texture_select, the paper's Application-2; the rule is stated in include/immesh_b200.h)
// and its OBJ / MTL export.  CUDA kernels (sm_90a, bodies in texture_core.cuh) and their C-ABI host orchestration.
//   Once: the live triangles in snapshot order (mesh_tri_order) and each slot's row (k_tex_init).  Per camera, in index order: the
// depth image's binning passes at the rule's positions (rf_bin_launch), one block per tile (k_tex_tile) that finds every pixel's
// winner with the view's tie-break, counts each facet's covered samples (per warp, per block, then one integer atomic per facet and
// tile) and its won pixels; then one thread per facet (k_tex_facet) applies the "seen" test and keeps the nearest camera with a strict
// <, and clears the counts for the next camera.  After the last camera, k_tex_rows writes the rows in snapshot order.
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "handles.hpp"
#include "texture_core.cuh"

using namespace immesh;

namespace {

// per live record (mesh_tri_order's rec index): this camera's counts, and the best camera so far with its distance and counts
struct TexFacets { int *won, *cov, *best_cam, *best_won, *best_cov; double* best_e2; };

__device__ __forceinline__ void tex_facet_corners(const MeshDev& M, int pos_mode, const int4& r, float4* q) {
    tex_corners(tex_vertex(M, pos_mode, r.x), tex_vertex(M, pos_mode, r.y), tex_vertex(M, pos_mode, r.z), (int)(M.tri_flip[r.w] & 1ull), q);
}

// each live slot's row, and the rows' state before the first camera
__global__ void __launch_bounds__(128) k_tex_init(const int4* rec, int n, int* row_of, TexFacets F) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        row_of[rec[e].w] = e;
        F.won[e] = 0; F.cov[e] = 0;
        F.best_cam[e] = -1; F.best_won[e] = 0; F.best_cov[e] = 0;
        F.best_e2[e] = INFINITY;
    }
}

// one thread per facet: camera k's "seen" test on the counts of k_tex_tile, the nearest camera kept with a strict <; the counts cleared
__global__ void __launch_bounds__(128) k_tex_facet(MeshDev M, int pos_mode, const DepthCam* cam, int k, TexRule rule, const int4* rec, int n, TexFacets F) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const int wn = F.won[e], cv = F.cov[e];
        if (wn == 0 && cv == 0) continue;   // tex_seen needs won >= 1; nothing to clear
        F.won[e] = 0; F.cov[e] = 0;
        if (wn < 1) continue;
        float4 q[3];
        tex_facet_corners(M, pos_mode, rec[e], q);
        double e2;
        if (tex_seen(*cam, q, wn, cv, rule, &e2) && e2 < F.best_e2[e]) {
            F.best_e2[e] = e2; F.best_cam[e] = k; F.best_won[e] = wn; F.best_cov[e] = cv;
        }
    }
}

// the rows in snapshot order: camera, texture coordinates (textured rows only), won / covered; counts [textured, untextured, cameras used]
__global__ void __launch_bounds__(128) k_tex_rows(MeshDev M, int pos_mode, const DepthCam* cams, const int4* rec, const unsigned int* order, int n, TexFacets F,
                                                  int* cam_out, float* uv_out, int* px_out, int* used, int* cnt) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int e = (int)order[i], k = F.best_cam[e];
        cam_out[i] = k;
        px_out[2 * (size_t)i] = k >= 0 ? F.best_won[e] : 0;
        px_out[2 * (size_t)i + 1] = k >= 0 ? F.best_cov[e] : 0;
        if (k < 0) { atomicAdd(&cnt[1], 1); continue; }
        float4 q[3];
        tex_facet_corners(M, pos_mode, rec[e], q);
        tex_uv(cams[k], q, uv_out + 6 * (size_t)i);
        atomicAdd(&cnt[0], 1);
        if (atomicExch(&used[k], 1) == 0) atomicAdd(&cnt[2], 1);
    }
}

// the positions the rule used, as floats
__global__ void __launch_bounds__(128) k_tex_vertices(MeshDev M, int pos_mode, int nv, float* out) {
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
        const float4 p = tex_vertex(M, pos_mode, v);
        out[3 * (size_t)v] = p.x; out[3 * (size_t)v + 1] = p.y; out[3 * (size_t)v + 2] = p.z;
    }
}

int tex_tiles(int w, int h) { return ((w + IM_RT_TILE - 1) / IM_RT_TILE) * ((h + IM_RT_TILE - 1) / IM_RT_TILE); }

}  // namespace

int immesh_mesh_texture_select(immesh_mesh_t* h, const immesh_texture_camera* cams, int n_cams, const immesh_texture_config* cfg, int32_t* facet_cam,
                               float* facet_uv, int32_t* facet_px, float* vertices, int64_t cap, int64_t* n_facets, int64_t* counts) {
    if (!h || !cams || !cfg || !n_facets || n_cams < 1 || cap < 0) return im_fail(IMMESH_E_INVALID, "texture_select: bad argument (NULL h, cams, cfg or n_facets; n_cams < 1; cap < 0)");
    if (!tex_config_ok(*cfg))
        return im_fail(IMMESH_E_INVALID, "texture_select: bad config (0 < z_near < z_far < inf; min_cos in [0, 1]; min_visible_permille in [0, 1000]; two_sided and positions 0 or 1)");
    for (int k = 0; k < n_cams; ++k)
        if (!tex_camera_ok(cams[k]))
            return im_fail(IMMESH_E_INVALID, ("texture_select: bad camera " + std::to_string(k) + " (1 <= width * height <= 2^26; finite intrinsics and pose; fx, fy != 0)").c_str());
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "texture_select: a sharded mesh handle is not supported");
    cudaStream_t st = h->stream;
    IM_CUDA(cudaStreamSynchronize(st));   // the frames already queued, the pipelined ones included
    int mc[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, mc));
    const int n = mc[IM_MC_TRIS_LIVE], nv = mc[IM_MC_VERTICES], nalloc = std::min(mc[IM_MC_TRIS_ALLOC], h->M.max_t);
    *n_facets = n;
    if (n > cap) return im_fail(IMMESH_E_CAPACITY, "texture_select: more live triangles than cap (*n_facets holds the number needed; nothing was written)");

    std::vector<DepthCam> hc(n_cams);
    long long pixels = 0;
    int max_tiles = 1;
    for (int k = 0; k < n_cams; ++k) {
        hc[k] = tex_camera(cams[k], cfg->z_near, cfg->z_far);
        pixels += (long long)cams[k].width * cams[k].height;
        max_tiles = std::max(max_tiles, tex_tiles(cams[k].width, cams[k].height));
    }
    const int pos = cfg->positions;
    const size_t n1 = (size_t)std::max(n, 1);
    MemSet mem;   // every buffer of the call, released on every return
    DepthCam* d_cams = nullptr;
    RfImage im;
    TriOrder o = {};
    TexFacets F = {};
    int *row_of = nullptr, *cam_out = nullptr, *px_out = nullptr, *used = nullptr, *cnt = nullptr;
    float *uv_out = nullptr, *v_out = nullptr;
    {
        cudaError_t e = cudaSuccess;
        auto add = [&e, &mem](auto** p, size_t count) { if (e == cudaSuccess) e = mem.alloc(p, std::max<size_t>(count, 1)); };
        add(&d_cams, (size_t)n_cams);
        if (n > 0) {
            im.ntiles = max_tiles;
            im.bin_cap = (int)std::min<long long>(INT_MAX, std::max<long long>({1LL << 22, 16LL * max_tiles, 8LL * nalloc}));
            add(&im.tile_cnt, (size_t)max_tiles); add(&im.tile_off, (size_t)max_tiles + 1); add(&im.bin, (size_t)im.bin_cap); add(&im.misc, 4);
            o.cap = n;
            add(&o.rec, n1);
            for (int b = 0; b < 2; ++b) { add(&o.k[b], n1); add(&o.v[b], n1); }
            add(&o.hist, mesh_sort_hist_ints(n1)); add(&o.misc, 8);
            add(&row_of, (size_t)nalloc);
            add(&F.won, n1); add(&F.cov, n1); add(&F.best_cam, n1); add(&F.best_won, n1); add(&F.best_cov, n1); add(&F.best_e2, n1);
            add(&cam_out, n1); add(&uv_out, n1 * 6); add(&px_out, n1 * 2);
        }
        add(&used, (size_t)n_cams); add(&cnt, 4);
        if (vertices) add(&v_out, (size_t)nv * 3);
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_select: allocation of the call's buffers failed");
    }
    IM_CUDA(cudaMemcpyAsync(d_cams, hc.data(), (size_t)n_cams * sizeof(DepthCam), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(used, 0, (size_t)n_cams * sizeof(int), st));
    IM_CUDA(cudaMemsetAsync(cnt, 0, 4 * sizeof(int), st));
    if (n > 0) {
        if (const int rc = mesh_tri_order(h, mc, 0.0, o)) return rc;
        IM_LAUNCH(k_tex_init, mesh_grid(h, n, 128), 128, 0, st, (const int4*)o.rec, n, row_of, F);
        const TexRule rule = tex_rule(*cfg);
        for (int k = 0; k < n_cams; ++k) {
            RfImage ik = im;
            ik.cam = d_cams + k;
            ik.ntiles = tex_tiles(cams[k].width, cams[k].height);
            IM_CUDA(cudaMemsetAsync(im.tile_cnt, 0, (size_t)ik.ntiles * sizeof(int), st));
            rf_bin_launch(h, ik, pos, st);
            IM_LAUNCH(k_tex_tile<TexRowOf>, ik.ntiles, IM_RT_THREADS, 0, st, h->M, pos, (const DepthCam*)ik.cam, (const int*)im.tile_off, (const int*)im.bin,
                      (const int*)im.misc, TexRowOf{row_of}, F.won, F.cov);
            IM_LAUNCH(k_tex_facet, mesh_grid(h, n, 128), 128, 0, st, h->M, pos, (const DepthCam*)ik.cam, k, rule, (const int4*)o.rec, n, F);
        }
        IM_LAUNCH(k_tex_rows, mesh_grid(h, n, 128), 128, 0, st, h->M, pos, (const DepthCam*)d_cams, (const int4*)o.rec, o.order, n, F, cam_out, uv_out, px_out, used, cnt);
    }
    if (vertices && nv > 0) IM_LAUNCH(k_tex_vertices, mesh_grid(h, nv, 128), 128, 0, st, h->M, pos, nv, v_out);
    IM_CUDA(cudaGetLastError());
    int hcnt[4] = {0, 0, 0, 0};
    std::vector<int32_t> hcam(n1);
    std::vector<float> huv;
    IM_CUDA(cudaMemcpyAsync(hcnt, cnt, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(hcam.data(), cam_out, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (facet_uv) {
            huv.resize((size_t)n * 6);
            IM_CUDA(cudaMemcpyAsync(huv.data(), uv_out, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
        if (facet_px) IM_CUDA(cudaMemcpyAsync(facet_px, px_out, (size_t)n * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    if (vertices && nv > 0) IM_CUDA(cudaMemcpyAsync(vertices, v_out, (size_t)nv * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (facet_cam && n > 0) std::memcpy(facet_cam, hcam.data(), (size_t)n * sizeof(int32_t));
    for (int i = 0; facet_uv && i < n; ++i)   // the rows of untextured facets are left as the caller had them
        if (hcam[i] >= 0) std::memcpy(facet_uv + 6 * (size_t)i, huv.data() + 6 * (size_t)i, 6 * sizeof(float));
    if (counts) {
        counts[0] = hcnt[0]; counts[1] = hcnt[1]; counts[2] = hcnt[2]; counts[3] = pixels;
    }
    return IMMESH_OK;
}

// The OBJ / MTL pair of a texture selection (the layout is stated in include/immesh_b200.h).  Host-side only.
int immesh_write_obj_textured(const char* obj_path, const char* mtl_path, const float* vertices, int nv, const int32_t* triangles, const int32_t* flips,
                              const int32_t* facet_cam, const float* facet_uv, int nt, const int32_t* cam_wh, const char* const* image_files, int n_cams) {
    if (!obj_path || !mtl_path || nv < 0 || nt < 0 || n_cams < 0 || (!vertices && nv > 0) || (nt > 0 && (!triangles || !facet_cam)) ||
        (n_cams > 0 && (!cam_wh || !image_files)))
        return im_fail(IMMESH_E_INVALID, "write_obj_textured: bad argument");
    for (int t = 0; t < nt * 3; ++t)
        if (triangles[t] < 0 || triangles[t] >= nv) return im_fail(IMMESH_E_RANGE, "write_obj_textured: a triangle refers to a vertex outside the vertex array");
    // the faces grouped by camera, ascending, the rows in order inside a group; the untextured group last
    std::vector<int> start(n_cams + 2, 0);
    for (int t = 0; t < nt; ++t) {
        const int k = facet_cam[t];
        if (k < -1 || k >= n_cams) return im_fail(IMMESH_E_INVALID, "write_obj_textured: facet_cam outside [-1, n_cams)");
        ++start[(k < 0 ? n_cams : k) + 1];
    }
    for (int k = 0; k < n_cams; ++k)
        if (start[k + 1] > 0 && (cam_wh[2 * k] < 1 || cam_wh[2 * k + 1] < 1 || !image_files[k] || !facet_uv))
            return im_fail(IMMESH_E_INVALID, "write_obj_textured: a used camera needs a size >= 1, an image file and facet_uv");
    for (int g = 0; g <= n_cams; ++g) start[g + 1] += start[g];
    std::vector<int> rows(nt);
    {
        std::vector<int> cur(start.begin(), start.end() - 1);
        for (int t = 0; t < nt; ++t) rows[cur[facet_cam[t] < 0 ? n_cams : facet_cam[t]]++] = t;
    }
    const char* slash = std::strrchr(mtl_path, '/');
    FILE* f = std::fopen(obj_path, "w");
    if (!f) return im_fail(IMMESH_E_INVALID, "write_obj_textured: cannot open the OBJ file");
    const int n_tex = start[n_cams];
    std::fprintf(f, "# immesh_b200 textured mesh: %d vertices, %d facets, %d textured\nmtllib %s\n", nv, nt, n_tex, slash ? slash + 1 : mtl_path);
    for (int v = 0; v < nv; ++v) std::fprintf(f, "v %.9g %.9g %.9g\n", vertices[3 * v], vertices[3 * v + 1], vertices[3 * v + 2]);
    for (int j = 0; j < n_tex; ++j) {   // the textured faces' coordinates in the order the faces are written
        const int t = rows[j], k = facet_cam[t];
        const double W = cam_wh[2 * k], H = cam_wh[2 * k + 1];
        for (int c = 0; c < 3; ++c)
            std::fprintf(f, "vt %.17g %.17g\n", ((double)facet_uv[6 * t + 2 * c] + 0.5) / W, 1.0 - ((double)facet_uv[6 * t + 2 * c + 1] + 0.5) / H);
    }
    for (int g = 0; g <= n_cams; ++g) {
        if (start[g + 1] == start[g]) continue;
        if (g < n_cams) std::fprintf(f, "usemtl tex_%d\n", g);
        else std::fprintf(f, "usemtl untextured\n");
        for (int j = start[g]; j < start[g + 1]; ++j) {
            const int t = rows[j];
            const int flip = flips && flips[t] != 0;
            const int a = triangles[3 * t] + 1, b = triangles[3 * t + 1] + 1, c = triangles[3 * t + 2] + 1;
            const int q[3] = {a, flip ? b : c, flip ? c : b};
            if (g < n_cams) std::fprintf(f, "f %d/%d %d/%d %d/%d\n", q[0], 3 * j + 1, q[1], 3 * j + 2, q[2], 3 * j + 3);
            else std::fprintf(f, "f %d %d %d\n", q[0], q[1], q[2]);
        }
    }
    if (std::fclose(f) != 0) return im_fail(IMMESH_E_INVALID, "write_obj_textured: writing the OBJ file failed");
    FILE* m = std::fopen(mtl_path, "w");
    if (!m) return im_fail(IMMESH_E_INVALID, "write_obj_textured: cannot open the MTL file");
    std::fprintf(m, "# immesh_b200 textured mesh materials\n");
    for (int k = 0; k < n_cams; ++k)
        if (start[k + 1] > start[k]) std::fprintf(m, "newmtl tex_%d\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd %s\n", k, image_files[k]);
    std::fprintf(m, "newmtl untextured\nKa 0.5 0.5 0.5\nKd 0.5 0.5 0.5\nKs 0 0 0\nillum 1\n");
    if (std::fclose(m) != 0) return im_fail(IMMESH_E_INVALID, "write_obj_textured: writing the MTL file failed");
    return IMMESH_OK;
}
