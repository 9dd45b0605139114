// immesh_b200 -- colour equalisation between cameras (immesh_mesh_texture_gains, immesh_texture_apply_gains, texture_gains.cu; the rule
// is stated in include/immesh_b200.h): the sample points, the nearest-pixel sample, the clipping test, one row of pair sums and the
// corrected channel value.  __host__ __device__ bodies shared by the kernels and the host emulation of the tests; float64 in the written
// order (built with -fmad=false on the device and -ffp-contract=off on the host).  Also the call's argument check and the host solve
// (normal equations and Jacobi-preconditioned CG), shared with the emulation so that both refuse the same inputs and solve alike.
#pragma once
#include <climits>
#include <cmath>
#include <string>
#include <vector>

#include "texture_bake_core.cuh"
#include "texture_core.cuh"

namespace immesh {

#define IM_TG_POINTS 10   // sample points per facet
#define IM_TG_SUMS 7      // a pair's sums: n, S_k[3], S_c[3]

// rule 1: sample point s (0..9) as integer barycentrics (i, j, l) / 6, i = 1..4, j = 1..5 - i, l = 6 - i - j
IM_HD void tg_point(int s, double* b) {
    int i = 1, j = 1;
    for (int r = 0; r < s; ++r) {
        if (j < 5 - i) ++j;
        else { ++i; j = 1; }
    }
    b[0] = (double)i / 6.0;
    b[1] = (double)j / 6.0;
    b[2] = (double)(6 - i - j) / 6.0;
}

// rules 1-2: the 10 nearest-pixel RGB samples (out [30]) of image I at scaled corners p (bake_scaled, face order)
IM_HD void tg_sample(const BakeImg& I, const double* p, unsigned char* out) {
    const double xm = (double)(I.w - 1), ym = (double)(I.h - 1);
    for (int s = 0; s < IM_TG_POINTS; ++s) {
        double b[3];
        tg_point(s, b);
        double x = floor(((b[0] * p[0] + b[1] * p[2]) + b[2] * p[4]) + 0.5), y = floor(((b[0] * p[1] + b[1] * p[3]) + b[2] * p[5]) + 0.5);
        x = x < 0.0 ? 0.0 : (x > xm ? xm : x);
        y = y < 0.0 ? 0.0 : (y > ym ? ym : y);
        const unsigned char* px = I.data + (long long)y * I.pitch + 3LL * (long long)x;
        out[3 * s] = px[0]; out[3 * s + 1] = px[1]; out[3 * s + 2] = px[2];
    }
}

// rules 4-5: the observer's samples ok [30] against the chosen side's oc [30]: kept sample pairs added into
// sum [7] (n, S_k[3], S_c[3]), dropped ones counted in *clipped
IM_HD void tg_accumulate(const unsigned char* ok, const unsigned char* oc, int* sum, int* clipped) {
    for (int s = 0; s < IM_TG_POINTS; ++s) {
        bool clip = false;
        for (int ch = 0; ch < 3; ++ch) {
            const int a = ok[3 * s + ch], b = oc[3 * s + ch];
            clip = clip || a == 0 || a == 255 || b == 0 || b == 255;
        }
        if (clip) { ++*clipped; continue; }
        ++sum[0];
        for (int ch = 0; ch < 3; ++ch) { sum[1 + ch] += ok[3 * s + ch]; sum[4 + ch] += oc[3 * s + ch]; }
    }
}

// immesh_texture_apply_gains: min(255, floor(v g + 0.5))
IM_HD unsigned char tg_apply(unsigned char v, double g) {
    const double x = floor((double)v * g + 0.5);
    return x >= 255.0 ? (unsigned char)255 : (unsigned char)x;
}

// ---- host code
// the argument check of immesh_mesh_texture_gains (n_live: the live triangle count; shard_n: the handle's shards): an empty string when
// the call may proceed, else the reason.  have [n_cams]: 1 for a camera with an image.
inline std::string tg_check(const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device, const int32_t* facet_cam,
                            const float* facet_uv, int64_t n_facets, const immesh_texture_gains_config* cfg, const double* gains, int64_t n_live, int shard_n,
                            std::vector<unsigned char>& have) {
    if (!cams || !images || !cfg || !gains || n_cams < 1 || n_facets < 0 || n_facets > INT_MAX || (n_facets > 0 && (!facet_cam || !facet_uv)) ||
        (on_device != 0 && on_device != 1))
        return "bad argument (NULL cams, images, cfg or gains; n_cams < 1; n_facets outside [0, 2^31) or rows NULL; on_device not 0 / 1)";
    if (!tex_config_ok(cfg->sel))
        return "bad select rule (0 < z_near < z_far < inf; min_cos in [0, 1]; min_visible_permille in [0, 1000]; two_sided and positions 0 or 1)";
    if (!std::isfinite(cfg->sigma_n) || !(cfg->sigma_n > 0.0) || !std::isfinite(cfg->sigma_g) || !(cfg->sigma_g > 0.0) || cfg->max_pairs < 1 ||
        cfg->max_image_bytes < 0)
        return "bad config (sigma_n and sigma_g finite and > 0; max_pairs >= 1; max_image_bytes >= 0)";
    if (shard_n > 1) return "a sharded mesh handle is not supported";
    if (n_facets != n_live) return "n_facets (" + std::to_string(n_facets) + ") is not the live triangle count (" + std::to_string(n_live) + ")";
    long long n_tex = 0;
    std::vector<unsigned char> used;
    std::string why = bake_check_rows(n_cams, facet_cam, facet_uv, n_facets, &n_tex, used);
    if (!why.empty()) return why;
    have.assign((size_t)n_cams, 0);
    for (int k = 0; k < n_cams; ++k) {
        if (!images[k].data) {
            if (used[k]) return "camera " + std::to_string(k) + " textures a row: it needs an image";
            continue;
        }
        why = bake_check_image(cams, images, on_device, bake_arena_bytes(cfg->max_image_bytes), k);
        if (!why.empty()) return why;
        if (!tex_camera_ok(cams[k])) return "bad camera " + std::to_string(k) + " (1 <= width * height <= 2^26; finite intrinsics and pose; fx, fy != 0)";
        have[k] = 1;
    }
    return std::string();
}

// rules 6-7: the gains [n_cams][3] of the pairs (cam [n_pairs][2], sums [n_pairs][7]); *iters: the most CG iterations over the
// channels; *left: the cameras in no pair (gain 1)
inline void tg_solve(int n_cams, const int* cam, const long long* sums, long long n_pairs, double sigma_n, double sigma_g, double* gains, int* iters,
                     int* left) {
    const double sn2 = sigma_n * sigma_n, sg2 = sigma_g * sigma_g;
    const size_t K = (size_t)n_cams;
    std::vector<unsigned char> in(K, 0);
    for (long long p = 0; p < n_pairs; ++p) { in[cam[2 * p]] = 1; in[cam[2 * p + 1]] = 1; }
    *left = 0;
    for (size_t k = 0; k < K; ++k) *left += in[k] ? 0 : 1;
    *iters = 0;
    const int max_it = std::max(100, 2 * n_cams);
    std::vector<double> d(K), rhs(K), off((size_t)n_pairs), g(K), r(K), z(K), pv(K), q(K);
    auto apply = [&](const std::vector<double>& x, std::vector<double>& y) {
        for (size_t k = 0; k < K; ++k) y[k] = d[k] * x[k];
        for (long long p = 0; p < n_pairs; ++p) {
            const int a = cam[2 * p], b = cam[2 * p + 1];
            y[a] += off[p] * x[b];
            y[b] += off[p] * x[a];
        }
    };
    auto dot = [&](const std::vector<double>& x, const std::vector<double>& y) {
        double s = 0.0;
        for (size_t k = 0; k < K; ++k) s += x[k] * y[k];
        return s;
    };
    for (int ch = 0; ch < 3; ++ch) {
        for (size_t k = 0; k < K; ++k) { d[k] = in[k] ? 0.0 : 1.0; rhs[k] = in[k] ? 0.0 : 1.0; }
        for (long long p = 0; p < n_pairs; ++p) {
            const int a = cam[2 * p], b = cam[2 * p + 1];
            const long long* s = sums + IM_TG_SUMS * p;
            const double n = (double)s[0], Sa = (double)s[1 + ch], Sb = (double)s[4 + ch];
            d[a] += (Sa * Sa / n) / sn2 + n / sg2;
            d[b] += (Sb * Sb / n) / sn2 + n / sg2;
            off[p] = -((Sa * Sb / n) / sn2);
            rhs[a] += n / sg2;
            rhs[b] += n / sg2;
        }
        for (size_t k = 0; k < K; ++k) g[k] = 1.0;
        apply(g, q);
        for (size_t k = 0; k < K; ++k) { r[k] = rhs[k] - q[k]; z[k] = r[k] / d[k]; pv[k] = z[k]; }
        const double stop = 1e-12 * std::sqrt(dot(rhs, rhs));
        double rz = dot(r, z);
        int it = 0;
        while (std::sqrt(dot(r, r)) > stop && it < max_it) {
            apply(pv, q);
            const double alpha = rz / dot(pv, q);
            for (size_t k = 0; k < K; ++k) { g[k] += alpha * pv[k]; r[k] -= alpha * q[k]; }
            ++it;
            for (size_t k = 0; k < K; ++k) z[k] = r[k] / d[k];
            const double rz2 = dot(r, z), beta = rz2 / rz;
            rz = rz2;
            for (size_t k = 0; k < K; ++k) pv[k] = z[k] + beta * pv[k];
        }
        *iters = std::max(*iters, it);
        for (size_t k = 0; k < K; ++k) gains[3 * k + ch] = g[k];
    }
}

// the argument check of immesh_texture_apply_gains (everything but h)
inline std::string tg_apply_check(const immesh_texture_image* in, const immesh_texture_image* out, int n, int on_device, const double* gains) {
    if (!in || !out || !gains || n < 0 || (on_device != 0 && on_device != 1)) return "bad argument (NULL in, out or gains; n < 0; on_device not 0 / 1)";
    for (int k = 0; k < n; ++k) {
        if (!in[k].data) continue;
        const immesh_texture_image &a = in[k], &b = out[k];
        if (!b.data || a.width < 1 || a.height < 1 || a.width != b.width || a.height != b.height || a.pitch < 3LL * a.width || b.pitch < 3LL * b.width)
            return "image " + std::to_string(k) + ": out needs data, sizes >= 1 equal to in's and pitches >= 3 width";
        for (int ch = 0; ch < 3; ++ch)
            if (!std::isfinite(gains[3 * k + ch]) || !(gains[3 * k + ch] >= 0.0)) return "gain of image " + std::to_string(k) + " not finite or < 0";
    }
    return std::string();
}

}  // namespace immesh
