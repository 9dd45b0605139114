// Host emulation of immesh_mesh_evaluate: the shipped per-element bodies (immesh_b200/csrc/mesh_eval.cuh) in a plain sequential
// evaluator with a brute-force nearest-neighbour search, for small hand-built meshes and clouds.  The tiling, the grids and the ring
// search of the device are not emulated: their results do not depend on them by construction, and the GPU tests check that.
#include <cmath>
#include <map>
#include <tuple>
#include <vector>

#include "../../immesh_b200/csrc/mesh_eval.cuh"

using namespace immesh;

namespace {
// nearest target within md by the defined distance; md and far when there is none
double nearest(const float* q, const std::vector<float>& t, double md, bool* far) {
    double best = INFINITY;
    for (size_t j = 0; j < t.size() / 3; ++j) best = std::fmin(best, eval_dist(q[0], q[1], q[2], t[j * 3], t[j * 3 + 1], t[j * 3 + 2]));
    *far = !(best <= md);
    return *far ? md : best;
}
}  // namespace

// verts [nv][3]; tris [nt][3] live triangles as ascending id triples in ascending order; gt [ngt][3].
// Returns 0, or -5 (IMMESH_E_RANGE) for a triangle with more than 2^15 subdivisions, -1 for a non-finite ground-truth point.
// samples_out [counts[2]][4] (x, y, z, facet) when not null and cap_samples suffices.
extern "C" int emu_evaluate(const float* verts, const int* tris, int nt, const float* gt, long long ngt, double spacing, double leaf, double thr,
                            double md, double ratio, long long* counts, double* metrics, int* rows, float* samples_out, long long cap_samples,
                            float* gt_out, long long cap_gt) {
    for (long long i = 0; i < ngt * 3; ++i)
        if (!std::isfinite(gt[i])) return -1;
    // the ground truth: leaves in first-seen order, each summed in input order
    std::vector<float> g;
    if (leaf > 0) {
        std::map<std::tuple<long long, long long, long long>, size_t> slot;
        std::vector<double> sum;
        std::vector<long long> cnt;
        for (long long i = 0; i < ngt; ++i) {
            const float* p = gt + i * 3;
            const auto key = std::make_tuple(eval_leaf_key(p[0], leaf), eval_leaf_key(p[1], leaf), eval_leaf_key(p[2], leaf));
            auto it = slot.find(key);
            if (it == slot.end()) { it = slot.emplace(key, cnt.size()).first; cnt.push_back(0); sum.insert(sum.end(), {0.0, 0.0, 0.0}); }
            for (int c = 0; c < 3; ++c) sum[it->second * 3 + c] += (double)p[c];
            ++cnt[it->second];
        }
        for (size_t l = 0; l < cnt.size(); ++l)
            for (int c = 0; c < 3; ++c) g.push_back((float)(sum[l * 3 + c] / (double)cnt[l]));
    } else {
        g.assign(gt, gt + ngt * 3);
    }
    // the triangles: fairness and samples
    long long c[12] = {nt, 0, 0, (long long)(g.size() / 3), 0, 0, 0, 0, 0, 0, 0, 0};
    double smm = 0, sc2 = 0;
    std::vector<float> s;
    std::vector<int> sf;
    for (int t = 0; t < nt; ++t) {
        const float *A = verts + (size_t)tris[t * 3] * 3, *B = verts + (size_t)tris[t * 3 + 1] * 3, *C = verts + (size_t)tris[t * 3 + 2] * 3;
        const EvalTri e = eval_triangle(A, B, C);
        if (e.degenerate) { ++c[1]; continue; }
        smm += e.maxmin;
        sc2 += e.c2se;
        const int n = eval_subdivisions(e.longest, spacing);
        if (n == 0) return -5;
        if (n > c[11]) c[11] = n;
        for (long long k = 0; k < (long long)n * n; ++k) {
            float p[3];
            eval_sample(A, B, C, n, k, p);
            s.insert(s.end(), p, p + 3);
            sf.push_back(t);
        }
    }
    const long long ns = (long long)sf.size(), ng = c[3];
    c[2] = ns;
    std::vector<int> f_s(nt, 0), f_f(nt, 0);
    for (long long i = 0; i < ns; ++i) {
        bool far;
        const double d = nearest(&s[i * 3], g, md, &far);
        c[4] += d < thr;
        c[6] += far;
        c[9] += eval_quant(d);
        ++f_s[sf[i]];
        f_f[sf[i]] += !(d < thr);
    }
    for (long long i = 0; i < ng; ++i) {
        bool far;
        const double d = nearest(&g[i * 3], s, md, &far);
        c[5] += d < thr;
        c[7] += far;
        c[10] += eval_quant(d);
    }
    for (int t = 0; t < nt; ++t) {
        c[8] += f_s[t] > 0 && (double)f_f[t] >= ratio * (double)f_s[t];
        if (rows) {
            for (int k = 0; k < 3; ++k) rows[t * 5 + k] = tris[t * 3 + k];
            rows[t * 5 + 3] = f_s[t];
            rows[t * 5 + 4] = f_f[t];
        }
    }
    for (int i = 0; i < 12; ++i) counts[i] = c[i];
    eval_metrics(c, smm, sc2, metrics);
    if (samples_out && cap_samples >= ns)
        for (long long i = 0; i < ns; ++i) {
            for (int k = 0; k < 3; ++k) samples_out[i * 4 + k] = s[i * 3 + k];
            samples_out[i * 4 + 3] = (float)sf[i];
        }
    if (gt_out && cap_gt >= ng)
        for (long long i = 0; i < ng * 3; ++i) gt_out[i] = g[i];
    return 0;
}
