// immesh_b200 -- the per-element bodies of immesh_mesh_evaluate (eval_capi.cu): the fairness terms of a triangle, its sub-triangle
// samples, the ground-truth leaf key and the defined distance with its quantisation.  IM_HD, so that the host emulation (tests/eval)
// runs the same code.  Every rule is stated in include/immesh_b200.h at immesh_mesh_evaluate.  Built with -fmad=false (device) and
// -ffp-contract=off (host): no FMA contraction anywhere.
#pragma once
#include <cmath>
#include <cstdint>

#include "hd_math.cuh"

namespace immesh {

constexpr int IM_EVAL_MAX_N = 1 << 15;            // subdivisions of one triangle
constexpr double IM_EVAL_QSCALE = 1048576.0;      // 2^20: distance quantum of the order-free sums
constexpr double IM_EVAL_PI = 3.14159265358979323846;

IM_HD double eval_norm3(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

// the defined distance: float32 coordinates, float64 arithmetic, sqrt((dx dx + dy dy) + dz dz)
IM_HD double eval_dist(float ax, float ay, float az, float bx, float by, float bz) {
    return eval_norm3((double)ax - (double)bx, (double)ay - (double)by, (double)az - (double)bz);
}
// q = rint(d 2^20) (ties to even)
IM_HD long long eval_quant(double d) { return (long long)rint(d * IM_EVAL_QSCALE); }

// ground-truth leaf key of one coordinate: floor((double)p / leaf)
IM_HD long long eval_leaf_key(float p, double leaf) { return (long long)floor((double)p / leaf); }

// angle between u and v in degrees: atan2(|u x v|, u . v)
IM_HD double eval_angle_deg(const double* u, const double* v) {
    const double cx = u[1] * v[2] - u[2] * v[1], cy = u[2] * v[0] - u[0] * v[2], cz = u[0] * v[1] - u[1] * v[0];
    const double dot = (u[0] * v[0] + u[1] * v[1]) + u[2] * v[2];
    return atan2(eval_norm3(cx, cy, cz), dot) * (180.0 / IM_EVAL_PI);
}

struct EvalTri {
    double maxmin;    // max - min interior angle (degrees)
    double c2se;      // circumradius / shortest edge
    double longest;   // longest edge (m)
    int degenerate;   // |AB x AC| == 0 in float64: no fairness terms, no samples
};

// fairness of the triangle (A, B, C), all in float64 from the float32 positions
IM_HD EvalTri eval_triangle(const float* A, const float* B, const float* C) {
    double ab[3], ac[3], bc[3], ba[3], ca[3], cb[3];
    for (int k = 0; k < 3; ++k) {
        ab[k] = (double)B[k] - (double)A[k]; ac[k] = (double)C[k] - (double)A[k]; bc[k] = (double)C[k] - (double)B[k];
        ba[k] = -ab[k]; ca[k] = -ac[k]; cb[k] = -bc[k];
    }
    EvalTri r;
    const double lab = eval_norm3(ab[0], ab[1], ab[2]), lac = eval_norm3(ac[0], ac[1], ac[2]), lbc = eval_norm3(bc[0], bc[1], bc[2]);
    r.longest = fmax(lab, fmax(lac, lbc));
    const double cx = ab[1] * ac[2] - ab[2] * ac[1], cy = ab[2] * ac[0] - ab[0] * ac[2], cz = ab[0] * ac[1] - ab[1] * ac[0];
    const double cross = eval_norm3(cx, cy, cz);
    r.degenerate = cross == 0.0;
    if (r.degenerate) { r.maxmin = 0; r.c2se = 0; return r; }
    const double a0 = eval_angle_deg(ab, ac), a1 = eval_angle_deg(bc, ba), a2 = eval_angle_deg(ca, cb);
    r.maxmin = fmax(a0, fmax(a1, a2)) - fmin(a0, fmin(a1, a2));
    r.c2se = ((lbc * lac) * lab) / (2.0 * cross) / fmin(lab, fmin(lac, lbc));
    return r;
}

// subdivisions of a triangle: n = max(1, ceil(longest / spacing)); 0 when n would exceed IM_EVAL_MAX_N
IM_HD int eval_subdivisions(double longest, double spacing) {
    const double n = ceil(longest / spacing);
    if (!(n <= (double)IM_EVAL_MAX_N)) return 0;
    return n < 1.0 ? 1 : (int)n;
}

// entries before row i of a triangular array whose row r holds m - r entries
IM_HD long long eval_row_start(long long i, long long m) { return i * m - i * (i - 1) / 2; }
// the row of entry k (0 <= k < m (m + 1) / 2) of that array
IM_HD long long eval_row_of(long long k, long long m) {
    const double b = 2.0 * (double)m + 1.0;
    long long i = (long long)((b - sqrt(b * b - 8.0 * (double)k)) * 0.5);
    if (i < 0) i = 0;
    if (i > m - 1) i = m - 1;
    while (i > 0 && eval_row_start(i, m) > k) --i;
    while (i + 1 < m && eval_row_start(i + 1, m) <= k) ++i;
    return i;
}

// sample k in [0, n^2) of the n-subdivision: the n (n + 1) / 2 "up" sub-triangles (i in [0, n), j in [0, n - i)) row by row, then the
// n (n - 1) / 2 "down" ones (j in [0, n - i - 1)); barycentrics ((3i + 1) / 3n, (3j + 1) / 3n), down (3i + 2, 3j + 2);
// sample = (float)(A + (u (B - A) + v (C - A))) in float64
IM_HD void eval_sample(const float* A, const float* B, const float* C, int n, long long k, float* out) {
    const long long up = (long long)n * (n + 1) / 2;
    const int down = k >= up;
    const long long m = down ? n - 1 : n, kk = down ? k - up : k;
    const long long i = eval_row_of(kk, m), j = kk - eval_row_start(i, m);
    const double den = 3.0 * (double)n;
    const double u = (3.0 * (double)i + (down ? 2.0 : 1.0)) / den, v = (3.0 * (double)j + (down ? 2.0 : 1.0)) / den;
    for (int c = 0; c < 3; ++c) {
        const double a = (double)A[c];
        out[c] = (float)(a + (u * ((double)B[c] - a) + v * ((double)C[c] - a)));
    }
}

// metrics[8] from counts[12] (the layout of immesh_mesh_evaluate) and the two fairness sums over the non-degenerate triangles
IM_HD void eval_metrics(const long long* c, double sum_maxmin, double sum_c2se, double* m) {
    const double nan = NAN, nf = (double)(c[0] - c[1]);
    const double p = c[2] ? (double)c[4] / (double)c[2] : nan, r = c[3] ? (double)c[5] / (double)c[3] : nan;
    m[0] = c[0] > c[1] ? sum_maxmin / nf : nan;
    m[1] = c[0] > c[1] ? sum_c2se / nf : nan;
    m[2] = c[2] ? (double)c[9] / IM_EVAL_QSCALE / (double)c[2] : nan;
    m[3] = c[3] ? (double)c[10] / IM_EVAL_QSCALE / (double)c[3] : nan;
    m[4] = p;
    m[5] = r;
    m[6] = (c[2] && c[3]) ? (p + r > 0 ? 2 * p * r / (p + r) : 0.0) : nan;
    m[7] = 0.0;
}

}  // namespace immesh
