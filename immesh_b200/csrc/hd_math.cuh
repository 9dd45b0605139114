// immesh_b200 -- scalar math used by every kernel on the localization + meshing path.
//
// Numerical contract (DESIGN.md "Numerics"): IEEE binary32/binary64, round-to-nearest-even,
// NO fused multiply-add (the library is built with -fmad=false; the reference builds with
// -O3 -msse2 and no -mfma, /root/reference/CMakeLists.txt:14), sums evaluated left to right
// exactly as written.  sin/cos/exp/acos are arithmetic-only so that results do not depend on
// the libm in use.  Everything here is __host__ __device__: the same source is compiled into
// the CUDA library and into the host-emulation harness used by the CPU-only logic tests.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define IM_HD __host__ __device__ __forceinline__
#define IM_HDN __host__ __device__
#else
#define IM_HD inline
#define IM_HDN
#endif

// Latency budget of a kernel, measured in place (debug variant of the library only: tools/debug/build_stamps.sh, -DIM_DEBUG_STAMPS):
// thread 0 of block 0 -- for the IESKF update, thread 0 of whichever block runs it -- stores clock64 at phase boundaries; `dep` is a value
// the phase before produced, so that the stamp is not taken before that value exists.  Empty in the product build and on the host.
#if defined(IM_DEBUG_STAMPS) && defined(__CUDACC__)
namespace immesh { static __device__ long long g_stamps[64]; }
#endif
#if defined(IM_DEBUG_STAMPS) && defined(__CUDA_ARCH__)
__device__ __forceinline__ void immesh_stamp_store(int k, long long v) { immesh::g_stamps[k] = v; }
#define IM_STAMP_IF(cond, k, dep) do { if ((cond) && (long long)(dep) != 0x7ffffffffffffLL) immesh::g_stamps[k] = clock64(); } while (0)
#define IM_STAMP(k, dep) IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0, k, dep)
#else
#define IM_STAMP_IF(cond, k, dep) do { } while (0)
#define IM_STAMP(k, dep) do { } while (0)
#endif

namespace immesh {

// ------------------------------------------------------------------ deterministic libm subset
IM_HD double im_rint(double x) {
#if defined(__CUDA_ARCH__)
    return rint(x);
#else
    return std::nearbyint(x);
#endif
}
IM_HD long long im_llrint(double x) {
#if defined(__CUDA_ARCH__)
    return __double2ll_rn(x);
#else
    return std::llrint(x);
#endif
}

IM_HD double sin_poly(double r) {  // |r| <= pi/4
    const double z = r * r;
    double p = -1.0 / 51090942171709440000.0;
    p = p * z + 1.0 / 121645100408832000.0;
    p = p * z - 1.0 / 355687428096000.0;
    p = p * z + 1.0 / 1307674368000.0;
    p = p * z - 1.0 / 6227020800.0;
    p = p * z + 1.0 / 39916800.0;
    p = p * z - 1.0 / 362880.0;
    p = p * z + 1.0 / 5040.0;
    p = p * z - 1.0 / 120.0;
    p = p * z + 1.0 / 6.0;
    return r - (r * z) * p;
}
IM_HD double cos_poly(double r) {
    const double z = r * r;
    double p = 1.0 / 2432902008176640000.0;
    p = p * z - 1.0 / 6402373705728000.0;
    p = p * z + 1.0 / 20922789888000.0;
    p = p * z - 1.0 / 87178291200.0;
    p = p * z + 1.0 / 479001600.0;
    p = p * z - 1.0 / 3628800.0;
    p = p * z + 1.0 / 40320.0;
    p = p * z - 1.0 / 720.0;
    p = p * z + 1.0 / 24.0;
    p = p * z - 1.0 / 2.0;
    return 1.0 + z * p;
}
IM_HD void im_sincos(double x, double* s, double* c) {
    const double kf = im_rint(x * 6.36619772367581382433e-01);
    const double r = (x - kf * 1.57079632673412561417e+00) - kf * 6.07710050650619224932e-11;
    const long long k = (long long)kf;
    const double sk = sin_poly(r), ck = cos_poly(r);
    switch ((int)(k & 3)) {
        case 0: *s = sk; *c = ck; break;
        case 1: *s = ck; *c = -sk; break;
        case 2: *s = -sk; *c = -ck; break;
        default: *s = -ck; *c = sk; break;
    }
}
IM_HD double im_sin(double x) { double s, c; im_sincos(x, &s, &c); return s; }

// exp(x), x <= 0
IM_HD double im_exp(double x) {
    if (!(x > -700.0)) return 0.0;
    const double kf = im_rint(x * 1.44269504088896338700e+00);
    const double r = (x - kf * 6.93147180369123816490e-01) - kf * 1.90821492927058770002e-10;
    double p = 1.0 / 87178291200.0;
    p = p * r + 1.0 / 6227020800.0;
    p = p * r + 1.0 / 479001600.0;
    p = p * r + 1.0 / 39916800.0;
    p = p * r + 1.0 / 3628800.0;
    p = p * r + 1.0 / 362880.0;
    p = p * r + 1.0 / 40320.0;
    p = p * r + 1.0 / 5040.0;
    p = p * r + 1.0 / 720.0;
    p = p * r + 1.0 / 120.0;
    p = p * r + 1.0 / 24.0;
    p = p * r + 1.0 / 6.0;
    p = p * r + 0.5;
    p = p * r + 1.0;
    p = p * r + 1.0;
    return ldexp(p, (int)kf);
}
IM_HD double asin_series(double s) {  // |s| <= 0.5
    const double z = s * s;
    double term = s, sum = s, c = 1.0;
    for (int k = 0; k < 40; ++k) {
        const double a = (double)(2 * k + 1);
        c = c * (a * a) / ((double)(2 * k + 2) * (double)(2 * k + 3));
        term = term * z;
        const double add = c * term;
        sum = sum + add;
        if (fabs(add) < 1e-19 * fabs(sum)) break;
    }
    return sum;
}
IM_HD double im_acos(double x) {
    if (x >= 1.0) return 0.0;
    if (x <= -1.0) return 3.14159265358979311600e+00;
    if (x > 0.5) return 2.0 * asin_series(sqrt((1.0 - x) * 0.5));
    if (x < -0.5) return 3.14159265358979311600e+00 - 2.0 * asin_series(sqrt((1.0 + x) * 0.5));
    return (1.57079632673412561417e+00 - asin_series(x)) + 6.07710050650619224932e-11;
}

// asin on [-1, 1] and atan2 (through asin on |argument| <= 0.7072), arithmetic only like the functions above
IM_HD double im_asin(double x) {
    const double ax = fabs(x);
    double r;
    if (ax <= 0.5) r = asin_series(ax);
    else r = (1.57079632673412561417e+00 - 2.0 * asin_series(sqrt((1.0 - ax) * 0.5))) + 6.07710050650619224932e-11;
    return x < 0 ? -r : r;
}
IM_HD double im_atan2(double y, double x) {
    if (x == 0.0 && y == 0.0) return 0.0;
    const double r = sqrt(x * x + y * y);
    const double kPi = 3.14159265358979311600e+00, kPio2 = 1.57079632679489655800e+00;
    if (fabs(x) >= fabs(y)) {
        const double a = im_asin(y / r);
        if (x > 0) return a;
        return (y >= 0 ? kPi : -kPi) - a;
    }
    const double a = im_asin(x / r);
    return y > 0 ? (kPio2 - a) : (a - kPio2);
}
// KITTI laser calibration of one point (voxel_mapping.cpp:1844-1859, preprocess/calib_laser): the vertical angle of every return
// is raised by 0.15 degrees.  float fields like PointType; range and the horizon angle go through float as in the reference
// (std::sqrt / std::atan2 on float arguments under `using namespace std`, include/common_lib.h:23).
IM_HD void kitti_calib_point(float* x, float* y, float* z) {
    const float fx = *x, fy = *y, fz = *z;
    const double range = (double)sqrtf((fx * fx + fy * fy) + fz * fz);
    const double calib_vertical_angle = 0.15 * 3.14159265358 / 180.0;   // deg2rad(0.15) with PI_M (common_lib.h:34,297-300)
    const double vertical_angle = im_asin((double)fz / range) + calib_vertical_angle;
    const double horizon_angle = (double)(float)im_atan2((double)fy, (double)fx);
    double sv, cv, sh, ch;
    im_sincos(vertical_angle, &sv, &cv);
    im_sincos(horizon_angle, &sh, &ch);
    *z = (float)(range * sv);
    const double project_len = range * cv;
    *x = (float)(project_len * ch);
    *y = (float)(project_len * sh);
}

// ------------------------------------------------------------------ small dense helpers (row-major 3x3)
IM_HD void m3_mul(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C[i * 3 + j] = (A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j]) + A[i * 3 + 2] * B[2 * 3 + j];
}
IM_HD void m3_mul_bt(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C[i * 3 + j] = (A[i * 3 + 0] * B[j * 3 + 0] + A[i * 3 + 1] * B[j * 3 + 1]) + A[i * 3 + 2] * B[j * 3 + 2];
}
IM_HD void m3_vec(const double* A, const double* v, double* o) {
#pragma unroll
    for (int i = 0; i < 3; ++i) o[i] = (A[i * 3 + 0] * v[0] + A[i * 3 + 1] * v[1]) + A[i * 3 + 2] * v[2];
}
IM_HD void skew3(const double* v, double* K) {
    K[0] = 0.0; K[1] = -v[2]; K[2] = v[1];
    K[3] = v[2]; K[4] = 0.0; K[5] = -v[0];
    K[6] = -v[1]; K[7] = v[0]; K[8] = 0.0;
}
IM_HD double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// symmetric 3x3 packed as [00,01,02,11,12,22]
IM_HD int s6(int i, int j) {
    const int a = i < j ? i : j, b = i < j ? j : i;
    return a * 3 - (a * (a - 1)) / 2 + (b - a);
}
IM_HD void s6_full(const double* s, double* M) {
    M[0] = s[0]; M[1] = s[1]; M[2] = s[2];
    M[3] = s[1]; M[4] = s[3]; M[5] = s[4];
    M[6] = s[2]; M[7] = s[4]; M[8] = s[5];
}
// out6 = upper triangle of A * B * A^T
IM_HD void congr6(const double* A, const double* Bfull, double* out6) {
    double T[9];
    m3_mul(A, Bfull, T);
    out6[0] = (T[0] * A[0] + T[1] * A[1]) + T[2] * A[2];
    out6[1] = (T[0] * A[3] + T[1] * A[4]) + T[2] * A[5];
    out6[2] = (T[0] * A[6] + T[1] * A[7]) + T[2] * A[8];
    out6[3] = (T[3] * A[3] + T[4] * A[4]) + T[5] * A[5];
    out6[4] = (T[3] * A[6] + T[4] * A[7]) + T[5] * A[8];
    out6[5] = (T[6] * A[6] + T[7] * A[7]) + T[8] * A[8];
}
// n^T V n for symmetric packed V
IM_HD double quad6(const double* n, const double* v) {
    const double r0 = (v[0] * n[0] + v[1] * n[1]) + v[2] * n[2];
    const double r1 = (v[1] * n[0] + v[3] * n[1]) + v[4] * n[2];
    const double r2 = (v[2] * n[0] + v[4] * n[1]) + v[5] * n[2];
    double acc = 0.0;
    acc = acc + n[0] * r0;
    acc = acc + n[1] * r1;
    acc = acc + n[2] * r2;
    return acc;
}
// upper-triangular 6x6 index (i <= j), 21 entries
IM_HD int u21(int i, int j) { return i * 6 - (i * (i - 1)) / 2 + (j - i); }

// SO(3) exponential / logarithm with the reference's thresholds (include/so3_math.h:54-81)
IM_HD void so3_exp3(double v1, double v2, double v3, double* R) {
    const double n = sqrt((v1 * v1 + v2 * v2) + v3 * v3);
    R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    if (n > 0.00001) {
        const double r[3] = {v1 / n, v2 / n, v3 / n};
        double K[9], KK[9];
        skew3(r, K);
        m3_mul(K, K, KK);
        double s, c;
        im_sincos(n, &s, &c);
        const double omc = 1.0 - c;
        for (int i = 0; i < 9; ++i) R[i] = (R[i] + s * K[i]) + omc * KK[i];
    }
}
IM_HD void so3_exp_dt(const double* w, double dt, double* R) {  // so3_math.h:31-51
    const double n = sqrt(dot3(w, w));
    R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    if (n > 0.0000001) {
        const double r[3] = {w[0] / n, w[1] / n, w[2] / n};
        double K[9], KK[9];
        skew3(r, K);
        m3_mul(K, K, KK);
        double s, c;
        im_sincos(n * dt, &s, &c);
        const double omc = 1.0 - c;
        for (int i = 0; i < 9; ++i) R[i] = (R[i] + s * K[i]) + omc * KK[i];
    }
}
IM_HD void so3_log3(const double* R, double* out) {
    const double tr = (R[0] + R[4]) + R[8];
    const double theta = (tr > 3.0 - 1e-6) ? 0.0 : im_acos(0.5 * (tr - 1.0));
    const double K[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    if (fabs(theta) < 0.001) {
        for (int i = 0; i < 3; ++i) out[i] = 0.5 * K[i];
    } else {
        const double f = 0.5 * theta / im_sin(theta);
        for (int i = 0; i < 3; ++i) out[i] = f * K[i];
    }
}

// Cyclic Jacobi eigen-decomposition of a symmetric 3x3 (packed in), eigenvalues d[3], eigenvectors in the
// columns of V (row-major), unsorted.  Replaces Eigen::EigenSolver / SelfAdjointEigenSolver on the path
// (voxel_loc.cpp:62, mesh_rec_geometry.cpp:199).
// One rotation, pair (p,q) = (0,1), (0,2), (1,2) for PQ = 0, 1, 2; the pair is a template parameter so that every index into the
// packed matrix and the eigenvector array is a constant: with a run-time pair the arrays lived in local memory and each rotation paid a
// dozen dependent local loads/stores on top of its 4 divisions and 2 square roots.
template <int PQ>
IM_HD void jacobi3_rotate(int sweep, double (&a)[6], double (&v)[9]) {
    constexpr int p = (PQ == 2) ? 1 : 0, q = (PQ == 0) ? 1 : 2;
    constexpr int ipp = (PQ == 2) ? 3 : 0, iqq = (PQ == 0) ? 3 : 5, ipq = (PQ == 0) ? 1 : (PQ == 1) ? 2 : 4;
    constexpr int irp = (PQ == 0) ? 2 : 1, irq = (PQ == 2) ? 2 : 4;   // the two off-diagonal entries that share an index with (p,q)
    double app = a[ipp], aqq = a[iqq], apq = a[ipq], arp = a[irp], arq = a[irq];
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq);
    bool zero_only = false;
    double t = 0.0;
    if (sweep > 3 && (fabs(app) + g == fabs(app)) && (fabs(aqq) + g == fabs(aqq))) {
        zero_only = true;
    } else {
        const double h = aqq - app;
        if (fabs(h) + g == fabs(h)) {
            t = apq / h;
        } else {
            const double theta = 0.5 * h / apq;
            t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
            if (theta < 0.0) t = -t;
        }
    }
    if (zero_only) {
        apq = 0.0;
    } else {
        const double c = 1.0 / sqrt(1.0 + t * t);
        const double s = t * c;
        const double tau = s / (1.0 + c);
        const double hh = t * apq;
        app = app - hh;
        aqq = aqq + hh;
        apq = 0.0;
        const double nrp = arp - s * (arq + arp * tau);
        const double nrq = arq + s * (arp - arq * tau);
        arp = nrp;
        arq = nrq;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double vkp = v[k * 3 + p], vkq = v[k * 3 + q];
            v[k * 3 + p] = vkp - s * (vkq + vkp * tau);
            v[k * 3 + q] = vkq + s * (vkp - vkq * tau);
        }
    }
    a[ipp] = app; a[iqq] = aqq; a[ipq] = apq; a[irp] = arp; a[irq] = arq;
}
IM_HD void jacobi3(const double* a6, double* d, double* V) {
    double a[6] = {a6[0], a6[1], a6[2], a6[3], a6[4], a6[5]};   // a00 a01 a02 a11 a12 a22
    double v[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int sweep = 0; sweep < 60; ++sweep) {
        const double off = (fabs(a[1]) + fabs(a[2])) + fabs(a[4]);
        if (off == 0.0) break;
        jacobi3_rotate<0>(sweep, a, v);
        jacobi3_rotate<1>(sweep, a, v);
        jacobi3_rotate<2>(sweep, a, v);
    }
    d[0] = a[0]; d[1] = a[3]; d[2] = a[5];
#pragma unroll
    for (int i = 0; i < 9; ++i) V[i] = v[i];
}

// Ascending order of three eigenvalues exactly as a bubble sort over an index array produces it (equal values keep their order), and
// the selection of an eigenvector column, both without indexed access (register arrays stay in registers).
IM_HD void order3(const double* ev, int* o) {
    double e0 = ev[0], e1 = ev[1], e2 = ev[2];
    int o0 = 0, o1 = 1, o2 = 2;
    if (e1 < e0) { const double t = e0; e0 = e1; e1 = t; const int u = o0; o0 = o1; o1 = u; }
    if (e2 < e1) { const double t = e1; e1 = e2; e2 = t; const int u = o1; o1 = o2; o2 = u; }
    if (e1 < e0) { const double t = e0; e0 = e1; e1 = t; const int u = o0; o0 = o1; o1 = u; }
    o[0] = o0; o[1] = o1; o[2] = o2;
}
IM_HD double col3(const double* U, int row, int c) { return c == 0 ? U[row * 3] : (c == 1 ? U[row * 3 + 1] : U[row * 3 + 2]); }

// order-free fixed-point accumulation of the normal equations (2^-20 quantum, 32-bit hi/lo split)
#define IM_FX_SCALE 1048576.0
IM_HD void fx_split(double x, long long* hi, long long* lo) {
    const long long t = im_llrint(x * IM_FX_SCALE);
    *hi = (t >> 32);
    *lo = (t & 0xffffffffLL);
}
IM_HD double fx_value(long long hi, long long lo) { return ((double)hi * 4294967296.0 + (double)lo) * (1.0 / IM_FX_SCALE); }

}  // namespace immesh
