// immesh_b200 -- version / error string / profiling entry points.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "common_host.hpp"

namespace immesh {
Profiler& profiler() {
    static Profiler p;
    return p;
}
}  // namespace immesh

extern "C" {
// save_to_ply_file (src/meshing/mesh_rec_geometry.cpp:71-131, smooth_factor == 0 branch): binary little-endian PLY, vertices as float
// x y z, one face per live triangle with the reference's orientation rule -- m_index_flip != 0 keeps (p0, p1, p2), == 0 writes
// (p0, p2, p1) (:108-121).  Host-side only: the arrays are what immesh_mesh_snapshot returns.
int immesh_write_ply(const char* path, const float* vertices, int nv, const int32_t* triangles, const int32_t* flips, int nt) {
    if (!path || (!vertices && nv > 0) || (!triangles && nt > 0) || nv < 0 || nt < 0) return immesh::im_fail(IMMESH_E_INVALID, "bad argument");
    for (int t = 0; t < nt * 3; ++t)
        if (triangles[t] < 0 || triangles[t] >= nv) return immesh::im_fail(IMMESH_E_RANGE, "triangle refers to a vertex outside the vertex array");
    FILE* f = std::fopen(path, "wb");
    if (!f) return immesh::im_fail(IMMESH_E_INVALID, "cannot open the output file");
    std::fprintf(f, "ply\nformat binary_little_endian 1.0\ncomment immesh_b200 (layout of pcl::io::savePLYFileBinary for a PolygonMesh of PointXYZ)\n"
                    "element vertex %d\nproperty float x\nproperty float y\nproperty float z\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n", nv, nt);
    if (nv > 0) std::fwrite(vertices, sizeof(float) * 3, (size_t)nv, f);
    for (int t = 0; t < nt; ++t) {
        const unsigned char three = 3;
        const int32_t a = triangles[3 * t], b = triangles[3 * t + 1], c = triangles[3 * t + 2];
        const int32_t face[3] = {a, (flips && flips[t] != 0) ? b : c, (flips && flips[t] != 0) ? c : b};
        std::fwrite(&three, 1, 1, f);
        std::fwrite(face, sizeof(int32_t), 3, f);
    }
    const bool ok = std::fclose(f) == 0;
    return ok ? IMMESH_OK : immesh::im_fail(IMMESH_E_INVALID, "write failed");
}
// pcl::io::savePCDFileBinary of the vertex cloud (save_to_ply_file writes it next to the PLY, mesh_rec_geometry.cpp:129): PCD v0.7
// header of a PointXYZ cloud, then the packed float x y z records.
int immesh_write_pcd(const char* path, const float* vertices, int nv) {
    if (!path || (!vertices && nv > 0) || nv < 0) return immesh::im_fail(IMMESH_E_INVALID, "bad argument");
    FILE* f = std::fopen(path, "wb");
    if (!f) return immesh::im_fail(IMMESH_E_INVALID, "cannot open the output file");
    std::fprintf(f, "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH %d\nHEIGHT 1\n"
                    "VIEWPOINT 0 0 0 1 0 0 0\nPOINTS %d\nDATA binary\n", nv, nv);
    if (nv > 0) std::fwrite(vertices, sizeof(float) * 3, (size_t)nv, f);
    const bool ok = std::fclose(f) == 0;
    return ok ? IMMESH_OK : immesh::im_fail(IMMESH_E_INVALID, "write failed");
}

// Voxel_mapping::kitti_log (src/voxel_mapping_common.cpp:43-70): the pose in the KITTI camera frame, T = T_lidar_to_cam * [R t; 0 1] *
// T_lidar_to_cam^-1, as "stamp tx ty tz qx qy qz qw\n" with %lf fields.  Eigen is absent: the 4x4 inverse is a partial-pivot
// Gauss-Jordan elimination and the quaternion follows Eigen's rotation-matrix conversion (trace branch / largest diagonal).
static void inv4(const double* A, double* Ai) {
    double a[4][8];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 8; ++j) a[i][j] = j < 4 ? A[i * 4 + j] : (j - 4 == i ? 1.0 : 0.0);
    for (int k = 0; k < 4; ++k) {
        int best = k;
        for (int i = k + 1; i < 4; ++i)
            if (std::fabs(a[i][k]) > std::fabs(a[best][k])) best = i;
        if (best != k)
            for (int j = 0; j < 8; ++j) { const double t = a[k][j]; a[k][j] = a[best][j]; a[best][j] = t; }
        const double p = a[k][k];
        for (int j = 0; j < 8; ++j) a[k][j] = a[k][j] / p;
        for (int i = 0; i < 4; ++i) {
            if (i == k) continue;
            const double f = a[i][k];
            for (int j = 0; j < 8; ++j) a[i][j] = a[i][j] - f * a[k][j];
        }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) Ai[i * 4 + j] = a[i][4 + j];
}
static void mul4(const double* A, const double* B, double* C) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = 0.0;
            for (int k = 0; k < 4; ++k) s = s + A[i * 4 + k] * B[k * 4 + j];
            C[i * 4 + j] = s;
        }
}
int immesh_kitti_pose_line(const double* state /*[>= 12]: rot_end[9] row-major, pos_end[3]*/, double stamp, char* buf, int cap) {
    if (!state || !buf || cap < 32) return immesh::im_fail(IMMESH_E_INVALID, "bad argument");
    static const double L2C[16] = {0.00554604, -0.999971, -0.00523653, 0.0316362, -0.000379382, 0.00523451, -0.999986, 0.0380934,
                                   0.999985, 0.00554795, -0.000350341, 0.409066, 0, 0, 0, 1};
    double T[16] = {state[0], state[1], state[2], state[9], state[3], state[4], state[5], state[10], state[6], state[7], state[8], state[11], 0, 0, 0, 1};
    double Li[16], A[16], B[16];
    inv4(L2C, Li);
    mul4(L2C, T, A);
    mul4(A, Li, B);
    const double m00 = B[0], m01 = B[1], m02 = B[2], m10 = B[4], m11 = B[5], m12 = B[6], m20 = B[8], m21 = B[9], m22 = B[10];
    double qw, qx, qy, qz;
    double t = m00 + m11 + m22;
    if (t > 0.0) {                      // Eigen::Quaterniond(Matrix3d): trace branch
        t = std::sqrt(t + 1.0);
        qw = 0.5 * t;
        t = 0.5 / t;
        qx = (m21 - m12) * t; qy = (m02 - m20) * t; qz = (m10 - m01) * t;
    } else {
        const double m[3][3] = {{m00, m01, m02}, {m10, m11, m12}, {m20, m21, m22}};
        int i = 0;
        if (m11 > m00) i = 1;
        if (m22 > m[i][i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        double q[3];
        t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        qw = (m[k][j] - m[j][k]) * t;
        q[j] = (m[j][i] + m[i][j]) * t;
        q[k] = (m[k][i] + m[i][k]) * t;
        qx = q[0]; qy = q[1]; qz = q[2];
    }
    const int n = std::snprintf(buf, (size_t)cap, "%lf %lf %lf %lf %lf %lf %lf %lf\n", stamp, B[3], B[7], B[11], qx, qy, qz, qw);
    return (n > 0 && n < cap) ? IMMESH_OK : immesh::im_fail(IMMESH_E_CAPACITY, "buffer too small");
}

// publish_odometry's pose: pos_end, then RotMtoEuler(rot_end) turned into a quaternion by tf's setRPY (the rule is in the header)
int immesh_odometry_pose(const double* s, double* out) {
    if (!s || !out) return immesh::im_fail(IMMESH_E_INVALID, "null argument");
    const double r00 = s[0], r10 = s[3], r11 = s[4], r12 = s[5], r20 = s[6], r21 = s[7], r22 = s[8];
    const double sy = std::sqrt(r00 * r00 + r10 * r10);
    double roll, pitch, yaw;
    if (!(sy < 1e-6)) {
        roll = std::atan2(r21, r22);
        pitch = std::atan2(-r20, sy);
        yaw = std::atan2(r10, r00);
    } else {
        roll = std::atan2(-r12, r11);
        pitch = std::atan2(-r20, sy);
        yaw = 0;
    }
    const double hy = yaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
    const double cy = std::cos(hy), sy2 = std::sin(hy), cp = std::cos(hp), sp = std::sin(hp), cr = std::cos(hr), sr = std::sin(hr);
    out[0] = s[9]; out[1] = s[10]; out[2] = s[11];
    out[3] = sr * cp * cy - cr * sp * sy2;
    out[4] = cr * sp * cy + sr * cp * sy2;
    out[5] = cr * cp * sy2 - sr * sp * cy;
    out[6] = cr * cp * cy + sr * sp * sy2;
    return IMMESH_OK;
}

// dump_lio_state_to_log's line (the rule is in the header)
int immesh_lio_state_line(const double* s, double t, char* buf, int cap) {
    if (!s || !buf || cap < 1) return immesh::im_fail(IMMESH_E_INVALID, "bad argument");
    const double tr = (s[0] + s[4]) + s[8];
    const double theta = (tr > 3.0 - 1e-6) ? 0.0 : std::acos(0.5 * (tr - 1));
    const double K[3] = {s[7] - s[5], s[2] - s[6], s[3] - s[1]};
    const double f = std::abs(theta) < 0.001 ? 0.5 : 0.5 * theta / std::sin(theta);
    const double v[24] = {K[0] * f, K[1] * f, K[2] * f, s[9], s[10], s[11], 0.0, 0.0, 0.0, s[12], s[13], s[14], 0.0, 0.0, 0.0,
                          s[15], s[16], s[17], s[18], s[19], s[20], s[21], s[22], s[23]};
    int len = std::snprintf(buf, (size_t)cap, "%lf ", t);
    for (int i = 0; i < 24 && len >= 0 && len < cap; ++i) len += std::snprintf(buf + len, (size_t)(cap - len), "%lf ", v[i]);
    if (len >= 0 && len < cap) len += std::snprintf(buf + len, (size_t)(cap - len), "\r\n");
    return (len > 0 && len < cap) ? IMMESH_OK : immesh::im_fail(IMMESH_E_CAPACITY, "buffer too small");
}

const char* immesh_last_error(void) { return immesh::last_error_storage().c_str(); }
const char* immesh_version(void) { return "immesh_b200 0.1.0 (sm_90a)"; }

int immesh_profile_enable(int on) {
    immesh::profiler().enabled = on != 0;
    if (on == 2) immesh::profiler().start_timeline();   // also record every launch's start / end time
    else immesh::profiler().timeline_on = false;
    return IMMESH_OK;
}
int immesh_profile_reset(void) {
    immesh::profiler().totals.clear();
    immesh::profiler().launches = 0;
    return IMMESH_OK;
}
long long immesh_launch_count(void) { return immesh::profiler().launches; }
// "name t0_ms t1_ms\n" per launch recorded since immesh_profile_enable(2); returns the number of bytes needed
int immesh_profile_timeline(char* buf, int cap) {
    std::string s;
    for (auto& sp : immesh::profiler().timeline) {
        char line[256];
        std::snprintf(line, sizeof(line), "%s %.6f %.6f\n", sp.name, sp.t0, sp.t1);
        s += line;
    }
    if (buf && cap > 0) {
        std::strncpy(buf, s.c_str(), (size_t)cap - 1);
        buf[cap - 1] = 0;
    }
    return (int)s.size() + 1;
}
// writes "name ms launches\n" lines into buf; returns the number of bytes needed
int immesh_profile_report(char* buf, int cap) {
    std::string s;
    for (auto& kv : immesh::profiler().totals) {
        char line[256];
        std::snprintf(line, sizeof(line), "%s %.6f %lld\n", kv.first.c_str(), kv.second.first, kv.second.second);
        s += line;
    }
    if (buf && cap > 0) {
        std::strncpy(buf, s.c_str(), (size_t)cap - 1);
        buf[cap - 1] = 0;
    }
    return (int)s.size() + 1;
}
}
