// g2o::SE3Quat and the Eigen quaternion routines it rests on, restated for device code in double precision. Used by the
// pose-only BA (pose_ba.cu), and through se3iso.h by the feature-graph constraint (feat_edge.cu) and the global pose graph
// (global_ba.cu).
#pragma once
#include <cuda_runtime.h>

namespace se2gpu {

struct Quat { double x, y, z, w; };
struct SE3 { Quat q; double t[3]; };

__device__ inline void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// Eigen Quaterniond(const Matrix3d&)
__device__ inline Quat quat_from_R(const double* m) {
    Quat q;
    double t = m[0] + m[4] + m[8];
    if (t > 0) {
        t = sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (m[7] - m[5]) * t;
        q.y = (m[2] - m[6]) * t;
        q.z = (m[3] - m[1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 4]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        double c[3];
        t = sqrt(m[i * 4] - m[j * 4] - m[k * 4] + 1.0);
        c[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (m[k * 3 + j] - m[j * 3 + k]) * t;
        c[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        c[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        q.x = c[0]; q.y = c[1]; q.z = c[2];
    }
    return q;
}

// Eigen QuaternionBase::toRotationMatrix
__device__ inline void quat_to_R(const Quat& q, double* R) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

__device__ inline Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// Eigen q * v (_transformVector)
__device__ inline void qrot(const Quat& q, const double* v, double* out) {
    const double qv[3] = {q.x, q.y, q.z};
    double uv[3], c[3];
    cross(qv, v, uv);
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    cross(qv, uv, c);
    for (int i = 0; i < 3; ++i) out[i] = v[i] + q.w * uv[i] + c[i];
}

// g2o SE3Quat::normalizeRotation
__device__ inline void normalize_rotation(Quat& q) {
    if (q.w < 0) { q.x = -q.x; q.y = -q.y; q.z = -q.z; q.w = -q.w; }
    const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    if (n2 > 0) {
        const double n = sqrt(n2);
        q.x /= n; q.y /= n; q.z /= n; q.w /= n;
    }
}

// converter.cpp toSE3Quat(cv::Mat) on a float 4x4 row-major
__device__ inline SE3 se3_from_f32(const float* T) {
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    SE3 r;
    r.q = quat_from_R(R);
    r.t[0] = T[3]; r.t[1] = T[7]; r.t[2] = T[11];
    normalize_rotation(r.q);
    return r;
}

// converter.cpp toCvMat(SE3Quat): to_homogeneous_matrix narrowed to a float 4x4 row-major
__device__ inline void se3_to_f32(const SE3& T, float* M) {
    double R[9];
    quat_to_R(T.q, R);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) M[r * 4 + c] = (float)R[r * 3 + c];
        M[r * 4 + 3] = (float)T.t[r];
    }
    M[12] = 0.f; M[13] = 0.f; M[14] = 0.f; M[15] = 1.f;
}

// the pose as the library returns it: (qx, qy, qz, qw, tx, ty, tz)
__device__ inline void store_pose(const SE3& T, double* p7) {
    p7[0] = T.q.x; p7[1] = T.q.y; p7[2] = T.q.z; p7[3] = T.q.w;
    p7[4] = T.t[0]; p7[5] = T.t[1]; p7[6] = T.t[2];
}

__device__ inline SE3 se3_mul(const SE3& a, const SE3& b) {
    SE3 r = a;
    double rt[3];
    qrot(a.q, b.t, rt);
    for (int i = 0; i < 3; ++i) r.t[i] += rt[i];
    r.q = qmul(a.q, b.q);
    normalize_rotation(r.q);
    return r;
}

__device__ inline SE3 se3_inv(const SE3& a) {
    SE3 r;
    r.q = {-a.q.x, -a.q.y, -a.q.z, a.q.w};
    const double mt[3] = {a.t[0] * -1., a.t[1] * -1., a.t[2] * -1.};
    qrot(r.q, mt, r.t);
    return r;
}

__device__ inline void skew(const double* v, double* S) {
    S[0] = 0;     S[1] = -v[2]; S[2] = v[1];
    S[3] = v[2];  S[4] = 0;     S[5] = -v[0];
    S[6] = -v[1]; S[7] = v[0];  S[8] = 0;
}

__device__ inline void mul3(const double* A, const double* B, double* C) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

// z component of Eigen 3.3's AngleAxisd(Quaterniond) as angle * axis: angle = 2 atan2(|vec|, |w|), axis = vec / (+-|vec|)
__device__ inline double rotvec_z(const Quat& q) {
    double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z), angle = 0, axis_z = 0;
    if (n != 0) {
        angle = 2 * atan2(n, fabs(q.w));
        if (q.w < 0) n = -n;
        axis_z = q.z / n;
    }
    return angle * axis_z;
}

}  // namespace se2gpu
