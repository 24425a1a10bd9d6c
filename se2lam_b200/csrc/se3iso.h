// g2o::VertexSE3 (an Eigen::Isometry3d estimate with oplus = X * fromVectorMQT) and the EdgeSE3Prior of
// addVertexSE3PlaneMotion, restated for device code in double precision, on top of se3quat.h. Used by the feature-graph
// constraint (feat_edge.cu) and the global pose graph (global_ba.cu). The functions that are not inline keep internal
// linkage, as they had inside feat_edge.cu, so each kernel file compiles them exactly as before.
#pragma once
#include "se3quat.h"

namespace se2gpu {

struct Iso { double R[9], t[3]; };  // Eigen::Isometry3d: rotation row-major, translation

// EdgeSE3Prior with an identity ParameterSE3Offset: the inverse of its measurement and its information
struct Prior {
    Iso meas_inv;
    double info[36];
};

__device__ inline void mulv3(const double* A, const double* v, double* o) {
#pragma unroll
    for (int r = 0; r < 3; ++r) o[r] = A[r * 3] * v[0] + A[r * 3 + 1] * v[1] + A[r * 3 + 2] * v[2];
}

__device__ inline Iso iso_mul(const Iso& a, const Iso& b) {
    Iso r;
    mul3(a.R, b.R, r.R);
    mulv3(a.R, b.t, r.t);
    for (int i = 0; i < 3; ++i) r.t[i] += a.t[i];
    return r;
}

// Eigen Transform::inverse(Isometry): R^T, -R^T t
__device__ inline Iso iso_inv(const Iso& a) {
    Iso r;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) r.R[i * 3 + j] = a.R[j * 3 + i];
    double v[3];
    mulv3(r.R, a.t, v);
    for (int i = 0; i < 3; ++i) r.t[i] = -v[i];
    return r;
}

// converter.cpp toIsometry3D(getPose().inv()): the rigid inverse in double, the rotation through an un-normalised Quaterniond
static __device__ Iso iso_from_Tcw(const float* T) {
    Iso cw;
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    for (int i = 0; i < 9; ++i) cw.R[i] = R[i];
    cw.t[0] = T[3]; cw.t[1] = T[7]; cw.t[2] = T[11];
    Iso wc = iso_inv(cw);
    const Quat q = quat_from_R(wc.R);
    quat_to_R(q, wc.R);
    return wc;
}

// g2o::internal::toSE3Quat(Isometry3D): SE3Quat(R, t)
static __device__ SE3 se3_from_iso(const Iso& X) {
    SE3 T;
    T.q = quat_from_R(X.R);
    for (int i = 0; i < 3; ++i) T.t[i] = X.t[i];
    normalize_rotation(T.q);
    return T;
}

// VertexSE3::oplusImpl: X * fromVectorMQT(d), d = (t, qx, qy, qz), w = sqrt(1 - |q|^2); the normalised (0, q) when |q|^2 >= 1
static __device__ Iso oplus(const Iso& X, const double* d) {
    const double n2 = d[3] * d[3] + d[4] * d[4] + d[5] * d[5], w = 1. - n2;
    Quat q;
    if (w < 0) {
        const double n = sqrt(n2);
        q = {d[3] / n, d[4] / n, d[5] / n, 0};
    } else {
        q = {d[3], d[4], d[5], sqrt(w)};
    }
    Iso D;
    quat_to_R(q, D.R);
    D.t[0] = d[0]; D.t[1] = d[1]; D.t[2] = d[2];
    return iso_mul(X, D);
}

// addVertexSE3PlaneMotion (src/optimizer.cpp:429-455) with AdjTR (:93-102) = [[R, skew(t) R], [0, R]]; Tbc = Config::bTc,
// xrot / yrot / zinfo = Config::PLANEMOTION_XROT_INFO / _YROT_INFO / _Z_INFO
static __device__ __noinline__ void plane_motion_prior(const Iso& pose, const float* Tbc_f, float xrot, float yrot, float zinfo,
                                                       Prior* pr) {
    const SE3 Tbc = se3_from_f32(Tbc_f);
    SE3 Twb = se3_mul(se3_from_iso(pose), se3_inv(Tbc));
    const double ha = 0.5 * rotvec_z(Twb.q);
    double s, c;
    sincos(ha, &s, &c);
    Twb.q = {s * 0.0, s * 0.0, s * 1.0, c};  // Quaterniond(AngleAxisd(yaw, UnitZ)); setRotation does not normalise
    Twb.t[2] = 0;
    const SE3 Twc = se3_mul(Twb, Tbc);
    Iso meas;
    quat_to_R(Twc.q, meas.R);
    for (int i = 0; i < 3; ++i) meas.t[i] = Twc.t[i];
    pr->meas_inv = iso_inv(meas);
    double R[9], S[9], SR[9], A[36];
    quat_to_R(Tbc.q, R);
    skew(Tbc.t, S);
    mul3(S, R, SR);
    for (int k = 0; k < 36; ++k) A[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 3; ++cc) {
            A[r * 6 + cc] = R[r * 3 + cc];
            A[(r + 3) * 6 + cc + 3] = R[r * 3 + cc];
            A[r * 6 + cc + 3] = SR[r * 3 + cc];
        }
    const double dg[6] = {1e-4, 1e-4, (double)zinfo, (double)xrot, (double)yrot, 1e-4};
    for (int r = 0; r < 6; ++r)
        for (int cc = 0; cc < 6; ++cc) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (A[k * 6 + r] * dg[k]) * A[k * 6 + cc];
            pr->info[r * 6 + cc] = acc;
        }
}

// EdgeSE3Prior: e = toVectorMQT(Z^-1 X), its chi2; with H also J^T Omega J into H [36] and -J^T Omega e into b [6], J the
// derivative of e through oplus: [[R_e, 0], [0, w I + skew(v)]]
static __device__ __noinline__ double prior_terms(const Prior& pr, const Iso& X, double* H, double* b) {
    const Iso E = iso_mul(pr.meas_inv, X);
    Quat q = quat_from_R(E.R);
    normalize_rotation(q);
    const double e[6] = {E.t[0], E.t[1], E.t[2], q.x, q.y, q.z};
    double Oe[6], chi = 0;
    for (int r = 0; r < 6; ++r) {
        double we = 0;
        for (int c = 0; c < 6; ++c) we += pr.info[r * 6 + c] * e[c];
        Oe[r] = we;
        chi += e[r] * we;
    }
    if (!H) return chi;
    double J[36], OJ[36];
    for (int k = 0; k < 36; ++k) J[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) J[r * 6 + c] = E.R[r * 3 + c];
    J[21] = q.w;  J[22] = -q.z; J[23] = q.y;
    J[27] = q.z;  J[28] = q.w;  J[29] = -q.x;
    J[33] = -q.y; J[34] = q.x;  J[35] = q.w;
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int m = 0; m < 6; ++m) acc += pr.info[r * 6 + m] * J[m * 6 + c];
            OJ[r * 6 + c] = acc;
        }
    for (int r = 0; r < 6; ++r) {
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int m = 0; m < 6; ++m) acc += J[m * 6 + r] * OJ[m * 6 + c];
            H[r * 6 + c] = acc;
        }
        double acc = 0;
        for (int m = 0; m < 6; ++m) acc += J[m * 6 + r] * Oe[m];
        b[r] = -acc;
    }
    return chi;
}

}  // namespace se2gpu
