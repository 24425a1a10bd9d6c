// g2o's VertexSE3Expmap edges (types_six_dof_expmap, g2o 20160424) restated for device code in double precision on top of
// se3quat.h: SE3Quat::exp / log / adj, the plane-motion EdgeSE3ExpmapPrior of addPlaneMotionSE3Expmap, EdgeProjectXYZ2UV
// (pose and point blocks) and EdgeSE3Expmap. Used by the pose-only BA (pose_ba.cu) and the SE(3)-XYZ window BA
// (se3_ba.cu). The functions that are not inline keep internal linkage, as they had inside pose_ba.cu, so each kernel file
// compiles them as before; the ones that read camera or prior parameters take any struct with the fields they name.
#pragma once
#include "se3quat.h"

namespace se2gpu {

// g2o SE3Quat::exp, update [omega, upsilon], small-angle branch below theta = 1e-5
static __device__ SE3 se3_exp(const double* u) {
    const double* omega = u;
    const double* upsilon = u + 3;
    const double theta = sqrt(omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2]);
    double O[9], O2[9], R[9], V[9];
    skew(omega, O);
    mul3(O, O, O2);
    if (theta < 0.00001) {
        for (int k = 0; k < 9; ++k) { R[k] = (k % 4 == 0 ? 1.0 : 0.0) + O[k] + O2[k]; V[k] = R[k]; }
    } else {
        double s, c;
        sincos(theta, &s, &c);
        const double a = s / theta, b = (1 - c) / (theta * theta), d = (theta - s) / (theta * theta * theta);
        for (int k = 0; k < 9; ++k) {
            const double I = (k % 4 == 0 ? 1.0 : 0.0);
            R[k] = I + a * O[k] + b * O2[k];
            V[k] = I + b * O[k] + d * O2[k];
        }
    }
    SE3 T;
    for (int r = 0; r < 3; ++r) T.t[r] = V[r * 3] * upsilon[0] + V[r * 3 + 1] * upsilon[1] + V[r * 3 + 2] * upsilon[2];
    T.q = quat_from_R(R);
    normalize_rotation(T.q);
    return T;
}

// g2o SE3Quat::log, small-rotation branch above d = 0.99999
static __device__ void se3_log(const SE3& T, double* res) {
    double R[9];
    quat_to_R(T.q, R);
    const double d = 0.5 * (R[0] + R[4] + R[8] - 1);
    const double dR[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    double omega[3], O[9], O2[9], f;
    if (d > 0.99999) {
        for (int i = 0; i < 3; ++i) omega[i] = 0.5 * dR[i];
        f = 1. / 12.;
    } else {
        const double theta = acos(d);
        const double s = theta / (2 * sqrt(1 - d * d));
        for (int i = 0; i < 3; ++i) omega[i] = s * dR[i];
        f = (1 - theta / (2 * tan(theta / 2))) / (theta * theta);
    }
    skew(omega, O);
    mul3(O, O, O2);
    for (int i = 0; i < 3; ++i) res[i] = omega[i];
    for (int r = 0; r < 3; ++r) {
        double acc = 0;
        for (int c = 0; c < 3; ++c) acc += ((r == c ? 1.0 : 0.0) - 0.5 * O[r * 3 + c] + f * O2[r * 3 + c]) * T.t[c];
        res[3 + r] = acc;
    }
}

// g2o SE3Quat::adj(): [[R, 0], [skew(t) R, R]], row-major 6 x 6
__device__ inline void se3_adj(const SE3& T, double* A) {
    double R[9], S[9], SR[9];
    quat_to_R(T.q, R);
    skew(T.t, S);
    mul3(S, R, SR);
    for (int k = 0; k < 36; ++k) A[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            A[r * 6 + c] = R[r * 3 + c];
            A[(r + 3) * 6 + c + 3] = R[r * 3 + c];
            A[(r + 3) * 6 + c] = SR[r * 3 + c];
        }
}

// addPlaneMotionSE3Expmap (src/optimizer.cpp:236-314, non-USE_EULER branch); p: Tbc[16], xrot, yrot, zinfo
template <class P>
static __device__ void plane_motion_prior(const SE3& pose, const P& p, SE3* meas, double* info) {
    const SE3 Tbc = se3_from_f32(p.Tbc);
    SE3 Tbw = se3_mul(Tbc, pose);
    const double ha = 0.5 * rotvec_z(Tbw.q);
    double s, c;
    sincos(ha, &s, &c);
    Tbw.q = {s * 0.0, s * 0.0, s * 1.0, c};  // Quaterniond(AngleAxisd(yaw, UnitZ)); setRotation does not normalise
    Tbw.t[2] = 0;
    *meas = se3_mul(se3_inv(Tbc), Tbw);
    // Info_cw = Adj(Tbc)^T diag(xrot, yrot, 1e-4, 1e-4, 1e-4, z) Adj(Tbc), Adj = [[R, 0], [skew(t) R, R]]
    double R[9], S[9], SR[9], J[36];
    quat_to_R(Tbc.q, R);
    skew(Tbc.t, S);
    mul3(S, R, SR);
    for (int k = 0; k < 36; ++k) J[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 3; ++cc) {
            J[r * 6 + cc] = R[r * 3 + cc];
            J[(r + 3) * 6 + cc + 3] = R[r * 3 + cc];
            J[(r + 3) * 6 + cc] = SR[r * 3 + cc];
        }
    const double dg[6] = {(double)p.xrot, (double)p.yrot, 1e-4, 1e-4, 1e-4, (double)p.zinfo};
    for (int r = 0; r < 6; ++r)
        for (int cc = r; cc < 6; ++cc) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (J[k * 6 + r] * dg[k]) * J[k * 6 + cc];
            info[r * 6 + cc] = acc;
            info[cc * 6 + r] = acc;  // symmetric from the upper triangle
        }
}

// log(meas * est^-1) and its chi2 under the prior's information
static __device__ double prior_error(const SE3& meas, const double* info, const SE3& T, double* e) {
    se3_log(se3_mul(meas, se3_inv(T)), e);
    double chi = 0;
    for (int r = 0; r < 6; ++r) {
        double we = 0;
        for (int c = 0; c < 6; ++c) we += info[r * 6 + c] * e[c];
        chi += e[r] * we;
    }
    return chi;
}

// one EdgeProjectXYZ2UV: robust chi2 into chi; with LIN also rho' J^T w J (upper triangle) into hb[0..20] and
// -rho' J^T w e into hb[21..26]; p: fx, cx, cy, delta
template <bool LIN, class P>
__device__ inline void edge_terms(const SE3& T, const float* xyz, const float* uv, float wf, const P& p, double& chi,
                                  double* hb) {
    const double X[3] = {xyz[0], xyz[1], xyz[2]};
    double pc[3];
    qrot(T.q, X, pc);
    for (int i = 0; i < 3; ++i) pc[i] += T.t[i];
    const double w = wf;
    const double e0 = (double)uv[0] - ((pc[0] / pc[2]) * p.fx + p.cx);
    const double e1 = (double)uv[1] - ((pc[1] / pc[2]) * p.fx + p.cy);
    const double c2 = e0 * (w * e0) + e1 * (w * e1);
    const double dsqr = p.delta * p.delta;
    const bool inlier = c2 <= dsqr;
    const double sq = inlier ? 0.0 : sqrt(c2);
    chi += inlier ? c2 : 2 * sq * p.delta - dsqr;
    if (!LIN) return;
    const double rho1 = inlier ? 1.0 : p.delta / sq;
    const double x = pc[0], y = pc[1], z = pc[2], z2 = z * z, fx = p.fx;
    const double J[12] = {x * y / z2 * fx,       -(1 + (x * x / z2)) * fx, y / z * fx,  -1. / z * fx, 0,            x / z2 * fx,
                          (1 + y * y / z2) * fx, -x * y / z2 * fx,         -x / z * fx, 0,            -1. / z * fx, y / z2 * fx};
    const double W = rho1 * w;
    const double r0 = -(w * e0) * rho1, r1 = -(w * e1) * rho1;
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        hb[21 + r] += J[r] * r0 + J[6 + r] * r1;
#pragma unroll
        for (int c = r; c < 6; ++c) hb[k++] += (J[r] * W) * J[c] + (J[6 + r] * W) * J[6 + c];
    }
}

// EdgeProjectXYZ2UV with a double point (the window BA's marginalised VertexSBAPointXYZ): the camera-frame point pc, the
// error e = uv - (pc_xy / pc_z * fx + c) and the raw chi2 e^T (w I) e. With Jp / Jl also linearizeOplus: the pose block
// _jacobianOplusXj (2 x 6, row-major) and the point block _jacobianOplusXi = -1/z [[fx, 0, -x/z fx], [0, fx, -y/z fx]] R
// (2 x 3, row-major).
template <class P>
__device__ inline double xyz2uv_terms(const SE3& T, const double* X, const float* uv, double w, const P& p, double* e,
                                      double* Jp, double* Jl) {
    double pc[3];
    qrot(T.q, X, pc);
    for (int i = 0; i < 3; ++i) pc[i] += T.t[i];
    e[0] = (double)uv[0] - ((pc[0] / pc[2]) * p.fx + p.cx);
    e[1] = (double)uv[1] - ((pc[1] / pc[2]) * p.fx + p.cy);
    const double c2 = e[0] * (w * e[0]) + e[1] * (w * e[1]);
    if (!Jp) return c2;
    const double x = pc[0], y = pc[1], z = pc[2], z2 = z * z, fx = p.fx;
    const double J[12] = {x * y / z2 * fx,       -(1 + (x * x / z2)) * fx, y / z * fx,  -1. / z * fx, 0,            x / z2 * fx,
                          (1 + y * y / z2) * fx, -x * y / z2 * fx,         -x / z * fx, 0,            -1. / z * fx, y / z2 * fx};
    for (int k = 0; k < 12; ++k) Jp[k] = J[k];
    double R[9];
    quat_to_R(T.q, R);
    const double iz = -1. / z;
    const double tmp[6] = {iz * fx, iz * 0.0, iz * (-x / z * fx), iz * 0.0, iz * fx, iz * (-y / z * fx)};
    for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 3; ++c) Jl[r * 3 + c] = tmp[r * 3] * R[c] + tmp[r * 3 + 1] * R[3 + c] + tmp[r * 3 + 2] * R[6 + c];
    return c2;
}

// Huber of g2o's RobustKernelHuber on a raw chi2: the robust chi2 rho0 and its weight rho1
__device__ inline double huber(double c2, double delta, double* rho1) {
    const double dsqr = delta * delta;
    if (c2 <= dsqr) { if (rho1) *rho1 = 1.0; return c2; }
    const double sq = sqrt(c2);
    if (rho1) *rho1 = delta / sq;
    return 2 * sq * delta - dsqr;
}

// EdgeSE3Expmap (vertices[0] = Ti, vertices[1] = Tj, measurement Z): e = log(Tj^-1 Z Ti) and e^T Om e. With Ji / Jj also
// g2o's analytic linearizeOplus, Ji = Adj(Tj^-1 Z) and Jj = -Adj(Ti^-1 Z^-1), which are the derivative of e only where
// e = 0 (g2o's approximation, kept).
__device__ inline double expmap_edge(const SE3& Z, const double* Om, const SE3& Ti, const SE3& Tj, double* e, double* Ji,
                                     double* Jj) {
    se3_log(se3_mul(se3_mul(se3_inv(Tj), Z), Ti), e);
    double chi = 0;
    for (int r = 0; r < 6; ++r) {
        double we = 0;
        for (int c = 0; c < 6; ++c) we += Om[r * 6 + c] * e[c];
        chi += e[r] * we;
    }
    if (!Ji) return chi;
    se3_adj(se3_mul(se3_inv(Tj), Z), Ji);
    se3_adj(se3_mul(se3_inv(Ti), se3_inv(Z)), Jj);
    for (int k = 0; k < 36; ++k) Jj[k] = -Jj[k];
    return chi;
}

}  // namespace se2gpu
