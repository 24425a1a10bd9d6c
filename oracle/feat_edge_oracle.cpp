// Feature-graph constraint ORACLE (GlobalMapper::CreateFeatEdge + Sparsifier) — TEST INFRASTRUCTURE ONLY.
//
// Sequential double-precision restatement of what the reference executes for one keyframe pair:
//   GlobalMapper::CreateFeatEdge, both overloads (src/GlobalMapper.cpp:737-843), OptKFPair (:847-927), OptKFPairMatch
//   (:929-1032), addVertexSE3PlaneMotion (src/optimizer.cpp:337-468, non-USE_OLD_SE3_PRIOR_JACOB branch), AdjTR (:93-102),
//   addEdgeSE3XYZ (:531-545), Sparsifier::JacobianSE3XYZ / HessianSE3XYZ / DoMarginalizeSE3XYZ / JacobianSE3 / InfoSE3
//   (src/sparsifier.cpp:59-274).
// g2o (tag 20160424) and Eigen are not vendored; their published definitions are restated: VertexSE3 (Isometry3D estimate,
// oplus = estimate * fromVectorMQT), VertexPointXYZ, EdgeSE3PointXYZ and EdgeSE3Prior with an identity ParameterSE3Offset,
// toVectorMQT / toCompactQuaternion, SE3Quat (operator*, inverse, map, toMinimalVector, fromMinimalVector),
// RobustKernelHuber, BaseBinaryEdge / BaseUnaryEdge::constructQuadraticForm (rho' * Omega, no second-order term),
// BlockSolver's Schur complement with lambda on the pose and the point diagonals, and
// OptimizationAlgorithmLevenberg::solve as oracle/ba_oracle.cpp and oracle/pose_ba_oracle.cpp have it.
//
// What is decided here and not copied from anywhere:
//  * The two edge Jacobians are the analytic first derivatives of the errors through the MQT oplus; they are unique, and
//    tests/test_feat_edge_oracle.py holds them to central differences through the real oplus.
//  * g2o re-orthogonalises a VertexSE3 only after 1000 oplus calls; 30 iterations of at most 10 trials never get there, so
//    it is not restated.
//  * The prior of a fixed vertex is left out of the active set (an edge whose vertices are all fixed); it would add a
//    constant to chi2 and cancels in rho either way.
//  * KeyFrame::getPose().inv() is a float LU of a 4 x 4 matrix in the reference; here the rigid inverse (R^T, -R^T t) is
//    taken in double from the float entries. The two agree to float rounding of the start estimate.
//  * OptKFPairMatch reads EdgeSE3PointXYZ::chi2() after optimize(): the error vector of the last evaluated trial, accepted
//    or not. That is kept. A trial whose factorisation failed leaves the errors as they were.
//  * H22 of DoMarginalizeSE3XYZ is block diagonal, so an unpivoted dense LDL^T never leaves the 3 x 3 blocks and is done
//    block by block; Eigen's diagonal pivoting is not restated. The 12 x 12 and 6 x 6 inverses are LU with partial
//    pivoting, the SVD is a one-sided Jacobi SVD.
// PARITY UNPINNED against real g2o (no g2o build exists here); pinned by self-consistency in
// tests/test_feat_edge_oracle.py (central-difference Jacobians, noise-free recovery, the eigenvalue form of the clamp).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

struct IterStats {  // must match se2gpu_ba_iter_stats (include/se2gpu.h)
    double chi2_before, chi2_after, lambda, rho;
    int trials, accepted, terminate, pad;
};

struct Params {  // must match se2gpu_feat_edge_params (include/se2gpu.h)
    float Tbc[16];
    float xrot, yrot, zinfo;
    float huber_delta;
    int iterations[2];
    float chi2_cut;
    int min_points[2];
};

struct Quat { double x, y, z, w; };
struct SE3 { Quat q; double t[3]; };   // g2o::SE3Quat
struct Iso { double R[9], t[3]; };     // Eigen::Isometry3d: rotation row-major, translation

void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// Eigen: Quaternion<double>(const Matrix3d&)
Quat quat_from_R(const double* m) {
    Quat q;
    double t = m[0] + m[4] + m[8];
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (m[7] - m[5]) * t;
        q.y = (m[2] - m[6]) * t;
        q.z = (m[3] - m[1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 4]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        double c[3];
        t = std::sqrt(m[i * 4] - m[j * 4] - m[k * 4] + 1.0);
        c[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (m[k * 3 + j] - m[j * 3 + k]) * t;
        c[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        c[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        q.x = c[0]; q.y = c[1]; q.z = c[2];
    }
    return q;
}

// Eigen: QuaternionBase::toRotationMatrix
void quat_to_R(const Quat& q, double* R) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// Eigen: q * v
void qrot(const Quat& q, const double* v, double* out) {
    const double qv[3] = {q.x, q.y, q.z};
    double uv[3], c[3];
    cross(qv, v, uv);
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    cross(qv, uv, c);
    for (int i = 0; i < 3; ++i) out[i] = v[i] + q.w * uv[i] + c[i];
}

// g2o SE3Quat::normalizeRotation
void normalize_rotation(Quat& q) {
    if (q.w < 0) { q.x = -q.x; q.y = -q.y; q.z = -q.z; q.w = -q.w; }
    const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    if (n2 > 0) {
        const double n = std::sqrt(n2);
        q.x /= n; q.y /= n; q.z /= n; q.w /= n;
    }
}

SE3 se3_from_Rt(const double* R, const double* t) {
    SE3 T;
    T.q = quat_from_R(R);
    for (int i = 0; i < 3; ++i) T.t[i] = t[i];
    normalize_rotation(T.q);
    return T;
}

SE3 se3_from_f32(const float* T) {
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    const double t[3] = {T[3], T[7], T[11]};
    return se3_from_Rt(R, t);
}

SE3 se3_mul(const SE3& a, const SE3& b) {
    SE3 r = a;
    double rt[3];
    qrot(a.q, b.t, rt);
    for (int i = 0; i < 3; ++i) r.t[i] += rt[i];
    r.q = qmul(a.q, b.q);
    normalize_rotation(r.q);
    return r;
}

SE3 se3_inv(const SE3& a) {
    SE3 r;
    r.q = {-a.q.x, -a.q.y, -a.q.z, a.q.w};
    const double mt[3] = {a.t[0] * -1., a.t[1] * -1., a.t[2] * -1.};
    qrot(r.q, mt, r.t);
    return r;
}

// SE3Quat::map / operator*(Vector3D)
void se3_map(const SE3& T, const double* p, double* out) {
    qrot(T.q, p, out);
    for (int i = 0; i < 3; ++i) out[i] += T.t[i];
}

// SE3Quat::toMinimalVector: (t, qx, qy, qz)
void se3_to_min(const SE3& T, double* v) {
    v[0] = T.t[0]; v[1] = T.t[1]; v[2] = T.t[2];
    v[3] = T.q.x; v[4] = T.q.y; v[5] = T.q.z;
}

// SE3Quat::fromMinimalVector
SE3 se3_from_min(const double* v) {
    SE3 T;
    const double w = 1. - v[3] * v[3] - v[4] * v[4] - v[5] * v[5];
    if (w > 0) T.q = {v[3], v[4], v[5], std::sqrt(w)};
    else T.q = {-v[3], -v[4], -v[5], 0};
    T.t[0] = v[0]; T.t[1] = v[1]; T.t[2] = v[2];
    return T;
}

void mul3(const double* A, const double* B, double* C) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}
void mulv3(const double* A, const double* v, double* o) {
    for (int r = 0; r < 3; ++r) o[r] = A[r * 3] * v[0] + A[r * 3 + 1] * v[1] + A[r * 3 + 2] * v[2];
}

Iso iso_mul(const Iso& a, const Iso& b) {
    Iso r;
    mul3(a.R, b.R, r.R);
    mulv3(a.R, b.t, r.t);
    for (int i = 0; i < 3; ++i) r.t[i] += a.t[i];
    return r;
}

// Eigen Transform::inverse(Isometry): R^T, -R^T t
Iso iso_inv(const Iso& a) {
    Iso r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.R[i * 3 + j] = a.R[j * 3 + i];
    double v[3];
    mulv3(r.R, a.t, v);
    for (int i = 0; i < 3; ++i) r.t[i] = -v[i];
    return r;
}

// converter.cpp toIsometry3D(getPose().inv()): the rotation goes through an un-normalised Quaterniond
Iso iso_from_Tcw(const float* T) {
    Iso cw;
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    std::memcpy(cw.R, R, sizeof R);
    cw.t[0] = T[3]; cw.t[1] = T[7]; cw.t[2] = T[11];
    Iso wc = iso_inv(cw);
    quat_to_R(quat_from_R(wc.R), wc.R);
    return wc;
}

// g2o::internal::toSE3Quat(Isometry3D)
SE3 se3_from_iso(const Iso& X) { return se3_from_Rt(X.R, X.t); }
Iso iso_from_se3(const SE3& T) {
    Iso X;
    quat_to_R(T.q, X.R);
    std::memcpy(X.t, T.t, sizeof X.t);
    return X;
}

// g2o::internal::fromVectorMQT: (t, qx, qy, qz), w = sqrt(1 - |q|^2); the normalised (0, q) when |q|^2 >= 1
Iso iso_from_mqt(const double* d) {
    const double n2 = d[3] * d[3] + d[4] * d[4] + d[5] * d[5];
    const double w = 1. - n2;
    Quat q;
    if (w < 0) {
        const double n = std::sqrt(n2);
        q = {d[3] / n, d[4] / n, d[5] / n, 0};
    } else {
        q = {d[3], d[4], d[5], std::sqrt(w)};
    }
    Iso X;
    quat_to_R(q, X.R);
    X.t[0] = d[0]; X.t[1] = d[1]; X.t[2] = d[2];
    return X;
}

// VertexSE3::oplusImpl
Iso oplus(const Iso& X, const double* d) { return iso_mul(X, iso_from_mqt(d)); }

// EdgeSE3PointXYZ::computeError with an identity offset: X^-1 p - z; pc = X^-1 p
void xyz_error(const Iso& Xinv, const double* p, const double* z, double* e, double* pc) {
    mulv3(Xinv.R, p, pc);
    for (int i = 0; i < 3; ++i) { pc[i] += Xinv.t[i]; e[i] = pc[i] - z[i]; }
}
// its Jacobians through oplus: pose [-I | 2 skew(pc)] (3 x 6), point R^T (3 x 3)
void xyz_jacobians(const Iso& Xinv, const double* pc, double* Jp, double* Jl) {
    for (int k = 0; k < 18; ++k) Jp[k] = 0;
    Jp[0] = -1; Jp[7] = -1; Jp[14] = -1;
    Jp[4] = -2 * pc[2];  Jp[5] = 2 * pc[1];
    Jp[9] = 2 * pc[2];   Jp[11] = -2 * pc[0];
    Jp[15] = -2 * pc[1]; Jp[16] = 2 * pc[0];
    std::memcpy(Jl, Xinv.R, 9 * sizeof(double));
}

struct Prior {
    Iso meas, meas_inv;
    double info[36];
};

// addVertexSE3PlaneMotion (src/optimizer.cpp:429-455)
Prior plane_motion_prior(const Iso& pose, const Params& p) {
    const SE3 Tbc = se3_from_f32(p.Tbc);
    SE3 Twb = se3_mul(se3_from_iso(pose), se3_inv(Tbc));
    const Quat& q = Twb.q;  // Eigen 3.3 AngleAxisd(Quaterniond)
    double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z), angle = 0, axis_z = 0;
    if (n != 0) {
        angle = 2 * std::atan2(n, std::fabs(q.w));
        if (q.w < 0) n = -n;
        axis_z = q.z / n;
    }
    const double ha = 0.5 * (angle * axis_z), s = std::sin(ha);
    Twb.q = {s * 0.0, s * 0.0, s * 1.0, std::cos(ha)};  // setRotation does not normalise
    Twb.t[2] = 0;
    Prior pr;
    pr.meas = iso_from_se3(se3_mul(Twb, Tbc));
    pr.meas_inv = iso_inv(pr.meas);
    // AdjTR (src/optimizer.cpp:93-102): [[R, skew(t) R], [0, R]]
    double R[9], SR[9], A[36];
    quat_to_R(Tbc.q, R);
    const double* t = Tbc.t;
    const double S[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    mul3(S, R, SR);
    for (int k = 0; k < 36; ++k) A[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            A[r * 6 + c] = R[r * 3 + c];
            A[(r + 3) * 6 + c + 3] = R[r * 3 + c];
            A[r * 6 + c + 3] = SR[r * 3 + c];
        }
    const double d[6] = {1e-4, 1e-4, (double)p.zinfo, (double)p.xrot, (double)p.yrot, 1e-4};
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (A[k * 6 + r] * d[k]) * A[k * 6 + c];
            pr.info[r * 6 + c] = acc;
        }
    return pr;
}

// EdgeSE3Prior::computeError: toVectorMQT(Z^-1 X); J [36] (may be NULL) its derivative through oplus
void prior_error(const Prior& pr, const Iso& X, double* e, double* J) {
    const Iso E = iso_mul(pr.meas_inv, X);
    Quat q = quat_from_R(E.R);
    normalize_rotation(q);
    e[0] = E.t[0]; e[1] = E.t[1]; e[2] = E.t[2];
    e[3] = q.x; e[4] = q.y; e[5] = q.z;
    if (!J) return;
    for (int k = 0; k < 36; ++k) J[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) J[r * 6 + c] = E.R[r * 3 + c];
    // vec(q (x) (w_d, d)) = w d + w_d v + v x d: derivative w I + skew(v) at d = 0
    J[21] = q.w;  J[22] = -q.z; J[23] = q.y;
    J[27] = q.z;  J[28] = q.w;  J[29] = -q.x;
    J[33] = -q.y; J[34] = q.x;  J[35] = q.w;
}

double quad(const double* M, const double* e, int n) {
    double chi = 0;
    for (int r = 0; r < n; ++r) {
        double we = 0;
        for (int c = 0; c < n; ++c) we += M[r * n + c] * e[c];
        chi += e[r] * we;
    }
    return chi;
}

// Eigen fixed-size 3 x 3 inverse: cofactors over the determinant
void inv3(const double* m, double* o) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02, id = 1. / det;
    o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = c01 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = c02 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// dense LL^T solve of the n x n system; false when not positive definite
bool chol_solve(int n, const double* H, const double* b, double* x) {
    std::vector<double> L((size_t)n * n);
    for (int r = 0; r < n; ++r)
        for (int c = 0; c <= r; ++c) {
            double s = H[r * n + c];
            for (int k = 0; k < c; ++k) s -= L[r * n + k] * L[c * n + k];
            if (c == r) {
                if (!(s > 0.0) || !std::isfinite(s)) return false;
                L[r * n + r] = std::sqrt(s);
            } else {
                L[r * n + c] = s / L[c * n + c];
            }
        }
    for (int r = 0; r < n; ++r) {
        double s = b[r];
        for (int k = 0; k < r; ++k) s -= L[r * n + k] * x[k];
        x[r] = s / L[r * n + r];
    }
    for (int r = n - 1; r >= 0; --r) {
        double s = x[r];
        for (int k = r + 1; k < n; ++k) s -= L[k * n + r] * x[k];
        x[r] = s / L[r * n + r];
    }
    return true;
}

// inverse by LU with partial pivoting (Eigen's inverse() above 4 x 4)
void lu_inverse(int n, const double* A, double* inv) {
    std::vector<double> M(A, A + (size_t)n * n);
    for (int i = 0; i < n * n; ++i) inv[i] = 0;
    for (int i = 0; i < n; ++i) inv[i * n + i] = 1;
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int r = c + 1; r < n; ++r)
            if (std::fabs(M[r * n + c]) > std::fabs(M[piv * n + c])) piv = r;
        if (piv != c)
            for (int k = 0; k < n; ++k) { std::swap(M[c * n + k], M[piv * n + k]); std::swap(inv[c * n + k], inv[piv * n + k]); }
        const double d = M[c * n + c];
        for (int r = c + 1; r < n; ++r) {
            const double f = M[r * n + c] / d;
            for (int k = c; k < n; ++k) M[r * n + k] -= f * M[c * n + k];
            for (int k = 0; k < n; ++k) inv[r * n + k] -= f * inv[c * n + k];
        }
    }
    for (int c = n - 1; c >= 0; --c) {
        const double d = M[c * n + c];
        for (int k = 0; k < n; ++k) inv[c * n + k] /= d;
        for (int r = 0; r < c; ++r) {
            const double f = M[r * n + c];
            for (int k = 0; k < n; ++k) inv[r * n + k] -= f * inv[c * n + k];
        }
    }
}

// one-sided Jacobi SVD of a 6 x 6 matrix: A = U diag(s) V^T
void svd6(const double* A, double* U, double* s, double* V) {
    double G[36];
    std::memcpy(G, A, sizeof G);
    for (int i = 0; i < 36; ++i) V[i] = (i % 7 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < 5; ++p)
            for (int q = p + 1; q < 6; ++q) {
                double a = 0, b = 0, g = 0;
                for (int r = 0; r < 6; ++r) { a += G[r * 6 + p] * G[r * 6 + p]; b += G[r * 6 + q] * G[r * 6 + q]; g += G[r * 6 + p] * G[r * 6 + q]; }
                if (std::fabs(g) <= 1e-17 * std::sqrt(a * b) || g == 0) continue;
                rotated = true;
                const double zeta = (b - a) / (2 * g);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1 + zeta * zeta));
                const double c = 1 / std::sqrt(1 + t * t), sn = c * t;
                for (int r = 0; r < 6; ++r) {
                    const double gp = G[r * 6 + p], gq = G[r * 6 + q];
                    G[r * 6 + p] = c * gp - sn * gq; G[r * 6 + q] = sn * gp + c * gq;
                    const double vp = V[r * 6 + p], vq = V[r * 6 + q];
                    V[r * 6 + p] = c * vp - sn * vq; V[r * 6 + q] = sn * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    for (int c = 0; c < 6; ++c) {
        double n = 0;
        for (int r = 0; r < 6; ++r) n += G[r * 6 + c] * G[r * 6 + c];
        n = std::sqrt(n);
        s[c] = n;
        for (int r = 0; r < 6; ++r) U[r * 6 + c] = n > 0 ? G[r * 6 + c] / n : V[r * 6 + c];
    }
}

// the tail of Sparsifier::InfoSE3 (:235-271): symmetrise, SVD, clamp the singular values, recompose, symmetrise
void clamp_info(double* I) {
    double S[36], U[36], s[6], V[36];
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) S[r * 6 + c] = (I[r * 6 + c] + I[c * 6 + r]) / 2;
    svd6(S, U, s, V);
    for (int i = 0; i < 6; ++i) {
        double dot = 0;
        for (int r = 0; r < 6; ++r) dot += U[r * 6 + i] * V[r * 6 + i];
        if (dot >= 0) { s[i] = std::max(s[i], 1e-6); s[i] = std::min(s[i], 1e4); }
        else s[i] = -1e-6;
    }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (U[r * 6 + k] * s[k]) * V[c * 6 + k];
            S[r * 6 + c] = acc;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) I[r * 6 + c] = (S[r * 6 + c] + S[c * 6 + r]) / 2;
}

// Sparsifier::JacobianSE3XYZ: forward differences, delta 1e-6, on toMinimalVector / fromMinimalVector
void marg_jacobian(const SE3& KF, const double* MP, double* J /*3x9*/) {
    const double delta = 1e-6;
    double zref[3], v6[6];
    se3_map(se3_inv(KF), MP, zref);
    se3_to_min(KF, v6);
    for (int i = 0; i < 9; ++i) {
        double zd[3];
        if (i < 6) {
            double v[6];
            std::memcpy(v, v6, sizeof v);
            v[i] += delta;
            se3_map(se3_inv(se3_from_min(v)), MP, zd);
        } else {
            double mp[3] = {MP[0], MP[1], MP[2]};
            mp[i - 6] += delta;
            se3_map(se3_inv(KF), mp, zd);
        }
        for (int r = 0; r < 3; ++r) J[r * 9 + i] = (zd[r] - zref[r]) / delta;
    }
}

// Sparsifier::JacobianSE3: 6 x 12
void rel_jacobian(const SE3& K1, const SE3& K2, double* J) {
    const double delta = 1e-6;
    double zref[6], v1[6], v2[6];
    se3_to_min(se3_mul(se3_inv(K1), K2), zref);
    se3_to_min(K1, v1);
    se3_to_min(K2, v2);
    for (int i = 0; i < 12; ++i) {
        double v[6], zd[6];
        std::memcpy(v, i < 6 ? v1 : v2, sizeof v);
        v[i % 6] += delta;
        const SE3 Kd = se3_from_min(v);
        se3_to_min(i < 6 ? se3_mul(se3_inv(Kd), K2) : se3_mul(se3_inv(K1), Kd), zd);
        for (int r = 0; r < 6; ++r) J[r * 12 + i] = (zd[r] - zref[r]) / delta;
    }
}

// Sparsifier::DoMarginalizeSE3XYZ + InfoSE3 over the N listed points. Hm [144] (may be NULL) receives H_marginal.
void marginalize(const SE3* KF, int N, const int* idx, const double* pts, const float* z0, const float* z1, const double* o0,
                 const double* o1, bool reverse, bool cofactor, SE3* z_out, double* info36, double* Hm_out) {
    double H11[144];
    for (int k = 0; k < 144; ++k) H11[k] = 0;
    std::vector<double> H22((size_t)N * 9, 0.0), H12((size_t)N * 36, 0.0);  // H12 block of point n: 12 x 3
    for (int n0 = 0; n0 < N; ++n0) {
        const int n = reverse ? N - 1 - n0 : n0, j = idx[n];
        for (int k = 0; k < 2; ++k) {
            const double* Om = (k ? o1 : o0) + 9 * (size_t)j;
            double J[27], OJ[27];
            marg_jacobian(KF[k], pts + 3 * (size_t)j, J);
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 9; ++c) OJ[r * 9 + c] = Om[r * 3] * J[c] + Om[r * 3 + 1] * J[9 + c] + Om[r * 3 + 2] * J[18 + c];
            for (int r = 0; r < 9; ++r)
                for (int c = 0; c < 9; ++c) {
                    const double h = J[r] * OJ[c] + J[9 + r] * OJ[9 + c] + J[18 + r] * OJ[18 + c];
                    if (r < 6 && c < 6) H11[(k * 6 + r) * 12 + k * 6 + c] += h;
                    else if (r >= 6 && c >= 6) H22[(size_t)n * 9 + (r - 6) * 3 + c - 6] += h;
                    else if (r < 6) H12[(size_t)n * 36 + (k * 6 + r) * 3 + c - 6] += h;
                }
        }
    }
    for (int i = 0; i < 12; ++i) H11[i * 13] += 1e-6;
    double Hm[144];
    std::memcpy(Hm, H11, sizeof Hm);
    for (int n0 = 0; n0 < N; ++n0) {
        const int n = reverse ? N - 1 - n0 : n0;
        const double* A = &H22[(size_t)n * 9];
        if (cofactor) {  // the kernel's route, for the conditioning measurement: Y = H12 inv3(H22), Hm -= Y H21
            double Di[9];
            inv3(A, Di);
            for (int r = 0; r < 12; ++r) {
                const double* h = &H12[(size_t)n * 36 + r * 3];
                double Y[3];
                for (int c = 0; c < 3; ++c) Y[c] = h[0] * Di[c] + h[1] * Di[3 + c] + h[2] * Di[6 + c];
                for (int c = 0; c < 12; ++c) {
                    const double* g = &H12[(size_t)n * 36 + c * 3];
                    Hm[r * 12 + c] -= Y[0] * g[0] + Y[1] * g[1] + Y[2] * g[2];
                }
            }
            continue;
        }
        // LDL^T of the 3 x 3 block, then T = H22^-1 H21 column by column
        double L10, L20, L21, D0, D1, D2;
        D0 = A[0]; L10 = A[3] / D0; L20 = A[6] / D0;
        D1 = A[4] - L10 * L10 * D0; L21 = (A[7] - L20 * L10 * D0) / D1;
        D2 = A[8] - L20 * L20 * D0 - L21 * L21 * D1;
        double T[36];  // 3 x 12
        for (int c = 0; c < 12; ++c) {
            const double* h = &H12[(size_t)n * 36 + c * 3];  // H21(:, c) = H12(c, :)
            double y0 = h[0], y1 = h[1] - L10 * y0, y2 = h[2] - L20 * y0 - L21 * y1;
            y0 /= D0; y1 /= D1; y2 /= D2;
            const double x2 = y2, x1 = y1 - L21 * x2, x0 = y0 - L10 * x1 - L20 * x2;
            T[c] = x0; T[12 + c] = x1; T[24 + c] = x2;
        }
        for (int r = 0; r < 12; ++r) {
            const double* h = &H12[(size_t)n * 36 + r * 3];
            for (int c = 0; c < 12; ++c) Hm[r * 12 + c] -= h[0] * T[c] + h[1] * T[12 + c] + h[2] * T[24 + c];
        }
    }
    if (Hm_out) std::memcpy(Hm_out, Hm, sizeof Hm);
    // InfoSE3
    double J[72], Hinv[144], JH[72], C[36], I[36];
    rel_jacobian(KF[0], KF[1], J);
    lu_inverse(12, Hm, Hinv);
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 12; ++c) {
            double acc = 0;
            for (int k = 0; k < 12; ++k) acc += J[r * 12 + k] * Hinv[k * 12 + c];
            JH[r * 12 + c] = acc;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 12; ++k) acc += JH[r * 12 + k] * J[c * 12 + k];
            C[r * 6 + c] = acc;
        }
    lu_inverse(6, C, I);
    clamp_info(I);
    std::memcpy(info36, I, sizeof I);
    *z_out = se3_mul(se3_inv(KF[0]), KF[1]);
}

struct PairBA {
    Params prm;
    int mode = 0, P = 0, nfree = 0, fk[2] = {0, 0};
    bool reverse = false;
    Iso X[2], lastX[2];
    Prior prior[2];
    std::vector<double> pts, lastPts;
    const float *z[2] = {nullptr, nullptr};
    const double* om[2] = {nullptr, nullptr};
    // linearisation
    double Hpp[2][36], bp[2][6];
    std::vector<double> Hll, bl, Hpl[2];

    int pt(int j0) const { return reverse ? P - 1 - j0 : j0; }

    double edge_chi2(const Iso& Xinv, int k, int j, const double* p, double* e, double* pc) const {
        const double zz[3] = {z[k][3 * (size_t)j], z[k][3 * (size_t)j + 1], z[k][3 * (size_t)j + 2]};
        xyz_error(Xinv, p, zz, e, pc);
        return quad(om[k] + 9 * (size_t)j, e, 3);
    }
    // activeRobustChi2
    double chi2(const Iso* Xs, const std::vector<double>& ps) const {
        double chi = 0;
        for (int f = 0; f < nfree; ++f) {
            double e[6];
            prior_error(prior[fk[f]], Xs[fk[f]], e, nullptr);
            chi += quad(prior[fk[f]].info, e, 6);
        }
        const Iso Xi[2] = {iso_inv(Xs[0]), iso_inv(Xs[1])};
        const double d = prm.huber_delta, dsqr = d * d;
        for (int j0 = 0; j0 < P; ++j0) {
            const int j = pt(j0);
            for (int k = 0; k < 2; ++k) {
                double e[3], pc[3];
                const double c2 = edge_chi2(Xi[k], k, j, &ps[3 * (size_t)j], e, pc);
                chi += (c2 <= dsqr) ? c2 : 2 * std::sqrt(c2) * d - dsqr;
            }
        }
        return chi;
    }
    void build() {
        for (int k = 0; k < 2; ++k) {
            for (int i = 0; i < 36; ++i) Hpp[k][i] = 0;
            for (int i = 0; i < 6; ++i) bp[k][i] = 0;
        }
        Hll.assign((size_t)P * 9, 0.0); bl.assign((size_t)P * 3, 0.0);
        Hpl[0].assign((size_t)P * 18, 0.0); Hpl[1].assign((size_t)P * 18, 0.0);
        for (int f = 0; f < nfree; ++f) {  // BaseUnaryEdge: H += J^T Omega J, b -= J^T Omega e
            const int k = fk[f];
            double e[6], J[36], OJ[36], Oe[6];
            prior_error(prior[k], X[k], e, J);
            for (int r = 0; r < 6; ++r) {
                Oe[r] = 0;
                for (int c = 0; c < 6; ++c) {
                    Oe[r] += prior[k].info[r * 6 + c] * e[c];
                    double acc = 0;
                    for (int m = 0; m < 6; ++m) acc += prior[k].info[r * 6 + m] * J[m * 6 + c];
                    OJ[r * 6 + c] = acc;
                }
            }
            for (int r = 0; r < 6; ++r) {
                for (int c = 0; c < 6; ++c) {
                    double acc = 0;
                    for (int m = 0; m < 6; ++m) acc += J[m * 6 + r] * OJ[m * 6 + c];
                    Hpp[k][r * 6 + c] += acc;
                }
                double acc = 0;
                for (int m = 0; m < 6; ++m) acc += J[m * 6 + r] * Oe[m];
                bp[k][r] -= acc;
            }
        }
        const Iso Xi[2] = {iso_inv(X[0]), iso_inv(X[1])};
        const double d = prm.huber_delta, dsqr = d * d;
        for (int j0 = 0; j0 < P; ++j0) {
            const int j = pt(j0);
            for (int k = 0; k < 2; ++k) {
                double e[3], pc[3], Jp[18], Jl[9];
                const double c2 = edge_chi2(Xi[k], k, j, &pts[3 * (size_t)j], e, pc);
                const double rho1 = (c2 <= dsqr) ? 1.0 : d / std::sqrt(c2);
                xyz_jacobians(Xi[k], pc, Jp, Jl);
                const double* Om = om[k] + 9 * (size_t)j;
                double W[9], We[3];
                for (int i = 0; i < 9; ++i) W[i] = rho1 * Om[i];
                mulv3(W, e, We);
                const bool free_k = !(mode == 0 && k == 0);
                double WJl[9];
                mul3(W, Jl, WJl);
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c)
                        Hll[(size_t)j * 9 + r * 3 + c] += Jl[r] * WJl[c] + Jl[3 + r] * WJl[3 + c] + Jl[6 + r] * WJl[6 + c];
                    bl[(size_t)j * 3 + r] -= Jl[r] * We[0] + Jl[3 + r] * We[1] + Jl[6 + r] * We[2];
                }
                if (!free_k) continue;
                double WJp[18];
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 6; ++c) WJp[r * 6 + c] = W[r * 3] * Jp[c] + W[r * 3 + 1] * Jp[6 + c] + W[r * 3 + 2] * Jp[12 + c];
                for (int r = 0; r < 6; ++r) {
                    for (int c = 0; c < 6; ++c) Hpp[k][r * 6 + c] += Jp[r] * WJp[c] + Jp[6 + r] * WJp[6 + c] + Jp[12 + r] * WJp[12 + c];
                    for (int c = 0; c < 3; ++c)
                        Hpl[k][(size_t)j * 18 + r * 3 + c] += Jp[r] * WJl[c] + Jp[6 + r] * WJl[3 + c] + Jp[12 + r] * WJl[6 + c];
                    bp[k][r] -= Jp[r] * We[0] + Jp[6 + r] * We[1] + Jp[12 + r] * We[2];
                }
            }
        }
    }
    double maxDiag() const {  // computeLambdaInit over every free vertex
        double m = 0;
        for (int f = 0; f < nfree; ++f)
            for (int i = 0; i < 6; ++i) m = std::max(m, std::fabs(Hpp[fk[f]][i * 7]));
        for (int j = 0; j < P; ++j)
            for (int i = 0; i < 3; ++i) m = std::max(m, std::fabs(Hll[(size_t)j * 9 + i * 4]));
        return m;
    }
    // BlockSolver::solve with lambda on both diagonals; xp [6*nfree], xl [3P]; scale = computeScale
    bool solve(double lambda, double* xp, std::vector<double>& xl, double* scale) const {
        const int n = 6 * nfree;
        std::vector<double> Hs((size_t)n * n, 0.0), bs(n, 0.0), Dinv((size_t)P * 9);
        for (int f = 0; f < nfree; ++f)
            for (int r = 0; r < 6; ++r) {
                for (int c = 0; c < 6; ++c) Hs[(f * 6 + r) * n + f * 6 + c] = Hpp[fk[f]][r * 6 + c] + (r == c ? lambda : 0.0);
                bs[f * 6 + r] = bp[fk[f]][r];
            }
        for (int j0 = 0; j0 < P; ++j0) {
            const int j = pt(j0);
            double D[9];
            for (int i = 0; i < 9; ++i) D[i] = Hll[(size_t)j * 9 + i] + (i % 4 == 0 ? lambda : 0.0);
            double* Di = &Dinv[(size_t)j * 9];
            inv3(D, Di);
            double Y[2][18], yb[3];  // Y = Hpl Dinv (6 x 3)
            mulv3(Di, &bl[(size_t)j * 3], yb);
            for (int f = 0; f < nfree; ++f) {
                const double* h = &Hpl[fk[f]][(size_t)j * 18];
                for (int r = 0; r < 6; ++r)
                    for (int c = 0; c < 3; ++c) Y[f][r * 3 + c] = h[r * 3] * Di[c] + h[r * 3 + 1] * Di[3 + c] + h[r * 3 + 2] * Di[6 + c];
            }
            for (int f = 0; f < nfree; ++f) {
                const double* h = &Hpl[fk[f]][(size_t)j * 18];
                for (int r = 0; r < 6; ++r) {
                    bs[f * 6 + r] -= h[r * 3] * yb[0] + h[r * 3 + 1] * yb[1] + h[r * 3 + 2] * yb[2];
                    for (int g = 0; g < nfree; ++g) {
                        const double* h2 = &Hpl[fk[g]][(size_t)j * 18];
                        for (int c = 0; c < 6; ++c)
                            Hs[(f * 6 + r) * n + g * 6 + c] -= Y[f][r * 3] * h2[c * 3] + Y[f][r * 3 + 1] * h2[c * 3 + 1] + Y[f][r * 3 + 2] * h2[c * 3 + 2];
                    }
                }
            }
        }
        if (!chol_solve(n, Hs.data(), bs.data(), xp)) return false;
        double sc = 0;
        for (int f = 0; f < nfree; ++f)
            for (int r = 0; r < 6; ++r) sc += xp[f * 6 + r] * (lambda * xp[f * 6 + r] + bp[fk[f]][r]);
        for (int j0 = 0; j0 < P; ++j0) {
            const int j = pt(j0);
            double rhs[3];
            for (int c = 0; c < 3; ++c) {
                double acc = bl[(size_t)j * 3 + c];
                for (int f = 0; f < nfree; ++f) {
                    const double* h = &Hpl[fk[f]][(size_t)j * 18];
                    for (int r = 0; r < 6; ++r) acc -= h[r * 3 + c] * xp[f * 6 + r];
                }
                rhs[c] = acc;
            }
            mulv3(&Dinv[(size_t)j * 9], rhs, &xl[(size_t)j * 3]);
            for (int c = 0; c < 3; ++c) sc += xl[(size_t)j * 3 + c] * (lambda * xl[(size_t)j * 3 + c] + bl[(size_t)j * 3 + c]);
        }
        *scale = sc;
        return true;
    }

    int optimize(int iterations, IterStats* stats, double* trace, int* not_pd) {
        *not_pd = 0;
        double lambda = 0, ni = 2;
        int done = 0;
        bool ok = true;
        std::vector<double> xl((size_t)P * 3);
        for (int it = 0; it < iterations && ok; ++it) {
            IterStats st{};
            double currentChi = chi2(X, pts);
            lastX[0] = X[0]; lastX[1] = X[1]; lastPts = pts;
            st.chi2_before = currentChi;
            build();
            if (it == 0) { lambda = 1e-5 * maxDiag(); ni = 2; }
            double rho = 0;
            int qmax = 0, failed = 0;
            do {
                const Iso bak[2] = {X[0], X[1]};
                const std::vector<double> bakp = pts;
                double xp[12], scale = 0;
                const bool ok2 = solve(lambda, xp, xl, &scale);
                double tempChi = std::numeric_limits<double>::max();
                if (ok2) {
                    for (int f = 0; f < nfree; ++f) X[fk[f]] = oplus(X[fk[f]], xp + 6 * f);
                    for (size_t i = 0; i < pts.size(); ++i) pts[i] += xl[i];
                    tempChi = chi2(X, pts);
                    lastX[0] = X[0]; lastX[1] = X[1]; lastPts = pts;
                } else {
                    ++failed;
                }
                rho = (currentChi - tempChi) / (scale + 1e-3);
                if (rho > 0 && std::isfinite(tempChi)) {
                    double alpha = 1. - std::pow((2 * rho - 1), 3);
                    alpha = std::min(alpha, 2. / 3.);
                    lambda *= std::max(1. / 3., alpha);
                    ni = 2;
                    currentChi = tempChi;
                    st.accepted = 1;
                } else {
                    lambda *= ni;
                    ni *= 2;
                    X[0] = bak[0]; X[1] = bak[1]; pts = bakp;
                }
                qmax++;
            } while (rho < 0 && qmax < 10);
            st.chi2_after = currentChi; st.lambda = lambda; st.rho = rho; st.trials = qmax;
            st.terminate = (qmax == 10 || rho == 0) ? 1 : 0;
            ok = !st.terminate;
            if (st.terminate && failed == qmax) *not_pd = 1;
            if (stats) stats[it] = st;
            if (trace)
                for (int k = 0; k < 2; ++k) {
                    std::memcpy(trace + 24 * (size_t)it + 12 * k, X[k].R, 9 * sizeof(double));
                    std::memcpy(trace + 24 * (size_t)it + 12 * k + 9, X[k].t, 3 * sizeof(double));
                }
            ++done;
        }
        return done;
    }
};

void pose_out(const SE3& T, double* p7) {
    p7[0] = T.q.x; p7[1] = T.q.y; p7[2] = T.q.z; p7[3] = T.q.w;
    p7[4] = T.t[0]; p7[5] = T.t[1]; p7[6] = T.t[2];
}

void iso_in(const double* v12, Iso* X) { std::memcpy(X->R, v12, 9 * sizeof(double)); std::memcpy(X->t, v12 + 9, 3 * sizeof(double)); }
void iso_out(const Iso& X, double* v12) { std::memcpy(v12, X.R, 9 * sizeof(double)); std::memcpy(v12 + 9, X.t, 3 * sizeof(double)); }

}  // namespace

extern "C" {

// One keyframe pair. mode 0 = CreateFeatEdge(from, to, cnstr), mode 1 = CreateFeatEdge(from, to, mapMatch, cnstr).
// Tcw0 / Tcw1 [16] float row-major; per point j < P: xyz [3] float (the start estimate), z0 / z1 [3] float (mViewMPs in
// keyframe 0 / 1), info0 / info1 [9] double (mViewMPsInfo). Outputs, untouched when the status is 1: measure [16] and info
// [36] float, outlier [P] bytes (mode 1), poses [14] (vSe3KFs as qx, qy, qz, qw, tx, ty, tz), points [3P] (every point's
// estimate, outliers included). stats [iterations] / trace [iterations*24] (R row-major, t per keyframe) / Hm [144] may be
// NULL. reverse & 1 runs every per-point sum in descending point order, reverse & 2 takes the Schur complement of the
// marginalisation through the cofactor inverse instead of LDL^T (both for the conditioning measurement).
// Returns the LM iterations done; *status: 0 OK, 1 too few points, 2 the last iteration failed every factorisation.
int feat_edge_oracle_run(int mode, const float* Tcw0, const float* Tcw1, int P, const float* xyz, const float* z0, const float* z1,
                         const double* info0, const double* info1, const void* params, float* measure, float* info,
                         uint8_t* outlier, double* poses, double* points, void* stats, double* trace, double* Hm, int reverse,
                         int* status) {
    PairBA b;
    std::memcpy(&b.prm, params, sizeof(Params));
    b.mode = mode; b.P = P; b.reverse = (reverse & 1) != 0;
    if (P < b.prm.min_points[mode]) { *status = 1; return 0; }
    b.X[0] = iso_from_Tcw(Tcw0);
    b.X[1] = iso_from_Tcw(Tcw1);
    if (mode == 0) { b.nfree = 1; b.fk[0] = 1; }
    else { b.nfree = 2; b.fk[0] = 0; b.fk[1] = 1; }
    for (int f = 0; f < b.nfree; ++f) b.prior[b.fk[f]] = plane_motion_prior(b.X[b.fk[f]], b.prm);
    b.pts.resize((size_t)P * 3);
    for (size_t i = 0; i < b.pts.size(); ++i) b.pts[i] = xyz[i];
    b.z[0] = z0; b.z[1] = z1; b.om[0] = info0; b.om[1] = info1;
    b.lastX[0] = b.X[0]; b.lastX[1] = b.X[1]; b.lastPts = b.pts;
    int not_pd = 0;
    const int done = b.optimize(b.prm.iterations[mode], (IterStats*)stats, trace, &not_pd);
    *status = not_pd ? 2 : 0;
    std::vector<int> keep;
    if (mode == 1) {  // EdgeSE3PointXYZ::chi2() on the errors of the last evaluated trial
        const Iso Xi[2] = {iso_inv(b.lastX[0]), iso_inv(b.lastX[1])};
        for (int j = 0; j < P; ++j) {
            bool out = false;
            for (int k = 0; k < 2; ++k) {
                double e[3], pc[3];
                if (b.edge_chi2(Xi[k], k, j, &b.lastPts[3 * (size_t)j], e, pc) > (double)b.prm.chi2_cut) out = true;
            }
            if (outlier) outlier[j] = out;
            if (!out) keep.push_back(j);
        }
    } else {
        for (int j = 0; j < P; ++j) keep.push_back(j);
    }
    const SE3 KF[2] = {se3_from_iso(b.X[0]), se3_from_iso(b.X[1])};
    SE3 zo;
    double I[36];
    marginalize(KF, (int)keep.size(), keep.data(), b.pts.data(), z0, z1, info0, info1, b.reverse, (reverse & 2) != 0, &zo, I, Hm);
    double R[9];  // converter.cpp toCvMat(SE3Quat) / toCvMat6f
    quat_to_R(zo.q, R);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) measure[r * 4 + c] = (float)R[r * 3 + c];
        measure[r * 4 + 3] = (float)zo.t[r];
    }
    measure[12] = 0; measure[13] = 0; measure[14] = 0; measure[15] = 1;
    for (int i = 0; i < 36; ++i) info[i] = (float)I[i];
    if (poses) { pose_out(KF[0], poses); pose_out(KF[1], poses + 7); }
    if (points) std::memcpy(points, b.pts.data(), b.pts.size() * sizeof(double));
    return done;
}

// Single pieces for the self-consistency tests. An isometry is 12 doubles: R row-major, then t.
void feat_edge_oracle_from_Tcw(const float* Tcw, double* X12) { iso_out(iso_from_Tcw(Tcw), X12); }
void feat_edge_oracle_oplus(const double* X12, const double* d6, double* out12) {
    Iso X; iso_in(X12, &X);
    iso_out(oplus(X, d6), out12);
}
// EdgeSE3PointXYZ at X: error [3], pose Jacobian [3x6], point Jacobian [3x3]
void feat_edge_oracle_xyz_edge(const double* X12, const double* p, const double* z, double* e, double* Jp, double* Jl) {
    Iso X; iso_in(X12, &X);
    const Iso Xi = iso_inv(X);
    double pc[3];
    xyz_error(Xi, p, z, e, pc);
    xyz_jacobians(Xi, pc, Jp, Jl);
}
// addVertexSE3PlaneMotion at X0: measurement [12] and information [36]; EdgeSE3Prior at X: error [6] and Jacobian [6x6]
void feat_edge_oracle_prior(const double* X0_12, const void* params, const double* X12, double* meas12, double* info36, double* e,
                            double* J) {
    Params p;
    std::memcpy(&p, params, sizeof p);
    Iso X0, X; iso_in(X0_12, &X0); iso_in(X12, &X);
    const Prior pr = plane_motion_prior(X0, p);
    iso_out(pr.meas, meas12);
    std::memcpy(info36, pr.info, sizeof pr.info);
    prior_error(pr, X, e, J);
}
// the singular-value clamp of InfoSE3 on a 6 x 6 matrix, in place
void feat_edge_oracle_clamp(double* I36) { clamp_info(I36); }

}  // extern "C"
