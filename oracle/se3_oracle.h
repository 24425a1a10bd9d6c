// SE(3) algebra of the BA oracles — TEST INFRASTRUCTURE ONLY.
//
// g2o (tag 20160424) and Eigen (3.3) are not vendored; their published definitions are restated: SE3Quat (exp with its
// theta < 1e-5 branch, log with its d > 0.99999 branch, operator*, inverse, adj, normalizeRotation), Eigen's
// Quaterniond(Matrix3d), Quaterniond * Vector3d, quaternion product, toRotationMatrix and AngleAxisd(Quaterniond),
// Isometry3d products and inverse, VertexSE3's MQT oplus, toSE3Quat, EdgeProjectXYZ2UV's error and Jacobians, and the
// two plane-motion priors of the reference (addPlaneMotionSE3Expmap on a VertexSE3Expmap, addVertexSE3PlaneMotion's
// EdgeSE3Prior on a VertexSE3). Each oracle library is one translation unit, so everything here has internal linkage.
#pragma once

#include <cmath>
#include <cstring>

namespace {

struct Quat { double x, y, z, w; };
struct SE3 { Quat q; double t[3]; };   // g2o::SE3Quat
struct Iso { double R[9], t[3]; };     // Eigen::Isometry3d: rotation row-major, translation

void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

void skew(const double* v, double* S) {
    S[0] = 0;     S[1] = -v[2]; S[2] = v[1];
    S[3] = v[2];  S[4] = 0;     S[5] = -v[0];
    S[6] = -v[1]; S[7] = v[0];  S[8] = 0;
}

void mul3(const double* A, const double* B, double* C) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

void mulv3(const double* A, const double* v, double* o) {
    for (int r = 0; r < 3; ++r) o[r] = A[r * 3] * v[0] + A[r * 3 + 1] * v[1] + A[r * 3 + 2] * v[2];
}

// e^T M e of an n x n information matrix
double quad(const double* M, const double* e, int n) {
    double chi = 0;
    for (int r = 0; r < n; ++r) {
        double we = 0;
        for (int c = 0; c < n; ++c) we += M[r * n + c] * e[c];
        chi += e[r] * we;
    }
    return chi;
}

// Eigen: Quaternion<double>(const Matrix3d&) (quaternion_from_matrix)
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

// Eigen: quat_product
Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// Eigen: QuaternionBase::_transformVector (q * v)
void qrot(const Quat& q, const double* v, double* out) {
    const double qv[3] = {q.x, q.y, q.z};
    double uv[3], c[3];
    cross(qv, v, uv);
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    cross(qv, uv, c);
    for (int i = 0; i < 3; ++i) out[i] = v[i] + q.w * uv[i] + c[i];
}

// g2o SE3Quat::normalizeRotation: w >= 0, then Eigen normalize()
void normalize_rotation(Quat& q) {
    if (q.w < 0) { q.x = -q.x; q.y = -q.y; q.z = -q.z; q.w = -q.w; }
    const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    if (n2 > 0) {
        const double n = std::sqrt(n2);
        q.x /= n; q.y /= n; q.z /= n; q.w /= n;
    }
}

// g2o SE3Quat(const Matrix3d& R, const Vector3d& t)
SE3 se3_from_Rt(const double* R, const double* t) {
    SE3 T;
    T.q = quat_from_R(R);
    for (int i = 0; i < 3; ++i) T.t[i] = t[i];
    normalize_rotation(T.q);
    return T;
}

// converter.cpp toSE3Quat(cv::Mat): float 4x4 row-major
SE3 se3_from_f32(const float* T) {
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    const double t[3] = {T[3], T[7], T[11]};
    return se3_from_Rt(R, t);
}

// g2o SE3Quat::operator*
SE3 se3_mul(const SE3& a, const SE3& b) {
    SE3 r = a;
    double rt[3];
    qrot(a.q, b.t, rt);
    for (int i = 0; i < 3; ++i) r.t[i] += rt[i];
    r.q = qmul(a.q, b.q);
    normalize_rotation(r.q);
    return r;
}

// g2o SE3Quat::inverse
SE3 se3_inv(const SE3& a) {
    SE3 r;
    r.q = {-a.q.x, -a.q.y, -a.q.z, a.q.w};
    const double mt[3] = {a.t[0] * -1., a.t[1] * -1., a.t[2] * -1.};
    qrot(r.q, mt, r.t);
    return r;
}

// g2o SE3Quat::exp, update ordered [omega, upsilon]
SE3 se3_exp(const double* u) {
    const double* omega = u;
    const double* upsilon = u + 3;
    const double theta = std::sqrt(omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2]);
    double O[9], O2[9], R[9], V[9];
    skew(omega, O);
    mul3(O, O, O2);
    if (theta < 0.00001) {
        for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0 ? 1.0 : 0.0) + O[k] + O2[k];
        std::memcpy(V, R, sizeof R);
    } else {
        const double s = std::sin(theta), c = std::cos(theta);
        const double a = s / theta, b = (1 - c) / (theta * theta), d = (theta - s) / std::pow(theta, 3);
        for (int k = 0; k < 9; ++k) {
            const double I = (k % 4 == 0 ? 1.0 : 0.0);
            R[k] = I + a * O[k] + b * O2[k];
            V[k] = I + b * O[k] + d * O2[k];
        }
    }
    double t[3];
    for (int r = 0; r < 3; ++r) t[r] = V[r * 3] * upsilon[0] + V[r * 3 + 1] * upsilon[1] + V[r * 3 + 2] * upsilon[2];
    SE3 T;
    T.q = quat_from_R(R);
    std::memcpy(T.t, t, sizeof t);
    normalize_rotation(T.q);
    return T;
}

// g2o SE3Quat::log
void se3_log(const SE3& T, double* res) {
    double R[9];
    quat_to_R(T.q, R);
    const double d = 0.5 * (R[0] + R[4] + R[8] - 1);
    const double dR[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    double omega[3], O[9], O2[9], Vinv[9];
    double f;
    if (d > 0.99999) {
        for (int i = 0; i < 3; ++i) omega[i] = 0.5 * dR[i];
        skew(omega, O);
        mul3(O, O, O2);
        for (int k = 0; k < 9; ++k) Vinv[k] = (k % 4 == 0 ? 1.0 : 0.0) - 0.5 * O[k] + (1. / 12.) * O2[k];
    } else {
        const double theta = std::acos(d);
        const double s = theta / (2 * std::sqrt(1 - d * d));
        for (int i = 0; i < 3; ++i) omega[i] = s * dR[i];
        skew(omega, O);
        mul3(O, O, O2);
        f = (1 - theta / (2 * std::tan(theta / 2))) / (theta * theta);
        for (int k = 0; k < 9; ++k) Vinv[k] = (k % 4 == 0 ? 1.0 : 0.0) - 0.5 * O[k] + f * O2[k];
    }
    for (int i = 0; i < 3; ++i) res[i] = omega[i];
    for (int r = 0; r < 3; ++r) res[3 + r] = Vinv[r * 3] * T.t[0] + Vinv[r * 3 + 1] * T.t[1] + Vinv[r * 3 + 2] * T.t[2];
}

// g2o SE3Quat::adj: [[R, 0], [skew(t) R, R]]
void se3_adj(const SE3& T, double* A) {
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

// poses as 7 doubles (qx, qy, qz, qw, tx, ty, tz)
void pose_out(const SE3& T, double* pose7) {
    pose7[0] = T.q.x; pose7[1] = T.q.y; pose7[2] = T.q.z; pose7[3] = T.q.w;
    pose7[4] = T.t[0]; pose7[5] = T.t[1]; pose7[6] = T.t[2];
}
SE3 pose_in(const double* p) { return {{p[0], p[1], p[2], p[3]}, {p[4], p[5], p[6]}}; }

// converter.cpp toCvMat(SE3Quat): to_homogeneous_matrix narrowed to float
void to_f32(const SE3& T, float* M) {
    double R[9];
    quat_to_R(T.q, R);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) M[r * 4 + c] = (float)R[r * 3 + c];
        M[r * 4 + 3] = (float)T.t[r];
    }
    M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
}

// Eigen::AngleAxisd(Quaterniond) (Eigen 3.3), then angle * axis_z: the yaw the plane-motion priors keep
double yaw_of(const Quat& q) {
    double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z), angle = 0, axis_z = 0;
    if (n != 0) {
        angle = 2 * std::atan2(n, std::fabs(q.w));
        if (q.w < 0) n = -n;
        axis_z = q.z / n;
    }
    return angle * axis_z;
}

// Quaterniond(AngleAxisd(yaw, UnitZ)); SE3Quat::setRotation does not normalise
Quat quat_yaw(double yaw) {
    const double ha = 0.5 * yaw, s = std::sin(ha);
    return {s * 0.0, s * 0.0, s * 1.0, std::cos(ha)};
}

// addPlaneMotionSE3Expmap (src/optimizer.cpp:236-314, non-USE_EULER branch): measurement and symmetric information of
// the EdgeSE3ExpmapPrior on a VertexSE3Expmap at pose
void plane_prior_expmap(const SE3& pose, const float* Tbc_f, float xrot, float yrot, float zinfo, SE3* meas, double* info) {
    const SE3 Tbc = se3_from_f32(Tbc_f);
    SE3 Tbw = se3_mul(Tbc, pose);
    Tbw.q = quat_yaw(yaw_of(Tbw.q));
    Tbw.t[2] = 0;
    *meas = se3_mul(se3_inv(Tbc), Tbw);
    double J[36], JtI[36];
    se3_adj(Tbc, J);
    const double d[6] = {(double)xrot, (double)yrot, 1e-4, 1e-4, 1e-4, (double)zinfo};
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) JtI[r * 6 + c] = J[c * 6 + r] * d[c];
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += JtI[r * 6 + k] * J[k * 6 + c];
            info[r * 6 + c] = acc;
        }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < i; ++j) info[i * 6 + j] = info[j * 6 + i];
}

// EdgeSE3ExpmapPrior::computeError: log(meas * T^-1); its Jacobian is the constant -I
void expmap_prior_error(const SE3& meas, const SE3& T, double* e) { se3_log(se3_mul(meas, se3_inv(T)), e); }

// EdgeProjectXYZ2UV::computeError: obs - cam_map(T.map(X)) with CameraParameters(fx, (cx, cy), 0); pc [3] receives T.map(X).
// Jp [2x6] (may be NULL): the pose block of linearizeOplus
void proj_error(const SE3& T, const double* X, const double* obs, double fx, double cx, double cy, double* err, double* pc,
                double* Jp) {
    qrot(T.q, X, pc);
    for (int i = 0; i < 3; ++i) pc[i] += T.t[i];
    err[0] = obs[0] - ((pc[0] / pc[2]) * fx + cx);
    err[1] = obs[1] - ((pc[1] / pc[2]) * fx + cy);
    if (!Jp) return;
    const double x = pc[0], y = pc[1], z = pc[2], z2 = z * z;
    Jp[0] = x * y / z2 * fx;        Jp[1] = -(1 + (x * x / z2)) * fx; Jp[2] = y / z * fx;
    Jp[3] = -1. / z * fx;           Jp[4] = 0;                        Jp[5] = x / z2 * fx;
    Jp[6] = (1 + y * y / z2) * fx;  Jp[7] = -x * y / z2 * fx;         Jp[8] = -x / z * fx;
    Jp[9] = 0;                      Jp[10] = -1. / z * fx;            Jp[11] = y / z2 * fx;
}

// its point block [2x3]: -1/z [[fx, 0, -x/z fx], [0, fx, -y/z fx]] R at pc = T.map(X)
void proj_point_block(const SE3& T, const double* pc, double fx, double* Jl) {
    const double x = pc[0], y = pc[1], z = pc[2];
    double R[9];
    quat_to_R(T.q, R);
    const double iz = -1. / z;
    const double tmp[6] = {iz * fx, iz * 0.0, iz * (-x / z * fx), iz * 0.0, iz * fx, iz * (-y / z * fx)};
    for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 3; ++c) Jl[r * 3 + c] = tmp[r * 3] * R[c] + tmp[r * 3 + 1] * R[3 + c] + tmp[r * 3 + 2] * R[6 + c];
}

// ---- VertexSE3 (Isometry3d estimate)

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

// an isometry as 12 doubles: R row-major, then t
void iso_in(const double* v12, Iso* X) { std::memcpy(X->R, v12, 9 * sizeof(double)); std::memcpy(X->t, v12 + 9, 3 * sizeof(double)); }
void iso_out(const Iso& X, double* v12) { std::memcpy(v12, X.R, 9 * sizeof(double)); std::memcpy(v12 + 9, X.t, 3 * sizeof(double)); }

struct Prior {  // EdgeSE3Prior with an identity ParameterSE3Offset
    Iso meas, meas_inv;
    double info[36];
};

// addVertexSE3PlaneMotion (src/optimizer.cpp:429-455, non-USE_OLD_SE3_PRIOR_JACOB branch) at pose
Prior plane_prior_se3(const Iso& pose, const float* Tbc_f, float xrot, float yrot, float zinfo) {
    const SE3 Tbc = se3_from_f32(Tbc_f);
    SE3 Twb = se3_mul(se3_from_iso(pose), se3_inv(Tbc));
    Twb.q = quat_yaw(yaw_of(Twb.q));
    Twb.t[2] = 0;
    Prior pr;
    pr.meas = iso_from_se3(se3_mul(Twb, Tbc));
    pr.meas_inv = iso_inv(pr.meas);
    // AdjTR (src/optimizer.cpp:93-102): [[R, skew(t) R], [0, R]]
    double R[9], S[9], SR[9], A[36];
    quat_to_R(Tbc.q, R);
    skew(Tbc.t, S);
    mul3(S, R, SR);
    for (int k = 0; k < 36; ++k) A[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            A[r * 6 + c] = R[r * 3 + c];
            A[(r + 3) * 6 + c + 3] = R[r * 3 + c];
            A[r * 6 + c + 3] = SR[r * 3 + c];
        }
    const double d[6] = {1e-4, 1e-4, (double)zinfo, (double)xrot, (double)yrot, 1e-4};
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (A[k * 6 + r] * d[k]) * A[k * 6 + c];
            pr.info[r * 6 + c] = acc;
        }
    return pr;
}

// EdgeSE3Prior::computeError: toVectorMQT(Z^-1 X); J [36] (may be NULL) its derivative through oplus
void se3_prior_error(const Prior& pr, const Iso& X, double* e, double* J) {
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

}  // namespace
