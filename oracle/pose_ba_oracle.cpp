// Pose-only SE(3) bundle adjustment ORACLE (Localizer::DoLocalBA) — TEST INFRASTRUCTURE ONLY.
//
// Sequential double-precision restatement of what the reference's Localizer::DoLocalBA (src/Localizer.cpp:233-302)
// hands to g2o: one VertexSE3Expmap (estimate toSE3Quat(Tcw)), one EdgeSE3ExpmapPrior built by addPlaneMotionSE3Expmap
// (src/optimizer.cpp:236-314, non-USE_EULER branch; error log(meas * est^-1), Jacobian the constant -I of :181-189),
// and one EdgeProjectXYZ2UV per observed map point (fixed VertexSBAPointXYZ, CameraParameters(fx, (cx, cy), 0),
// information w_e * I, RobustKernelHuber(delta)), then initializeOptimization(0); optimize(iterations).
//
// g2o (tag 20160424) and Eigen are not vendored; their published algorithms are restated: SE3Quat (exp with its
// theta < 1e-5 branch, log with its d > 0.99999 branch, operator*, inverse, map, adj, normalizeRotation),
// Eigen's Quaterniond(Matrix3d), Quaterniond * Vector3d, quaternion product, toRotationMatrix and AngleAxisd(Quaterniond)
// (Eigen 3.3), EdgeProjectXYZ2UV::computeError / linearizeOplus (pose block), BaseUnaryEdge / BaseBinaryEdge
// constructQuadraticForm with the Huber weighting rho'(e) * Omega, and OptimizationAlgorithmLevenberg::solve exactly as
// oracle/ba_oracle.cpp restates it (tau 1e-5, nu schedule, 10 trials, rho test, Terminate on 10 failed trials or rho == 0).
// The pose system is 6 x 6 and is factorised with a dense LL^T (what CHOLMOD does on it).
// PARITY UNPINNED against real g2o (no g2o build exists here); pinned by self-consistency in tests/test_pose_ba_oracle.py
// (numeric Jacobians, exp/log round trips, an independent numpy restatement in oracle/pose_ba_numpy.py).
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

struct Quat { double x, y, z, w; };
struct SE3 { Quat q; double t[3]; };

void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
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

void skew(const double* v, double* S) {
    S[0] = 0;     S[1] = -v[2]; S[2] = v[1];
    S[3] = v[2];  S[4] = 0;     S[5] = -v[0];
    S[6] = -v[1]; S[7] = v[0];  S[8] = 0;
}

void mul3(const double* A, const double* B, double* C) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
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

// addPlaneMotionSE3Expmap (src/optimizer.cpp:236-314, non-USE_EULER branch): measurement and symmetric information
void plane_motion_prior(const SE3& pose, const float* Tbc_f, float xrot, float yrot, float zinfo, SE3* meas, double* info) {
    const SE3 Tbc = se3_from_f32(Tbc_f);
    SE3 Tbw = se3_mul(Tbc, pose);
    // Eigen::AngleAxisd(Quaterniond) (Eigen 3.3), then angle * axis
    const Quat& q = Tbw.q;
    double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    double angle, axis_z;
    if (n != 0) {
        angle = 2 * std::atan2(n, std::fabs(q.w));
        if (q.w < 0) n = -n;
        axis_z = q.z / n;
    } else {
        angle = 0; axis_z = 0;
    }
    const double yaw = angle * axis_z;
    // Quaterniond(AngleAxisd(yaw, UnitZ)); SE3Quat::setRotation does not normalise
    const double ha = 0.5 * yaw, s = std::sin(ha);
    Tbw.q = {s * 0.0, s * 0.0, s * 1.0, std::cos(ha)};
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

struct PoseBA {
    SE3 est;
    SE3 meas;
    double prior_info[36];
    int E = 0;
    std::vector<double> xyz, uv, w;
    double fx, cx, cy, delta;

    // EdgeProjectXYZ2UV::computeError: obs - cam_map(T.map(xyz)); optionally the pose block of linearizeOplus
    void proj_edge(const SE3& T, int e, double* err, double* J /*2x6*/) const {
        double p[3];
        qrot(T.q, &xyz[3 * (size_t)e], p);
        for (int i = 0; i < 3; ++i) p[i] += T.t[i];
        err[0] = uv[2 * (size_t)e] - ((p[0] / p[2]) * fx + cx);
        err[1] = uv[2 * (size_t)e + 1] - ((p[1] / p[2]) * fx + cy);
        if (!J) return;
        const double x = p[0], y = p[1], z = p[2], z2 = z * z;
        J[0] = x * y / z2 * fx;        J[1] = -(1 + (x * x / z2)) * fx; J[2] = y / z * fx;
        J[3] = -1. / z * fx;           J[4] = 0;                        J[5] = x / z2 * fx;
        J[6] = (1 + y * y / z2) * fx;  J[7] = -x * y / z2 * fx;         J[8] = -x / z * fx;
        J[9] = 0;                      J[10] = -1. / z * fx;            J[11] = y / z2 * fx;
    }
    void prior_error(const SE3& T, double* e) const { se3_log(se3_mul(meas, se3_inv(T)), e); }
    double prior_chi2(const double* e) const {
        double chi = 0;
        for (int r = 0; r < 6; ++r) {
            double we = 0;
            for (int c = 0; c < 6; ++c) we += prior_info[r * 6 + c] * e[c];
            chi += e[r] * we;
        }
        return chi;
    }
    // activeRobustChi2: the prior (edge added first) then every projection edge through RobustKernelHuber
    double chi2(const SE3& T) const {
        double e6[6];
        prior_error(T, e6);
        double chi = prior_chi2(e6);
        const double dsqr = delta * delta;
        for (int k = 0; k < E; ++k) {
            double e[2];
            proj_edge(T, k, e, nullptr);
            const double c2 = e[0] * (w[k] * e[0]) + e[1] * (w[k] * e[1]);
            chi += (c2 <= dsqr) ? c2 : 2 * std::sqrt(c2) * delta - dsqr;
        }
        return chi;
    }
    // buildSystem: H [36] full symmetric, b [6]
    void build(double* H, double* b) const {
        double e6[6];
        prior_error(est, e6);
        // BaseUnaryEdge with J = -I: H += Omega, b -= J^T Omega e = Omega e
        for (int r = 0; r < 6; ++r) {
            double we = 0;
            for (int c = 0; c < 6; ++c) { H[r * 6 + c] = prior_info[r * 6 + c]; we += prior_info[r * 6 + c] * e6[c]; }
            b[r] = we;
        }
        const double dsqr = delta * delta;
        for (int k = 0; k < E; ++k) {
            double e[2], J[12];
            proj_edge(est, k, e, J);
            const double c2 = e[0] * (w[k] * e[0]) + e[1] * (w[k] * e[1]);
            const double rho1 = (c2 <= dsqr) ? 1.0 : delta / std::sqrt(c2);
            const double W = rho1 * w[k];
            const double r0 = -(w[k] * e[0]) * rho1, r1 = -(w[k] * e[1]) * rho1;
            for (int r = 0; r < 6; ++r) {
                b[r] += J[r] * r0 + J[6 + r] * r1;
                for (int c = 0; c < 6; ++c) H[r * 6 + c] += (J[r] * W) * J[c] + (J[6 + r] * W) * J[6 + c];
            }
        }
    }
    // dense LL^T of H + lam I; false when not positive definite
    static bool solve(const double* H, const double* b, double lam, double* x) {
        double L[36];
        for (int r = 0; r < 6; ++r) {
            for (int c = 0; c <= r; ++c) {
                double s = H[r * 6 + c] + (r == c ? lam : 0.0);
                for (int k = 0; k < c; ++k) s -= L[r * 6 + k] * L[c * 6 + k];
                if (c == r) {
                    if (!(s > 0.0) || !std::isfinite(s)) return false;
                    L[r * 6 + r] = std::sqrt(s);
                } else {
                    L[r * 6 + c] = s / L[c * 6 + c];
                }
            }
        }
        for (int r = 0; r < 6; ++r) {
            double s = b[r];
            for (int k = 0; k < r; ++k) s -= L[r * 6 + k] * x[k];
            x[r] = s / L[r * 6 + r];
        }
        for (int r = 5; r >= 0; --r) {
            double s = x[r];
            for (int k = r + 1; k < 6; ++k) s -= L[k * 6 + r] * x[k];
            x[r] = s / L[r * 6 + r];
        }
        return true;
    }

    // SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg::solve; returns iterations done
    int optimize(int iterations, IterStats* stats, double* trace, int* status) {
        *status = 0;
        if (E == 0) { *status = 1; return 0; }
        double lambda = 0, ni = 2;
        int done = 0;
        bool ok = true;
        for (int it = 0; it < iterations && ok; ++it) {
            IterStats st{};
            double currentChi = chi2(est);
            st.chi2_before = currentChi;
            double H[36], b[6], x[6];
            build(H, b);
            if (it == 0) {
                double m = 0;
                for (int r = 0; r < 6; ++r) m = std::max(m, std::fabs(H[r * 7]));
                lambda = 1e-5 * m; ni = 2;
            }
            double rho = 0;
            int qmax = 0, failed = 0;
            do {
                const SE3 bak = est;
                const bool ok2 = solve(H, b, lambda, x);
                if (ok2) est = se3_mul(se3_exp(x), est);
                else ++failed;
                double tempChi = ok2 ? chi2(est) : std::numeric_limits<double>::max();
                rho = currentChi - tempChi;
                double scale = 0;
                if (ok2) for (int r = 0; r < 6; ++r) scale += x[r] * (lambda * x[r] + b[r]);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && std::isfinite(tempChi)) {
                    double alpha = 1. - std::pow((2 * rho - 1), 3);
                    alpha = std::min(alpha, 2. / 3.);
                    const double scaleFactor = std::max(1. / 3., alpha);
                    lambda *= scaleFactor;
                    ni = 2;
                    currentChi = tempChi;
                    st.accepted = 1;
                } else {
                    lambda *= ni;
                    ni *= 2;
                    est = bak;
                }
                qmax++;
            } while (rho < 0 && qmax < 10);
            st.chi2_after = currentChi; st.lambda = lambda; st.rho = rho; st.trials = qmax;
            st.terminate = (qmax == 10 || rho == 0) ? 1 : 0;
            ok = !st.terminate;
            if (st.terminate && failed == qmax) *status = 2;
            if (stats) stats[it] = st;
            if (trace) {
                double* p = trace + 7 * (size_t)it;
                p[0] = est.q.x; p[1] = est.q.y; p[2] = est.q.z; p[3] = est.q.w;
                p[4] = est.t[0]; p[5] = est.t[1]; p[6] = est.t[2];
            }
            ++done;
        }
        return done;
    }
};

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

}  // namespace

extern "C" {

// One problem of Localizer::DoLocalBA. Tcw [16] float row-major in/out (untouched when status is 1, "no edges"); xyz [E*3],
// uv [E*2], w [E] (information scale) float; Tbc [16] float. stats [iterations] / trace [iterations*7] / pose7 [7] may be NULL.
// Returns the number of LM iterations done; *status: 0 OK, 1 no edges, 2 the last iteration's 10 trials all failed Cholesky.
int pose_ba_oracle_run(float* Tcw, int E, const float* xyz, const float* uv, const float* w, float fx, float cx, float cy,
                       const float* Tbc, float huber_delta, float xrot, float yrot, float zinfo, int iterations, void* stats,
                       double* trace, double* pose7, int* status) {
    PoseBA p;
    p.est = se3_from_f32(Tcw);
    plane_motion_prior(p.est, Tbc, xrot, yrot, zinfo, &p.meas, p.prior_info);
    p.E = E;
    p.xyz.assign(xyz, xyz + 3 * (size_t)E);
    p.uv.assign(uv, uv + 2 * (size_t)E);
    p.w.assign(w, w + E);
    p.fx = fx; p.cx = cx; p.cy = cy; p.delta = huber_delta;
    const int done = p.optimize(iterations, (IterStats*)stats, trace, status);
    if (pose7) pose_out(p.est, pose7);
    if (*status != 1) to_f32(p.est, Tcw);
    return done;
}

// Single pieces for the self-consistency tests. Poses are 7 doubles (qx, qy, qz, qw, tx, ty, tz).
void pose_ba_oracle_from_f32(const float* T, double* pose7) { pose_out(se3_from_f32(T), pose7); }
void pose_ba_oracle_exp(const double* u6, double* pose7) { pose_out(se3_exp(u6), pose7); }
void pose_ba_oracle_log(const double* pose7, double* u6) { se3_log(pose_in(pose7), u6); }
void pose_ba_oracle_mul(const double* a7, const double* b7, double* out7) { pose_out(se3_mul(pose_in(a7), pose_in(b7)), out7); }
void pose_ba_oracle_prior(const double* pose7, const float* Tbc, float xrot, float yrot, float zinfo, double* meas7, double* info36) {
    SE3 m;
    plane_motion_prior(pose_in(pose7), Tbc, xrot, yrot, zinfo, &m, info36);
    pose_out(m, meas7);
}
// error [2] and pose Jacobian [2x6] of one projection edge at pose7
void pose_ba_oracle_edge(const double* pose7, const double* xyz, const double* uv, double fx, double cx, double cy, double* err,
                         double* J12) {
    PoseBA p;
    p.E = 1; p.xyz.assign(xyz, xyz + 3); p.uv.assign(uv, uv + 2); p.w.assign(1, 1.0);
    p.fx = fx; p.cx = cx; p.cy = cy; p.delta = 1;
    p.proj_edge(pose_in(pose7), 0, err, J12);
}

}  // extern "C"
