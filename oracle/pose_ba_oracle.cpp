// Pose-only SE(3) bundle adjustment ORACLE (Localizer::DoLocalBA) — TEST INFRASTRUCTURE ONLY.
//
// Sequential double-precision restatement of what the reference's Localizer::DoLocalBA (src/Localizer.cpp:233-302)
// hands to g2o: one VertexSE3Expmap (estimate toSE3Quat(Tcw)), one EdgeSE3ExpmapPrior built by addPlaneMotionSE3Expmap
// (src/optimizer.cpp:236-314, non-USE_EULER branch; error log(meas * est^-1), Jacobian the constant -I of :181-189),
// and one EdgeProjectXYZ2UV per observed map point (fixed VertexSBAPointXYZ, CameraParameters(fx, (cx, cy), 0),
// information w_e * I, RobustKernelHuber(delta)), then initializeOptimization(0); optimize(iterations).
//
// g2o (tag 20160424) and Eigen are not vendored; their published algorithms are restated: the SE3Quat algebra, the prior
// and EdgeProjectXYZ2UV (oracle/se3_oracle.h), BaseUnaryEdge / BaseBinaryEdge constructQuadraticForm with the Huber
// weighting rho'(e) * Omega, and OptimizationAlgorithmLevenberg::solve (oracle/g2o_lm_oracle.h).
// The pose system is 6 x 6 and is factorised with a dense LL^T (what CHOLMOD does on it).
// PARITY UNPINNED against real g2o (no g2o build exists here); pinned by self-consistency in tests/test_pose_ba_oracle.py
// (numeric Jacobians, exp/log round trips, an independent numpy restatement in oracle/pose_ba_numpy.py).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "g2o_lm_oracle.h"
#include "se3_oracle.h"

namespace {

struct PoseBA {
    SE3 est, bak;
    SE3 meas;
    double prior_info[36];
    int E = 0;
    std::vector<double> xyz, uv, w;
    double fx, cx, cy, delta;
    double H[36], b[6];
    double* trace = nullptr;

    // EdgeProjectXYZ2UV::computeError; optionally the pose block of linearizeOplus
    void proj_edge(const SE3& T, int e, double* err, double* J) const {
        double pc[3];
        proj_error(T, &xyz[3 * (size_t)e], &uv[2 * (size_t)e], fx, cx, cy, err, pc, J);
    }
    // activeRobustChi2: the prior (edge added first) then every projection edge through RobustKernelHuber
    double chi2(const SE3& T) const {
        double e6[6];
        expmap_prior_error(meas, T, e6);
        double chi = quad(prior_info, e6, 6);
        const double dsqr = delta * delta;
        for (int k = 0; k < E; ++k) {
            double e[2];
            proj_edge(T, k, e, nullptr);
            const double c2 = e[0] * (w[k] * e[0]) + e[1] * (w[k] * e[1]);
            chi += (c2 <= dsqr) ? c2 : 2 * std::sqrt(c2) * delta - dsqr;
        }
        return chi;
    }

    // the LM hooks of lm_optimize
    double start_chi2(int, double) const { return chi2(est); }  // evaluated at every iteration's start
    // buildSystem: H [36] full symmetric, b [6]
    void build() {
        double e6[6];
        expmap_prior_error(meas, est, e6);
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
    double max_diag() const {
        double m = 0;
        for (int r = 0; r < 6; ++r) m = std::max(m, std::fabs(H[r * 7]));
        return m;
    }
    bool trial(double lambda, double* tempChi, double* scale) {
        double A[36], x[6];
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) A[r * 6 + c] = H[r * 6 + c] + (r == c ? lambda : 0.0);
        bak = est;
        if (!dense_llt_solve(6, A, b, x)) return false;
        est = se3_mul(se3_exp(x), est);
        *tempChi = chi2(est);
        for (int r = 0; r < 6; ++r) *scale += x[r] * (lambda * x[r] + b[r]);
        return true;
    }
    void accept() {}
    void reject() { est = bak; }
    void record(int it) {
        if (trace) pose_out(est, trace + 7 * (size_t)it);
    }
};

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
    plane_prior_expmap(p.est, Tbc, xrot, yrot, zinfo, &p.meas, p.prior_info);
    p.E = E;
    p.xyz.assign(xyz, xyz + 3 * (size_t)E);
    p.uv.assign(uv, uv + 2 * (size_t)E);
    p.w.assign(w, w + E);
    p.fx = fx; p.cx = cx; p.cy = cy; p.delta = huber_delta;
    p.trace = trace;
    bool not_pd = false;
    const int done = E > 0 ? lm_optimize(p, iterations, (IterStats*)stats, &not_pd) : 0;
    *status = E == 0 ? 1 : not_pd ? 2 : 0;
    if (pose7) pose_out(p.est, pose7);
    if (E > 0) to_f32(p.est, Tcw);
    return done;
}

// Single pieces for the self-consistency tests. Poses are 7 doubles (qx, qy, qz, qw, tx, ty, tz).
void pose_ba_oracle_from_f32(const float* T, double* pose7) { pose_out(se3_from_f32(T), pose7); }
void pose_ba_oracle_exp(const double* u6, double* pose7) { pose_out(se3_exp(u6), pose7); }
void pose_ba_oracle_log(const double* pose7, double* u6) { se3_log(pose_in(pose7), u6); }
void pose_ba_oracle_mul(const double* a7, const double* b7, double* out7) { pose_out(se3_mul(pose_in(a7), pose_in(b7)), out7); }
void pose_ba_oracle_prior(const double* pose7, const float* Tbc, float xrot, float yrot, float zinfo, double* meas7, double* info36) {
    SE3 m;
    plane_prior_expmap(pose_in(pose7), Tbc, xrot, yrot, zinfo, &m, info36);
    pose_out(m, meas7);
}
// error [2] and pose Jacobian [2x6] of one projection edge at pose7
void pose_ba_oracle_edge(const double* pose7, const double* xyz, const double* uv, double fx, double cx, double cy, double* err,
                         double* J12) {
    double pc[3];
    proj_error(pose_in(pose7), xyz, uv, fx, cx, cy, err, pc, J12);
}

}  // extern "C"
