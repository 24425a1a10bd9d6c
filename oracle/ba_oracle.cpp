// SE(2)-XYZ local bundle adjustment ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement (double precision, sequential) of what LocalMapper::localBA does once
// Map::loadLocalGraph has filled the g2o graph (reference src/LocalMapper.cpp:232-302,
// src/Map.cpp:891-1053):  optimizer.initializeOptimization(0); optimizer.optimize(LOCAL_ITER)
// over VertexSE2 / VertexSBAPointXYZ vertices, EdgeSE2XYZ (src/EdgeSE2XYZ.cpp:61-106, Huber kernel
// set in src/optimizer.cpp:17-32) and PreEdgeSE2 (include/se2lam/EdgeSE2XYZ.h:62-102) edges with
// the solver stack of include/se2lam/optimizer.h:30-33 (BlockSolverX + Schur + Cholesky, LM).
//
// g2o (tag 20160424_git, README.MD:29) is an un-vendored dependency that is absent from
// /root/reference and from this container: its published algorithm is restated here
// (OptimizationAlgorithmLevenberg::solve in oracle/g2o_lm_oracle.h, BlockSolver::buildSystem/solve with Schur complement,
// BaseBinaryEdge::constructQuadraticForm, RobustKernelHuber, VertexSE2/VertexSBAPointXYZ oplus).
// PARITY UNPINNED against real g2o: no g2o build or golden vector exists (SURVEY.md section 8c).  The oracle
// is instead pinned by self-consistency (tests/test_ba_oracle.py): analytic vs numeric Jacobians,
// Schur == full-system solve, convergence to ground truth on noise-free data, gauge fixing, and an
// independent numpy restatement (oracle/ba_numpy.py).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "g2o_lm_oracle.h"

namespace {

inline double normalize_theta(double theta) {  // g2o/stuff/misc.h
    if (theta >= -M_PI && theta < M_PI) return theta;
    double multiplier = std::floor(theta / (2 * M_PI));
    theta = theta - multiplier * 2 * M_PI;
    if (theta >= M_PI) theta -= 2 * M_PI;
    if (theta < -M_PI) theta += 2 * M_PI;
    return theta;
}

// 3x3 inverse via partial-pivot Gaussian elimination (Eigen dynamic-size .inverse() == PartialPivLU)
bool inv3(const double* A, double* R) {
    double m[3][6];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { m[i][j] = A[i * 3 + j]; m[i][3 + j] = (i == j); }
    for (int c = 0; c < 3; ++c) {
        int p = c;
        for (int r = c + 1; r < 3; ++r) if (std::fabs(m[r][c]) > std::fabs(m[p][c])) p = r;
        if (m[p][c] == 0.0) return false;
        if (p != c) for (int j = 0; j < 6; ++j) std::swap(m[p][j], m[c][j]);
        double d = 1.0 / m[c][c];
        for (int j = 0; j < 6; ++j) m[c][j] *= d;
        for (int r = 0; r < 3; ++r) if (r != c) {
            double f = m[r][c];
            if (f != 0.0) for (int j = 0; j < 6; ++j) m[r][j] -= f * m[c][j];
        }
    }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[i * 3 + j] = m[i][3 + j];
    return true;
}

struct BA {
    int P, L, E, O;
    std::vector<double> pose, point, uv, info, odo_meas, odo_info;
    std::vector<uint8_t> fixed;
    std::vector<int> ep, el, oi, oj;
    double fx, cx, cy, Rcb[9], tcb[3], delta;
    // index mapping (SparseOptimizer::buildIndexMapping): free poses by id, then active landmarks by id
    std::vector<int> hidx;  // pose -> free index or -1
    int nf = 0;
    std::vector<uint8_t> lm_active;
    // edges grouped per landmark (CSR) for the Schur pass
    std::vector<int> lm_ptr, lm_edges;
    // linear system
    Skyline Hpp, S;
    std::vector<int> first;
    std::vector<double> bp, Hll, bl, Hpl, bs, dx_p, dx_l, HllInv;
    std::vector<double> e_xyz, e_odo;
    std::vector<double> pose_bak, point_bak;
    double* trace_poses = nullptr;
    double* trace_points = nullptr;

    void indexing() {
        hidx.assign(P, -1); nf = 0;
        for (int i = 0; i < P; ++i) if (!fixed[i]) hidx[i] = nf++;
        lm_active.assign(L, 0);
        std::vector<int> cnt(L + 1, 0);
        for (int e = 0; e < E; ++e) { lm_active[el[e]] = 1; cnt[el[e] + 1]++; }
        lm_ptr.assign(L + 1, 0);
        for (int j = 0; j < L; ++j) lm_ptr[j + 1] = lm_ptr[j] + cnt[j + 1];
        lm_edges.assign(E, 0);
        std::vector<int> cur(lm_ptr.begin(), lm_ptr.end() - 1);
        for (int e = 0; e < E; ++e) lm_edges[cur[el[e]]++] = e;
        // skyline profile of the pose block: odometry neighbours and co-observing pose pairs
        std::vector<int> bfirst(nf);
        for (int i = 0; i < nf; ++i) bfirst[i] = i;
        auto touch = [&](int a, int b) { if (a < 0 || b < 0) return; if (a < b) std::swap(a, b); bfirst[a] = std::min(bfirst[a], b); };
        for (int o = 0; o < O; ++o) touch(hidx[oi[o]], hidx[oj[o]]);
        for (int j = 0; j < L; ++j) {
            int mn = nf;
            for (int k = lm_ptr[j]; k < lm_ptr[j + 1]; ++k) { int h = hidx[ep[lm_edges[k]]]; if (h >= 0) mn = std::min(mn, h); }
            for (int k = lm_ptr[j]; k < lm_ptr[j + 1]; ++k) { int h = hidx[ep[lm_edges[k]]]; if (h >= 0) touch(h, mn); }
        }
        first.assign(3 * nf, 0);
        for (int i = 0; i < nf; ++i) for (int r = 0; r < 3; ++r) first[3 * i + r] = 3 * bfirst[i];
        Hpp.build(3 * nf, first);
        S.build(3 * nf, first);
        bp.assign(3 * nf, 0); bs.assign(3 * nf, 0); dx_p.assign(3 * nf, 0);
        Hll.assign(9 * (size_t)L, 0); HllInv.assign(9 * (size_t)L, 0); bl.assign(3 * (size_t)L, 0); dx_l.assign(3 * (size_t)L, 0);
        Hpl.assign(9 * (size_t)E, 0);
        e_xyz.assign(2 * (size_t)E, 0); e_odo.assign(3 * (size_t)O, 0);
    }

    // EdgeSE2XYZ::computeError (EdgeSE2XYZ.cpp:61-72); optionally the Jacobians of :75-106
    inline void xyz_edge(int e, double* err, double* Ji /*2x3*/, double* Jj /*2x3*/) const {
        const double* ps = &pose[3 * ep[e]];
        const double* lw = &point[3 * el[e]];
        double c = std::cos(ps[2]), s = std::sin(ps[2]);
        // Rcw = Rcb * Rz(-theta)
        double Rcw[9];
        for (int r = 0; r < 3; ++r) {
            Rcw[r * 3 + 0] = Rcb[r * 3 + 0] * c - Rcb[r * 3 + 1] * s;
            Rcw[r * 3 + 1] = Rcb[r * 3 + 0] * s + Rcb[r * 3 + 1] * c;
            Rcw[r * 3 + 2] = Rcb[r * 3 + 2];
        }
        double d[3] = {lw[0] - ps[0], lw[1] - ps[1], lw[2]};
        double lc[3];
        for (int r = 0; r < 3; ++r) lc[r] = Rcw[r * 3] * d[0] + Rcw[r * 3 + 1] * d[1] + Rcw[r * 3 + 2] * d[2] + tcb[r];
        double zi = 1.0 / lc[2];
        err[0] = lc[0] * zi * fx + cx - uv[2 * e];
        err[1] = lc[1] * zi * fx + cy - uv[2 * e + 1];
        if (!Ji) return;
        double zi2 = zi * zi;
        double Jpi[6] = {fx * zi, 0, -fx * lc[0] * zi2, 0, fx * zi, -fx * lc[1] * zi2};
        double M[6];
        for (int r = 0; r < 2; ++r)
            for (int k = 0; k < 3; ++k) M[r * 3 + k] = Jpi[r * 3] * Rcw[k] + Jpi[r * 3 + 1] * Rcw[3 + k] + Jpi[r * 3 + 2] * Rcw[6 + k];
        for (int r = 0; r < 2; ++r) {
            Ji[r * 3 + 0] = -M[r * 3 + 0];
            Ji[r * 3 + 1] = -M[r * 3 + 1];
            Ji[r * 3 + 2] = M[r * 3 + 0] * d[1] - M[r * 3 + 1] * d[0];  // (M*skew(lw-pi))[:,2]
            Jj[r * 3 + 0] = M[r * 3 + 0]; Jj[r * 3 + 1] = M[r * 3 + 1]; Jj[r * 3 + 2] = M[r * 3 + 2];
        }
    }
    // PreEdgeSE2 (EdgeSE2XYZ.h:68-99)
    inline void odo_edge(int o, double* err, double* Ji /*3x3*/, double* Jj /*3x3*/) const {
        const double* pi = &pose[3 * oi[o]];
        const double* pj = &pose[3 * oj[o]];
        double c = std::cos(pi[2]), s = std::sin(pi[2]);
        double dx = pj[0] - pi[0], dy = pj[1] - pi[1];
        err[0] = c * dx + s * dy - odo_meas[3 * o];
        err[1] = -s * dx + c * dy - odo_meas[3 * o + 1];
        err[2] = pj[2] - pi[2] - odo_meas[3 * o + 2];
        if (!Ji) return;
        // rij_x = (-dy, dx);  Ji[0:2,2] = -Ri^T rij_x
        double rx = -dy, ry = dx;
        double J1[9] = {-c, -s, -(c * rx + s * ry), s, -c, -(-s * rx + c * ry), 0, 0, -1};
        double J2[9] = {c, s, 0, -s, c, 0, 0, 0, 1};
        memcpy(Ji, J1, sizeof J1); memcpy(Jj, J2, sizeof J2);
    }

    // SparseOptimizer::computeActiveErrors + activeRobustChi2
    double chi2() {
        double chi = 0;
        for (int o = 0; o < O; ++o) {
            double* e = &e_odo[3 * o];
            odo_edge(o, e, nullptr, nullptr);
            const double* W = &odo_info[6 * o];
            double we0 = W[0] * e[0] + W[1] * e[1] + W[2] * e[2];
            double we1 = W[1] * e[0] + W[3] * e[1] + W[4] * e[2];
            double we2 = W[2] * e[0] + W[4] * e[1] + W[5] * e[2];
            chi += e[0] * we0 + e[1] * we1 + e[2] * we2;
        }
        const double dsqr = delta * delta;
        for (int k = 0; k < E; ++k) {
            double* e = &e_xyz[2 * k];
            xyz_edge(k, e, nullptr, nullptr);
            const double* W = &info[3 * k];
            double c2 = e[0] * (W[0] * e[0] + W[1] * e[1]) + e[1] * (W[1] * e[0] + W[2] * e[1]);
            chi += (c2 <= dsqr) ? c2 : 2 * std::sqrt(c2) * delta - dsqr;  // RobustKernelHuber rho[0]
        }
        return chi;
    }

    inline void addHpp(int a, int b, const double* blk /*3x3: rows a, cols b*/) {
        // symmetric accumulate into the lower skyline; (a,b) free indices
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                int R = 3 * a + r, Cc = 3 * b + c;
                if (a == b) { if (Cc <= R) Hpp.at(R, Cc) += blk[r * 3 + c]; }
                else if (a > b) Hpp.at(R, Cc) += blk[r * 3 + c];
                else Hpp.at(Cc, R) += blk[r * 3 + c];
            }
    }

    // BlockSolver::buildSystem: linearizeOplus + constructQuadraticForm over all active edges
    void build() {
        std::fill(Hpp.v.begin(), Hpp.v.end(), 0.0);
        std::fill(bp.begin(), bp.end(), 0.0);
        std::fill(Hll.begin(), Hll.end(), 0.0);
        std::fill(bl.begin(), bl.end(), 0.0);
        std::fill(Hpl.begin(), Hpl.end(), 0.0);
        for (int o = 0; o < O; ++o) {
            double e[3], A[9], B[9];
            odo_edge(o, e, A, B);
            const double* w = &odo_info[6 * o];
            double W[9] = {w[0], w[1], w[2], w[1], w[3], w[4], w[2], w[4], w[5]};
            double We[3];
            for (int r = 0; r < 3; ++r) We[r] = -(W[r * 3] * e[0] + W[r * 3 + 1] * e[1] + W[r * 3 + 2] * e[2]);
            int a = hidx[oi[o]], b = hidx[oj[o]];
            double AtW[9], BtW[9];
            for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) {
                AtW[r * 3 + c] = A[0 * 3 + r] * W[0 * 3 + c] + A[1 * 3 + r] * W[1 * 3 + c] + A[2 * 3 + r] * W[2 * 3 + c];
                BtW[r * 3 + c] = B[0 * 3 + r] * W[0 * 3 + c] + B[1 * 3 + r] * W[1 * 3 + c] + B[2 * 3 + r] * W[2 * 3 + c];
            }
            auto mul = [](const double* X, const double* Y, double* Z) {
                for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Z[r * 3 + c] = X[r * 3] * Y[c] + X[r * 3 + 1] * Y[3 + c] + X[r * 3 + 2] * Y[6 + c];
            };
            double blk[9];
            if (a >= 0) {
                for (int r = 0; r < 3; ++r) bp[3 * a + r] += A[0 * 3 + r] * We[0] + A[1 * 3 + r] * We[1] + A[2 * 3 + r] * We[2];
                mul(AtW, A, blk); addHpp(a, a, blk);
                if (b >= 0) { mul(AtW, B, blk); addHpp(a, b, blk); }
            }
            if (b >= 0) {
                for (int r = 0; r < 3; ++r) bp[3 * b + r] += B[0 * 3 + r] * We[0] + B[1 * 3 + r] * We[1] + B[2 * 3 + r] * We[2];
                mul(BtW, B, blk); addHpp(b, b, blk);
            }
        }
        const double dsqr = delta * delta;
        for (int k = 0; k < E; ++k) {
            double e[2], A[6], B[6];
            xyz_edge(k, e, A, B);
            const double* w = &info[3 * k];
            double c2 = e[0] * (w[0] * e[0] + w[1] * e[1]) + e[1] * (w[1] * e[0] + w[2] * e[1]);
            double rho1 = (c2 <= dsqr) ? 1.0 : delta / std::sqrt(c2);
            double W[4] = {rho1 * w[0], rho1 * w[1], rho1 * w[1], rho1 * w[2]};       // robustInformation
            double We[2] = {-(w[0] * e[0] + w[1] * e[1]) * rho1, -(w[1] * e[0] + w[2] * e[1]) * rho1};
            int a = hidx[ep[k]], j = el[k];
            double AtW[6], BtW[6];  // 3x2
            for (int r = 0; r < 3; ++r) for (int c = 0; c < 2; ++c) {
                AtW[r * 2 + c] = A[r] * W[c] + A[3 + r] * W[2 + c];
                BtW[r * 2 + c] = B[r] * W[c] + B[3 + r] * W[2 + c];
            }
            if (a >= 0) {
                double blk[9];
                for (int r = 0; r < 3; ++r) {
                    bp[3 * a + r] += A[r] * We[0] + A[3 + r] * We[1];
                    for (int c = 0; c < 3; ++c) {
                        blk[r * 3 + c] = AtW[r * 2] * A[c] + AtW[r * 2 + 1] * A[3 + c];
                        Hpl[9 * (size_t)k + r * 3 + c] = AtW[r * 2] * B[c] + AtW[r * 2 + 1] * B[3 + c];
                    }
                }
                addHpp(a, a, blk);
            }
            for (int r = 0; r < 3; ++r) {
                bl[3 * j + r] += B[r] * We[0] + B[3 + r] * We[1];
                for (int c = 0; c < 3; ++c) Hll[9 * (size_t)j + r * 3 + c] += BtW[r * 2] * B[c] + BtW[r * 2 + 1] * B[3 + c];
            }
        }
    }

    double max_diag() const {  // OptimizationAlgorithmLevenberg::computeLambdaInit
        double m = 0;
        for (int r = 0; r < 3 * nf; ++r) m = std::max(m, std::fabs(Hpp.get(r, r)));
        for (int j = 0; j < L; ++j) if (lm_active[j]) for (int r = 0; r < 3; ++r) m = std::max(m, std::fabs(Hll[9 * (size_t)j + 4 * r]));
        return m;
    }

    // BlockSolver::solve with Schur complement; lambda added to every diagonal first (setLambda)
    bool solve(double lam) {
        S.v = Hpp.v;
        for (int r = 0; r < 3 * nf; ++r) S.at(r, r) += lam;
        bs = bp;
        for (int j = 0; j < L; ++j) {
            if (!lm_active[j]) continue;
            double D[9];
            memcpy(D, &Hll[9 * (size_t)j], sizeof D);
            D[0] += lam; D[4] += lam; D[8] += lam;
            double* Dinv = &HllInv[9 * (size_t)j];
            if (!inv3(D, Dinv)) return false;
            double db[3];
            for (int r = 0; r < 3; ++r) db[r] = Dinv[r * 3] * bl[3 * j] + Dinv[r * 3 + 1] * bl[3 * j + 1] + Dinv[r * 3 + 2] * bl[3 * j + 2];
            for (int k1 = lm_ptr[j]; k1 < lm_ptr[j + 1]; ++k1) {
                int e1 = lm_edges[k1], a = hidx[ep[e1]];
                if (a < 0) continue;
                const double* Bi = &Hpl[9 * (size_t)e1];
                double BD[9];
                for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) BD[r * 3 + c] = Bi[r * 3] * Dinv[c] + Bi[r * 3 + 1] * Dinv[3 + c] + Bi[r * 3 + 2] * Dinv[6 + c];
                for (int r = 0; r < 3; ++r) bs[3 * a + r] -= Bi[r * 3] * db[0] + Bi[r * 3 + 1] * db[1] + Bi[r * 3 + 2] * db[2];
                for (int k2 = lm_ptr[j]; k2 < lm_ptr[j + 1]; ++k2) {
                    int e2 = lm_edges[k2], b = hidx[ep[e2]];
                    if (b < 0 || b > a) continue;  // lower triangle (incl. diagonal blocks) only
                    const double* Bj = &Hpl[9 * (size_t)e2];
                    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) {
                        if (a == b && c > r) continue;
                        double vv = BD[r * 3] * Bj[c * 3] + BD[r * 3 + 1] * Bj[c * 3 + 1] + BD[r * 3 + 2] * Bj[c * 3 + 2];
                        S.at(3 * a + r, 3 * b + c) -= vv;
                    }
                }
            }
        }
        if (!S.cholesky()) return false;
        dx_p = bs;
        S.solve(dx_p.data());
        for (int j = 0; j < L; ++j) {
            if (!lm_active[j]) { dx_l[3 * j] = dx_l[3 * j + 1] = dx_l[3 * j + 2] = 0; continue; }
            double cl[3] = {bl[3 * j], bl[3 * j + 1], bl[3 * j + 2]};
            for (int k = lm_ptr[j]; k < lm_ptr[j + 1]; ++k) {
                int e = lm_edges[k], a = hidx[ep[e]];
                if (a < 0) continue;
                const double* B = &Hpl[9 * (size_t)e];
                for (int c = 0; c < 3; ++c) cl[c] -= B[0 * 3 + c] * dx_p[3 * a] + B[1 * 3 + c] * dx_p[3 * a + 1] + B[2 * 3 + c] * dx_p[3 * a + 2];
            }
            const double* Dinv = &HllInv[9 * (size_t)j];
            for (int r = 0; r < 3; ++r) dx_l[3 * j + r] = Dinv[r * 3] * cl[0] + Dinv[r * 3 + 1] * cl[1] + Dinv[r * 3 + 2] * cl[2];
        }
        return true;
    }

    void applyUpdate() {  // SparseOptimizer::update -> VertexSE2::oplusImpl / VertexSBAPointXYZ::oplusImpl
        for (int i = 0; i < P; ++i) {
            int a = hidx[i];
            if (a < 0) continue;
            pose[3 * i] += dx_p[3 * a]; pose[3 * i + 1] += dx_p[3 * a + 1];
            pose[3 * i + 2] = normalize_theta(pose[3 * i + 2] + dx_p[3 * a + 2]);
        }
        for (int j = 0; j < L; ++j) if (lm_active[j]) for (int r = 0; r < 3; ++r) point[3 * j + r] += dx_l[3 * j + r];
    }

    double computeScale(double lam) const {  // OptimizationAlgorithmLevenberg::computeScale
        double s = 0;
        for (int r = 0; r < 3 * nf; ++r) s += dx_p[r] * (lam * dx_p[r] + bp[r]);
        for (int j = 0; j < L; ++j) if (lm_active[j]) for (int r = 0; r < 3; ++r) s += dx_l[3 * j + r] * (lam * dx_l[3 * j + r] + bl[3 * j + r]);
        return s;
    }

    // the other LM hooks of lm_optimize (build and max_diag are above); chi2 is evaluated at every iteration's start
    double start_chi2(int, double) { return chi2(); }
    bool trial(double lam, double* tempChi, double* scale) {
        pose_bak = pose; point_bak = point;  // push()
        const bool ok = solve(lam);
        if (ok) applyUpdate();
        *tempChi = chi2();
        if (ok) *scale = computeScale(lam);
        return ok;
    }
    void accept() {}
    void reject() { pose = pose_bak; point = point_bak; }  // pop()
    void record(int it) {
        if (trace_poses) memcpy(trace_poses + (size_t)it * 3 * P, pose.data(), sizeof(double) * 3 * P);
        if (trace_points) memcpy(trace_points + (size_t)it * 3 * L, point.data(), sizeof(double) * 3 * L);
    }
};

}  // namespace

extern "C" {

void* ba_oracle_create(int P, int L, int E, int O, const double* poses, const uint8_t* fixed, const double* points,
                       const int* edge_pose, const int* edge_point, const double* uv, const double* info,
                       const int* odo_i, const int* odo_j, const double* odo_meas, const double* odo_info,
                       double fx, double cx, double cy, const double* Tcb, double huber_delta) {
    BA* b = new BA;
    b->P = P; b->L = L; b->E = E; b->O = O;
    b->pose.assign(poses, poses + 3 * (size_t)P);
    b->fixed.assign(fixed, fixed + P);
    b->point.assign(points, points + 3 * (size_t)L);
    b->ep.assign(edge_pose, edge_pose + E); b->el.assign(edge_point, edge_point + E);
    b->uv.assign(uv, uv + 2 * (size_t)E); b->info.assign(info, info + 3 * (size_t)E);
    b->oi.assign(odo_i, odo_i + O); b->oj.assign(odo_j, odo_j + O);
    b->odo_meas.assign(odo_meas, odo_meas + 3 * (size_t)O); b->odo_info.assign(odo_info, odo_info + 6 * (size_t)O);
    b->fx = fx; b->cx = cx; b->cy = cy; b->delta = huber_delta;
    memcpy(b->Rcb, Tcb, sizeof(double) * 9); memcpy(b->tcb, Tcb + 9, sizeof(double) * 3);
    b->indexing();
    return b;
}
void ba_oracle_destroy(void* h) { delete (BA*)h; }
// SparseOptimizer::optimize(iters); stop (may be NULL) is polled like g2o's force-stop flag. The NOT_PD status is not reported.
int ba_oracle_optimize(void* h, int iters, void* stats, double* trace_poses, double* trace_points, const volatile uint8_t* stop) {
    BA* b = (BA*)h;
    b->trace_poses = trace_poses; b->trace_points = trace_points;
    bool not_pd = false;
    return lm_optimize(*b, iters, (IterStats*)stats, &not_pd, stop);
}
void ba_oracle_get(void* h, double* poses, double* points) {
    BA* b = (BA*)h;
    memcpy(poses, b->pose.data(), sizeof(double) * 3 * b->P);
    memcpy(points, b->point.data(), sizeof(double) * 3 * b->L);
}
void ba_oracle_set(void* h, const double* poses, const double* points) {
    BA* b = (BA*)h;
    memcpy(b->pose.data(), poses, sizeof(double) * 3 * b->P);
    memcpy(b->point.data(), points, sizeof(double) * 3 * b->L);
}
int ba_oracle_num_free(void* h) { return ((BA*)h)->nf; }
double ba_oracle_chi2(void* h) { return ((BA*)h)->chi2(); }
// introspection for kernel-level parity: errors + linear system at the current estimate.
// Hpp_dense/S_dense are [3nf x 3nf] row-major full symmetric; Hll [L*9]; Hpl [E*9] (rows: pose, cols: point).
double ba_oracle_linearize(void* h, double* Hpp_dense, double* bp, double* Hll, double* bl, double* Hpl) {
    BA* b = (BA*)h;
    double chi = b->chi2();
    b->build();
    int n = 3 * b->nf;
    if (Hpp_dense) for (int r = 0; r < n; ++r) for (int c = 0; c < n; ++c) Hpp_dense[(size_t)r * n + c] = b->Hpp.get(r, c);
    if (bp) memcpy(bp, b->bp.data(), sizeof(double) * n);
    if (Hll) memcpy(Hll, b->Hll.data(), sizeof(double) * 9 * b->L);
    if (bl) memcpy(bl, b->bl.data(), sizeof(double) * 3 * b->L);
    if (Hpl) memcpy(Hpl, b->Hpl.data(), sizeof(double) * 9 * b->E);
    return chi;
}
// after ba_oracle_linearize: Schur-reduce with damping lam and solve. S_dense (pre-factorisation) optional.
int ba_oracle_schur_solve(void* h, double lam, double* S_dense, double* bs, double* dx_p, double* dx_l) {
    BA* b = (BA*)h;
    int n = 3 * b->nf;
    if (S_dense) {
        // rebuild S without factorising: run solve() on a copy
        BA tmp = *b;
        Skyline keep;
        // compute S by replaying the Schur loop but stopping before cholesky: emulate via solve on copy and recompute S
        tmp.S.v = tmp.Hpp.v;
        for (int r = 0; r < n; ++r) tmp.S.at(r, r) += lam;
        for (int j = 0; j < tmp.L; ++j) {
            if (!tmp.lm_active[j]) continue;
            double D[9], Dinv[9];
            memcpy(D, &tmp.Hll[9 * (size_t)j], sizeof D);
            D[0] += lam; D[4] += lam; D[8] += lam;
            if (!inv3(D, Dinv)) return 0;
            for (int k1 = tmp.lm_ptr[j]; k1 < tmp.lm_ptr[j + 1]; ++k1) {
                int e1 = tmp.lm_edges[k1], a = tmp.hidx[tmp.ep[e1]];
                if (a < 0) continue;
                const double* Bi = &tmp.Hpl[9 * (size_t)e1];
                double BD[9];
                for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) BD[r * 3 + c] = Bi[r * 3] * Dinv[c] + Bi[r * 3 + 1] * Dinv[3 + c] + Bi[r * 3 + 2] * Dinv[6 + c];
                for (int k2 = tmp.lm_ptr[j]; k2 < tmp.lm_ptr[j + 1]; ++k2) {
                    int e2 = tmp.lm_edges[k2], bb = tmp.hidx[tmp.ep[e2]];
                    if (bb < 0 || bb > a) continue;
                    const double* Bj = &tmp.Hpl[9 * (size_t)e2];
                    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) {
                        if (a == bb && c > r) continue;
                        tmp.S.at(3 * a + r, 3 * bb + c) -= BD[r * 3] * Bj[c * 3] + BD[r * 3 + 1] * Bj[c * 3 + 1] + BD[r * 3 + 2] * Bj[c * 3 + 2];
                    }
                }
            }
        }
        for (int r = 0; r < n; ++r) for (int c = 0; c < n; ++c) S_dense[(size_t)r * n + c] = tmp.S.get(r, c);
    }
    bool ok = b->solve(lam);
    if (bs) memcpy(bs, b->bs.data(), sizeof(double) * n);
    if (dx_p) memcpy(dx_p, b->dx_p.data(), sizeof(double) * n);
    if (dx_l) memcpy(dx_l, b->dx_l.data(), sizeof(double) * 3 * b->L);
    return ok ? 1 : 0;
}
// Map::loadLocalGraph's per-edge information matrix (reference src/Map.cpp:1024-1049) from the reference's float data,
// written with generic small-matrix products in the order of the reference's Eigen expressions.
void ba_oracle_edge_information(int E, const float* view_mp, const int* edge_pose, const int* edge_point, const int* octave,
                                const float* kf_Rcw, const float* kf_twb_xy, const float* mp_pos, const float* level_sigma2,
                                float fx_f, float xrot_info, float z_info, double* info) {
    for (int e = 0; e < E; ++e) {
        const int p = edge_pose[e], j = edge_point[e];
        const float Sigma2 = level_sigma2[octave[e]];
        double Sigma_u[4] = {Sigma2, 0, 0, Sigma2};                                   // Matrix2d::Identity() * Sigma2
        double lc[3] = {view_mp[3 * e], view_mp[3 * e + 1], view_mp[3 * e + 2]};       // toVector3d(pKF->mViewMPs[ftrIdx])
        double zc = lc[2], zc_inv = 1. / zc, zc_inv2 = zc_inv * zc_inv;
        const float& fx = fx_f;
        double J_pi[6] = {fx * zc_inv, 0, -fx * lc[0] * zc_inv2, 0, fx * zc_inv, -fx * lc[1] * zc_inv2};
        double Rcw[9];
        for (int k = 0; k < 9; ++k) Rcw[k] = kf_Rcw[9 * (size_t)p + k];                // toMatrix3d(pKF->Tcw.rowRange(0,3).colRange(0,3))
        double pi[3] = {kf_twb_xy[2 * (size_t)p], kf_twb_xy[2 * (size_t)p + 1], 0};     // Vector3d pi(pKF->Twb.x, pKF->Twb.y, 0)
        double lw[3] = {mp_pos[3 * (size_t)j], mp_pos[3 * (size_t)j + 1], mp_pos[3 * (size_t)j + 2]};
        double J_pi_Rcw[6];
        for (int r = 0; r < 2; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += J_pi[r * 3 + k] * Rcw[k * 3 + c]; J_pi_Rcw[r * 3 + c] = s; }
        double v[3] = {lw[0] - pi[0], lw[1] - pi[1], lw[2] - pi[2]};
        double S[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};                 // g2o skew()
        double MS[6];
        for (int r = 0; r < 2; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += J_pi_Rcw[r * 3 + k] * S[k * 3 + c]; MS[r * 3 + c] = s; }
        double J_rotxy[4] = {MS[0], MS[1], MS[3], MS[4]};
        double J_z[2] = {-J_pi_Rcw[2], -J_pi_Rcw[5]};
        float Sigma_rotxy = 1. / xrot_info;
        float Sigma_z = 1. / z_info;
        double A[4], Sigma_all[4];
        for (int k = 0; k < 4; ++k) A[k] = Sigma_rotxy * J_rotxy[k];                    // (Sigma_rotxy*J_rotxy) * J_rotxy^T
        for (int r = 0; r < 2; ++r) for (int c = 0; c < 2; ++c)
            Sigma_all[r * 2 + c] = (A[r * 2] * J_rotxy[c * 2] + A[r * 2 + 1] * J_rotxy[c * 2 + 1]) + (Sigma_z * J_z[r]) * J_z[c] + Sigma_u[r * 2 + c];
        double det = Sigma_all[0] * Sigma_all[3] - Sigma_all[1] * Sigma_all[2];
        double inv[4] = {Sigma_all[3] / det, -Sigma_all[1] / det, -Sigma_all[2] / det, Sigma_all[0] / det};
        info[3 * (size_t)e] = inv[0]; info[3 * (size_t)e + 1] = 0.5 * (inv[1] + inv[2]); info[3 * (size_t)e + 2] = inv[3];
    }
}
// Map::optimizeLocalGraph's narrowing (Map.cpp:768-779): Se2(float, float, float) normalises the float angle (Config.cpp:194-195)
void ba_oracle_writeback_f32(void* h, float* poses, float* points) {
    BA* b = (BA*)h;
    for (int i = 0; i < b->P; ++i) {
        float x = (float)b->pose[3 * i], y = (float)b->pose[3 * i + 1], th = (float)b->pose[3 * i + 2];
        poses[3 * i] = x; poses[3 * i + 1] = y; poses[3 * i + 2] = (float)normalize_theta((double)th);
    }
    for (int j = 0; j < 3 * b->L; ++j) points[j] = (float)b->point[j];
}
// single-edge evaluation for the Jacobian self-check
void ba_oracle_edge_xyz(void* h, int e, double* err2, double* Ji6, double* Jj6) { ((BA*)h)->xyz_edge(e, err2, Ji6, Jj6); }
void ba_oracle_edge_odo(void* h, int o, double* err3, double* Ji9, double* Jj9) { ((BA*)h)->odo_edge(o, err3, Ji9, Jj9); }

}  // extern "C"
