// Global pose graph ORACLE (GlobalMapper::GlobalBA) — TEST INFRASTRUCTURE ONLY.
//
// Sequential double-precision restatement of GlobalMapper::GlobalBA (src/GlobalMapper.cpp:328-535) without the
// PRE_REJECT_FTR_OUTLIER and REJECT_IF_LARGE_LAMBDA blocks, which the reference does not define: one g2o VertexSE3 per
// keyframe with addVertexSE3PlaneMotion's EdgeSE3Prior, addEdgeSE3 for every odometry and feature constraint, and
// optimize(GLOBAL_ITER) under OptimizationAlgorithmLevenberg with BlockSolverX and a sparse Cholesky.
//
// The SE(3) pieces — Isometry3d products and inverse, VertexSE3 oplus, toSE3Quat, the plane-motion prior with its analytic
// Jacobian — are oracle/se3_oracle.h's, the Levenberg-Marquardt loop and the skyline Cholesky oracle/g2o_lm_oracle.h's: the
// feature-graph oracle runs the same definitions.
//
// What is decided here and not copied from anywhere:
//  * EdgeSE3's Jacobians are the analytic first derivatives of e = toVectorMQT(Z^-1 Xi^-1 Xj) through the MQT oplus of both
//    vertices: with A = Z^-1, B = Xi^-1 Xj, E = A B and (v, w) the quaternion of E with w >= 0,
//      Ji = [[-R_A, 2 R_A skew(t_B)], [0, -(w I - skew(v)) R_A]],  Jj = [[R_E, 0], [0, w I + skew(v)]].
//    tests/test_global_ba_oracle.py holds them to central differences through the real oplus.
//  * Every vertex has its prior, the fixed one included; the fixed vertex's prior is constant and counts in chi2, as in
//    g2o's activeChi2. With no free vertex g2o's optimize() returns before any iteration; so does this.
//  * cvu::inv is the float rigid inverse: R^T, and -R^T t accumulated in double (OpenCV's float gemm) and rounded once.
//    KeyFrame::getPose().inv() of the map-point write-back is a float LU inverse in the reference; it is restated as the
//    same rigid inverse. toIsometry3D(cv::Mat) takes the rotation through an un-normalised Quaterniond.
//  * The map-point position Rwc * v + twc is one double accumulation rounded to float once (OpenCV folds the sum into gemm).
//  * g2o re-orthogonalises a VertexSE3 only after 1000 oplus calls; GLOBAL_ITER = 15 iterations of at most 10 trials never
//    get there, so it is not restated.
//  * The linear solve is a scalar envelope (skyline) Cholesky in an elimination order the caller passes (oracle/pyglobal.py
//    takes scipy's reverse Cuthill-McKee; the product computes its own order, so the two factorise in different orders).
//    The order changes only the rounding; the natural order of a graph with loop closures has an envelope too wide for the
//    larger test scenes. A pivot <= 0 fails the trial, as CHOLMOD's minor != n does.
// PARITY UNPINNED against real g2o (no g2o build exists here); pinned by self-consistency in tests/test_global_ba_oracle.py.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "g2o_lm_oracle.h"
#include "se3_oracle.h"

namespace {

struct GParams {  // must match se2gpu_global_ba_params (include/se2gpu.h)
    float Tbc[16];
    float xrot, yrot, zinfo;
    int iterations;
};

void rigid_inv_f32(const float* T, float* out) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) out[i * 4 + j] = T[j * 4 + i];
        const double s = ((double)T[i] * T[3] + (double)T[4 + i] * T[7]) + (double)T[8 + i] * T[11];
        out[i * 4 + 3] = (float)(-s);
    }
    out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = 1.f;
}

// converter.cpp toIsometry3D(cv::Mat)
Iso iso_from_f32(const float* T) {
    Iso X;
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    quat_to_R(quat_from_R(R), X.R);
    X.t[0] = T[3]; X.t[1] = T[7]; X.t[2] = T[11];
    return X;
}

// EdgeSE3: error e [6], returns e^T Om e; Ji / Jj [36] (may be NULL)
double edge_se3(const Iso& Zinv, const double* Om, const Iso& Xi, const Iso& Xj, double* e, double* Ji, double* Jj) {
    const Iso B = iso_mul(iso_inv(Xi), Xj);
    const Iso E = iso_mul(Zinv, B);
    Quat q = quat_from_R(E.R);
    normalize_rotation(q);
    e[0] = E.t[0]; e[1] = E.t[1]; e[2] = E.t[2]; e[3] = q.x; e[4] = q.y; e[5] = q.z;
    const double chi = quad(Om, e, 6);
    if (!Ji) return chi;
    for (int k = 0; k < 36; ++k) { Ji[k] = 0; Jj[k] = 0; }
    const double* RA = Zinv.R;
    const double S[9] = {0, -B.t[2], B.t[1], B.t[2], 0, -B.t[0], -B.t[1], B.t[0], 0};
    const double W[9] = {q.w, q.z, -q.y, -q.z, q.w, q.x, q.y, -q.x, q.w};  // w I - skew(v)
    double RS[9], WR[9];
    mul3(RA, S, RS);
    mul3(W, RA, WR);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            Ji[r * 6 + c] = -RA[r * 3 + c];
            Ji[r * 6 + 3 + c] = 2 * RS[r * 3 + c];
            Ji[(r + 3) * 6 + 3 + c] = -WR[r * 3 + c];
            Jj[r * 6 + c] = E.R[r * 3 + c];
        }
    Jj[21] = q.w;  Jj[22] = -q.z; Jj[23] = q.y;
    Jj[27] = q.z;  Jj[28] = q.w;  Jj[29] = -q.x;
    Jj[33] = -q.y; Jj[34] = q.x;  Jj[35] = q.w;
    return chi;
}

// A^T M B for 6 x 6 matrices
void atmb(const double* A, const double* M, const double* B, double* out) {
    double MB[36];
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int m = 0; m < 6; ++m) acc += M[r * 6 + m] * B[m * 6 + c];
            MB[r * 6 + c] = acc;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int m = 0; m < 6; ++m) acc += A[m * 6 + r] * MB[m * 6 + c];
            out[r * 6 + c] = acc;
        }
}

// -A^T M e
void atme(const double* A, const double* M, const double* e, double* out) {
    double Me[6];
    for (int r = 0; r < 6; ++r) {
        Me[r] = 0;
        for (int c = 0; c < 6; ++c) Me[r] += M[r * 6 + c] * e[c];
    }
    for (int r = 0; r < 6; ++r) {
        double acc = 0;
        for (int m = 0; m < 6; ++m) acc += A[m * 6 + r] * Me[m];
        out[r] = -acc;
    }
}

struct Graph {
    int N = 0, E = 0, n = 0;  // n = 6 * free vertices
    bool reverse = false;
    std::vector<Iso> X, Xt, Zinv;
    std::vector<Prior> prior;
    std::vector<double> Om;
    std::vector<int> from, to;
    std::vector<int> pos, vert;     // vertex -> elimination position (-1 fixed), position -> vertex
    Skyline H, L;                   // one profile: a scalar row's first column is its block row's first block column
    std::vector<double> b, x;

    int edge(int k) const { return reverse ? E - 1 - k : k; }

    double chi2(const std::vector<Iso>& Xs) const {
        double chi = 0;
        for (int v = 0; v < N; ++v) {
            double e[6];
            se3_prior_error(prior[v], Xs[v], e, nullptr);
            chi += quad(prior[v].info, e, 6);
        }
        for (int k = 0; k < E; ++k) {
            const int e = edge(k);
            double err[6];
            chi += edge_se3(Zinv[e], &Om[36 * (size_t)e], Xs[from[e]], Xs[to[e]], err, nullptr, nullptr);
        }
        return chi;
    }
    void add_block(int p, int q, const double* M, bool transpose) {  // lower triangle only
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
                const int i = 6 * p + r, j = 6 * q + c;
                if (j > i) continue;
                H.at(i, j) += transpose ? M[c * 6 + r] : M[r * 6 + c];
            }
    }

    // the LM hooks of lm_optimize
    double start_chi2(int it, double carried) const { return it == 0 ? chi2(X) : carried; }  // carried after the first
    void build() {  // BlockSolver::buildSystem: priors first, then the edges in order
        std::fill(H.v.begin(), H.v.end(), 0.0);
        std::fill(b.begin(), b.end(), 0.0);
        for (int v = 0; v < N; ++v) {
            const int p = pos[v];
            if (p < 0) continue;
            double e[6], J[36], Hb[36], bb[6];
            se3_prior_error(prior[v], X[v], e, J);
            atmb(J, prior[v].info, J, Hb);
            atme(J, prior[v].info, e, bb);
            add_block(p, p, Hb, false);
            for (int r = 0; r < 6; ++r) b[6 * p + r] += bb[r];
        }
        for (int k = 0; k < E; ++k) {
            const int e = edge(k), pi = pos[from[e]], pj = pos[to[e]];
            const double* O = &Om[36 * (size_t)e];
            double err[6], Ji[36], Jj[36], Hb[36], bb[6];
            edge_se3(Zinv[e], O, X[from[e]], X[to[e]], err, Ji, Jj);
            if (pi >= 0) {
                atmb(Ji, O, Ji, Hb); add_block(pi, pi, Hb, false);
                atme(Ji, O, err, bb);
                for (int r = 0; r < 6; ++r) b[6 * pi + r] += bb[r];
            }
            if (pj >= 0) {
                atmb(Jj, O, Jj, Hb); add_block(pj, pj, Hb, false);
                atme(Jj, O, err, bb);
                for (int r = 0; r < 6; ++r) b[6 * pj + r] += bb[r];
            }
            if (pi >= 0 && pj >= 0) {
                atmb(Ji, O, Jj, Hb);  // H_ij
                if (pi > pj) add_block(pi, pj, Hb, false);
                else add_block(pj, pi, Hb, true);
            }
        }
    }
    double max_diag() {
        double m = 0;
        for (int i = 0; i < n; ++i) m = std::max(m, std::fabs(H.at(i, i)));
        return m;
    }
    // (H + lambda I) x = b by skyline Cholesky; false when a pivot is not positive
    bool trial(double lambda, double* tempChi, double* scale) {
        L.v = H.v;
        for (int i = 0; i < n; ++i) L.at(i, i) += lambda;
        if (!L.cholesky()) return false;
        x = b;
        L.solve(x.data());
        Xt = X;
        for (int p = 0; p < (int)vert.size(); ++p) Xt[vert[p]] = oplus(X[vert[p]], &x[6 * (size_t)p]);
        for (int i = 0; i < n; ++i) *scale += x[i] * (lambda * x[i] + b[i]);
        *tempChi = chi2(Xt);
        return true;
    }
    void accept() { X = Xt; }
    void reject() {}
    void record(int) {}
};

}  // namespace

extern "C" {

// One GlobalBA. N keyframes: Tcw [N*16] float, fixed [N]; E edges: from / to [E], measure [E*16] float, info [E*36] float;
// params: se2gpu_global_ba_params. Outputs: Tcw_out [N*16] float, poses [N*7] (qx, qy, qz, qw, tx, ty, tz, may be NULL),
// stats [iterations] (may be NULL). order [free vertices]: the elimination order, position -> vertex, each free vertex once.
// reverse = 1 sums the edges in descending order (the summation-order spread).
// Returns the LM iterations done; *status 0 OK, 2 the last iteration failed every factorisation.
int global_ba_oracle_run(int N, const float* Tcw, const uint8_t* fixed, int E, const int* from, const int* to, const float* measure,
                         const float* info, const void* params, const int* order, float* Tcw_out, double* poses, void* stats, int reverse,
                         int* status) {
    GParams gp;
    std::memcpy(&gp, params, sizeof gp);
    Graph g;
    g.N = N; g.E = E; g.reverse = reverse != 0;
    g.from.assign(from, from + E); g.to.assign(to, to + E);
    g.X.resize(N); g.prior.resize(N);
    for (int v = 0; v < N; ++v) {
        float Twc[16];
        rigid_inv_f32(Tcw + 16 * (size_t)v, Twc);
        g.X[v] = iso_from_f32(Twc);
        g.prior[v] = plane_prior_se3(g.X[v], gp.Tbc, gp.xrot, gp.yrot, gp.zinfo);
    }
    g.Zinv.resize(E); g.Om.resize(36 * (size_t)E);
    for (int e = 0; e < E; ++e) {
        g.Zinv[e] = iso_inv(iso_from_f32(measure + 16 * (size_t)e));
        for (int k = 0; k < 36; ++k) g.Om[36 * (size_t)e + k] = info[36 * (size_t)e + k];
    }
    int nf = 0;
    for (int v = 0; v < N; ++v) nf += !fixed[v];
    g.vert.assign(order, order + nf);
    g.pos.assign(N, -1);
    for (int p = 0; p < nf; ++p) g.pos[g.vert[p]] = p;
    std::vector<int> first(nf);
    for (int p = 0; p < nf; ++p) first[p] = p;
    for (int e = 0; e < E; ++e) {
        const int a = g.pos[from[e]], b = g.pos[to[e]];
        if (a >= 0 && b >= 0) first[std::max(a, b)] = std::min(first[std::max(a, b)], std::min(a, b));
    }
    g.n = 6 * nf;
    std::vector<int> fcol(g.n);
    for (int i = 0; i < g.n; ++i) fcol[i] = 6 * first[i / 6];
    g.H.build(g.n, fcol); g.L.build(g.n, fcol);
    g.b.assign(g.n, 0.0);
    bool not_pd = false;
    // with no free vertex g2o's optimize() returns before any iteration
    const int done = g.n > 0 ? lm_optimize(g, gp.iterations, (IterStats*)stats, &not_pd) : 0;
    *status = not_pd ? 2 : 0;
    for (int v = 0; v < N; ++v) {
        const SE3 T = se3_from_iso(g.X[v]);
        float Twc[16];
        to_f32(T, Twc);
        rigid_inv_f32(Twc, Tcw_out + 16 * (size_t)v);
        if (poses) pose_out(T, poses + 7 * (size_t)v);
    }
    return done;
}

// EdgeSE3 at (Xi, Xj) (12 doubles each: R row-major, t) with measurement [16] float and information [36] double
double global_ba_oracle_edge(const double* Xi12, const double* Xj12, const float* measure, const double* info, double* e, double* Ji,
                             double* Jj) {
    Iso Xi, Xj;
    iso_in(Xi12, &Xi); iso_in(Xj12, &Xj);
    return edge_se3(iso_inv(iso_from_f32(measure)), info, Xi, Xj, e, Ji, Jj);
}

// toIsometry3D(cvu::inv(Tcw))
void global_ba_oracle_from_Tcw(const float* Tcw, double* X12) {
    float Twc[16];
    rigid_inv_f32(Tcw, Twc);
    iso_out(iso_from_f32(Twc), X12);
}

// the map-point write-back: pos [M*3] from kf [M], view [M*3] and Tcw [*16]
void global_ba_oracle_update_points(int M, const int* kf, const float* view, const float* Tcw, float* pos) {
    for (int m = 0; m < M; ++m) {
        float Twc[16];
        rigid_inv_f32(Tcw + 16 * (size_t)kf[m], Twc);
        const float* v = view + 3 * (size_t)m;
        for (int r = 0; r < 3; ++r) {
            const double s = ((double)Twc[r * 4] * v[0] + (double)Twc[r * 4 + 1] * v[1]) + (double)Twc[r * 4 + 2] * v[2];
            pos[3 * (size_t)m + r] = (float)(s + (double)Twc[r * 4 + 3]);
        }
    }
}

}  // extern "C"
