// SE(3)-XYZ window BA ORACLE (Map::loadLocalGraph / loadLocalGraphOnlyBa + LocalMapper::removeOutlierChi2) — TEST
// INFRASTRUCTURE ONLY.
//
// Sequential double-precision restatement of the window the reference builds in Map::loadLocalGraph (src/Map.cpp:414-566)
// and Map::loadLocalGraphOnlyBa (:568-698), optimised by g2o's OptimizationAlgorithmLevenberg, and of removeOutlierChi2's
// per-edge cut (src/LocalMapper.cpp:172-230): VertexSE3Expmap keyframes with the plane-motion EdgeSE3ExpmapPrior where
// asked, EdgeSE3Expmap odometry (information permuted [trans rot] -> [rot trans], optimizer.cpp:489-494), marginalised
// VertexSBAPointXYZ points and Huber EdgeProjectXYZ2UV edges (information w * I).
//
// The SE3Quat pieces and the plane-motion prior are the pose-only BA oracle's: pose_ba_oracle.cpp is compiled into this
// translation unit, so both oracles run one definition of each.
//
// What is decided here:
//  * EdgeSE3Expmap's Jacobians are g2o's adjoints Adj(Tj^-1 Z) and -Adj(Ti^-1 Z^-1) (exact only at zero error, as in g2o).
//  * EdgeProjectXYZ2UV's point block is -1/z [[fx, 0, -x/z fx], [0, fx, -y/z fx]] R.
//  * A keyframe no edge touches, and a point without edges, are not in the optimised graph (initializeOptimization leaves
//    them out). The prior of a fixed keyframe and an odometry link between fixed keyframes count in chi2 (activeChi2).
//  * The points are eliminated by the Schur complement with (Hll + lambda I)^-1 by cofactors (Eigen's 3 x 3 inverse); the
//    reduced system is a dense LL^T in an elimination order the caller passes. A pivot <= 0 fails the trial.
//  * rev_sums = 1 takes every sum over edges in descending edge order instead of ascending, and rev_order = 1 eliminates
//    the free keyframes in reversed order: tests/test_se3_ba_cpp_oracle.py measures the oracle's own spread with them.
// PARITY UNPINNED against real g2o (no g2o build exists here); pinned by self-consistency and by the independent numpy
// restatement oracle/se3_ba_numpy.py.
#pragma GCC visibility push(hidden)
#include "pose_ba_oracle.cpp"
#pragma GCC visibility pop

namespace {

struct WParams {  // must match se2gpu_se3_ba_params (include/se2gpu.h)
    float fx, cx, cy;
    float Tbc[16];
    float huber_delta;
    float xrot, yrot, zinfo;
    int iterations;
    float chi2_cut;
};

struct Window {
    int N, O, L, E, rev_sums, rev_order;
    const WParams* p;
    std::vector<SE3> T, prior_meas, Z;
    std::vector<double> X, prior_info, Om;
    std::vector<uint8_t> has_prior;
    const int *from, *to, *ept, *ekf;
    std::vector<double> uv, w;
    std::vector<int> fpos, free_kf, order;  // fpos[k]: position of a free keyframe or -1; order: elimination order
    std::vector<std::vector<int>> pt_edges;

    int edge_at(int i) const { return rev_sums ? E - 1 - i : i; }

    // EdgeProjectXYZ2UV: error, raw chi2; optionally the pose (2 x 6) and point (2 x 3) blocks
    double proj(const SE3& Tk, const double* Xj, int e, double* err, double* Jp, double* Jl) const {
        double pc[3];
        qrot(Tk.q, Xj, pc);
        for (int i = 0; i < 3; ++i) pc[i] += Tk.t[i];
        const double fx = p->fx;
        err[0] = uv[2 * (size_t)e] - ((pc[0] / pc[2]) * fx + (double)p->cx);
        err[1] = uv[2 * (size_t)e + 1] - ((pc[1] / pc[2]) * fx + (double)p->cy);
        const double c2 = err[0] * (w[e] * err[0]) + err[1] * (w[e] * err[1]);
        if (!Jp) return c2;
        const double x = pc[0], y = pc[1], z = pc[2], z2 = z * z;
        Jp[0] = x * y / z2 * fx;        Jp[1] = -(1 + (x * x / z2)) * fx; Jp[2] = y / z * fx;
        Jp[3] = -1. / z * fx;           Jp[4] = 0;                        Jp[5] = x / z2 * fx;
        Jp[6] = (1 + y * y / z2) * fx;  Jp[7] = -x * y / z2 * fx;         Jp[8] = -x / z * fx;
        Jp[9] = 0;                      Jp[10] = -1. / z * fx;            Jp[11] = y / z2 * fx;
        double R[9];
        quat_to_R(Tk.q, R);
        const double iz = -1. / z;
        const double tmp[6] = {iz * fx, iz * 0.0, iz * (-x / z * fx), iz * 0.0, iz * fx, iz * (-y / z * fx)};
        for (int r = 0; r < 2; ++r)
            for (int c = 0; c < 3; ++c) Jl[r * 3 + c] = tmp[r * 3] * R[c] + tmp[r * 3 + 1] * R[3 + c] + tmp[r * 3 + 2] * R[6 + c];
        return c2;
    }
    double huber(double c2, double* rho1) const {
        const double d = p->huber_delta, dsqr = d * d;
        if (c2 <= dsqr) { if (rho1) *rho1 = 1.0; return c2; }
        const double sq = std::sqrt(c2);
        if (rho1) *rho1 = d / sq;
        return 2 * sq * d - dsqr;
    }
    static double quad(const double* I, const double* e) {
        double chi = 0;
        for (int r = 0; r < 6; ++r) {
            double we = 0;
            for (int c = 0; c < 6; ++c) we += I[r * 6 + c] * e[c];
            chi += e[r] * we;
        }
        return chi;
    }
    void odo(int o, const std::vector<SE3>& P, double* e, double* Ji, double* Jj) const {
        const SE3 TjZ = se3_mul(se3_inv(P[to[o]]), Z[o]);
        se3_log(se3_mul(TjZ, P[from[o]]), e);
        if (!Ji) return;
        se3_adj(TjZ, Ji);
        se3_adj(se3_mul(se3_inv(P[from[o]]), se3_inv(Z[o])), Jj);
        for (int k = 0; k < 36; ++k) Jj[k] = -Jj[k];
    }
    double chi2(const std::vector<SE3>& P, const std::vector<double>& Xs) const {
        double s = 0, err[2], e[6];
        for (int i = 0; i < E; ++i) {
            const int k = edge_at(i);
            s += huber(proj(P[ekf[k]], &Xs[3 * (size_t)ept[k]], k, err, nullptr, nullptr), nullptr);
        }
        for (int v = 0; v < N; ++v)
            if (has_prior[v]) { se3_log(se3_mul(prior_meas[v], se3_inv(P[v])), e); s += quad(&prior_info[36 * (size_t)v], e); }
        for (int o = 0; o < O; ++o) { odo(o, P, e, nullptr, nullptr); s += quad(&Om[36 * (size_t)o], e); }
        return s;
    }

    int optimize(IterStats* stats, double* trace, int* status) {
        const int nf = (int)free_kf.size(), n = 6 * nf;
        *status = 0;
        int iterations = (nf > 0 || E > 0) ? p->iterations : 0;
        double cur = chi2(T, X), lambda = 0, ni = 2;
        std::vector<double> Hpp(n * (size_t)n), bp(n), Hll(9 * (size_t)L), bl(3 * (size_t)L), Hpl(18 * (size_t)E), D(9 * (size_t)L);
        std::vector<double> S(n * (size_t)n), rs(n), dp(n), dl(3 * (size_t)L);
        int done = 0;
        for (int it = 0; it < iterations; ++it) {
            std::fill(Hpp.begin(), Hpp.end(), 0.0); std::fill(bp.begin(), bp.end(), 0.0);
            std::fill(Hll.begin(), Hll.end(), 0.0); std::fill(bl.begin(), bl.end(), 0.0);
            for (int i = 0; i < E; ++i) {  // the projection edges
                const int e = edge_at(i), k = ekf[e], j = ept[e];
                double err[2], Jp[12], Jl[6], rho1;
                const double c2 = proj(T[k], &X[3 * (size_t)j], e, err, Jp, Jl);
                huber(c2, &rho1);
                const double W = rho1 * w[e], r0 = -(w[e] * err[0]) * rho1, r1 = -(w[e] * err[1]) * rho1;
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c) Hll[9 * (size_t)j + r * 3 + c] += (Jl[r] * W) * Jl[c] + (Jl[3 + r] * W) * Jl[3 + c];
                    bl[3 * (size_t)j + r] += Jl[r] * r0 + Jl[3 + r] * r1;
                }
                const int f = fpos[k];
                if (f < 0) continue;
                for (int r = 0; r < 6; ++r) {
                    for (int c = 0; c < 6; ++c) Hpp[(6 * f + r) * (size_t)n + 6 * f + c] += (Jp[r] * W) * Jp[c] + (Jp[6 + r] * W) * Jp[6 + c];
                    bp[6 * f + r] += Jp[r] * r0 + Jp[6 + r] * r1;
                    for (int c = 0; c < 3; ++c) Hpl[18 * (size_t)e + r * 3 + c] = (Jp[r] * W) * Jl[c] + (Jp[6 + r] * W) * Jl[3 + c];
                }
            }
            for (int v = 0; v < N; ++v) {  // the priors: J = -I
                const int f = fpos[v];
                if (f < 0 || !has_prior[v]) continue;
                double e[6];
                se3_log(se3_mul(prior_meas[v], se3_inv(T[v])), e);
                const double* I = &prior_info[36 * (size_t)v];
                for (int r = 0; r < 6; ++r) {
                    double we = 0;
                    for (int c = 0; c < 6; ++c) { Hpp[(6 * f + r) * (size_t)n + 6 * f + c] += I[r * 6 + c]; we += I[r * 6 + c] * e[c]; }
                    bp[6 * f + r] += we;
                }
            }
            for (int o = 0; o < O; ++o) {  // the odometry
                double e[6], J[2][36];
                odo(o, T, e, J[0], J[1]);
                const double* Om_ = &Om[36 * (size_t)o];
                const int fs[2] = {fpos[from[o]], fpos[to[o]]};
                for (int a = 0; a < 2; ++a) {
                    if (fs[a] < 0) continue;
                    for (int r = 0; r < 6; ++r) {
                        double acc = 0;
                        for (int m = 0; m < 6; ++m) {
                            double oe = 0;
                            for (int c = 0; c < 6; ++c) oe += Om_[m * 6 + c] * e[c];
                            acc += J[a][m * 6 + r] * oe;
                        }
                        bp[6 * fs[a] + r] -= acc;
                    }
                    for (int b = 0; b < 2; ++b) {
                        if (fs[b] < 0) continue;
                        for (int r = 0; r < 6; ++r)
                            for (int c = 0; c < 6; ++c) {
                                double acc = 0;
                                for (int m = 0; m < 6; ++m) {
                                    double oj = 0;
                                    for (int q = 0; q < 6; ++q) oj += Om_[m * 6 + q] * J[b][q * 6 + c];
                                    acc += J[a][m * 6 + r] * oj;
                                }
                                Hpp[(6 * fs[a] + r) * (size_t)n + 6 * fs[b] + c] += acc;
                            }
                    }
                }
            }
            if (it == 0) {  // computeLambdaInit over every free vertex, points included
                double m = 0;
                for (int i = 0; i < n; ++i) m = std::max(m, std::fabs(Hpp[i * (size_t)n + i]));
                for (int j = 0; j < L; ++j)
                    if (!pt_edges[j].empty())
                        for (int r = 0; r < 3; ++r) m = std::max(m, std::fabs(Hll[9 * (size_t)j + 4 * r]));
                lambda = 1e-5 * m; ni = 2;
            }
            const double before = cur;
            int qmax = 0, failed = 0, accepted = 0;
            double rho = 0;
            for (;;) {
                // (Hll + lambda I)^-1 by cofactors, the Schur complement and the reduced right-hand side
                for (int j = 0; j < L; ++j) {
                    const double* h = &Hll[9 * (size_t)j];
                    const double a = h[0] + lambda, b = h[1], c = h[2], e_ = h[4] + lambda, f = h[5], i2 = h[8] + lambda;
                    const double c00 = e_ * i2 - f * f, c01 = c * f - b * i2, c02 = b * f - c * e_;
                    const double id = 1.0 / (a * c00 + b * c01 + c * c02);
                    double* d = &D[9 * (size_t)j];
                    d[0] = c00 * id; d[1] = c01 * id; d[2] = c02 * id; d[4] = (a * i2 - c * c) * id; d[5] = (b * c - a * f) * id;
                    d[8] = (a * e_ - b * b) * id; d[3] = d[1]; d[6] = d[2]; d[7] = d[5];
                }
                S = Hpp;
                for (int i = 0; i < n; ++i) S[i * (size_t)n + i] += lambda;
                rs = bp;
                for (int jj = 0; jj < L; ++jj) {
                    const int j = rev_sums ? L - 1 - jj : jj;
                    const double* d = &D[9 * (size_t)j];
                    for (int ea : pt_edges[j]) {
                        const int fa = fpos[ekf[ea]];
                        if (fa < 0) continue;
                        double Y[18];
                        for (int r = 0; r < 6; ++r)
                            for (int c = 0; c < 3; ++c) {
                                const double* W = &Hpl[18 * (size_t)ea + r * 3];
                                Y[r * 3 + c] = W[0] * d[c] + W[1] * d[3 + c] + W[2] * d[6 + c];
                            }
                        for (int r = 0; r < 6; ++r) rs[6 * fa + r] -= Y[r * 3] * bl[3 * (size_t)j] + Y[r * 3 + 1] * bl[3 * (size_t)j + 1] + Y[r * 3 + 2] * bl[3 * (size_t)j + 2];
                        for (int eb : pt_edges[j]) {
                            const int fb = fpos[ekf[eb]];
                            if (fb < 0) continue;
                            for (int r = 0; r < 6; ++r)
                                for (int c = 0; c < 6; ++c) {
                                    const double* W = &Hpl[18 * (size_t)eb + c * 3];
                                    S[(6 * fa + r) * (size_t)n + 6 * fb + c] -= Y[r * 3] * W[0] + Y[r * 3 + 1] * W[1] + Y[r * 3 + 2] * W[2];
                                }
                        }
                    }
                }
                // dense LL^T in the elimination order
                std::vector<double> A(n * (size_t)n);
                std::vector<int> perm(n);
                for (int q = 0; q < nf; ++q)
                    for (int r = 0; r < 6; ++r) perm[6 * q + r] = 6 * order[q] + r;
                for (int r = 0; r < n; ++r)
                    for (int c = 0; c < n; ++c) A[r * (size_t)n + c] = S[perm[r] * (size_t)n + perm[c]];
                bool ok = true;
                for (int r = 0; r < n && ok; ++r)
                    for (int c = 0; c <= r; ++c) {
                        double s = A[r * (size_t)n + c];
                        for (int k = 0; k < c; ++k) s -= A[r * (size_t)n + k] * A[c * (size_t)n + k];
                        if (c == r) {
                            if (!(s > 0.0) || !std::isfinite(s)) { ok = false; break; }
                            A[r * (size_t)n + r] = std::sqrt(s);
                        } else {
                            A[r * (size_t)n + c] = s / A[c * (size_t)n + c];
                        }
                    }
                double temp = std::numeric_limits<double>::max(), scale = 0;
                std::vector<SE3> Tt = T;
                std::vector<double> Xt = X;
                if (ok) {
                    std::vector<double> y(n);
                    for (int r = 0; r < n; ++r) {
                        double s = rs[perm[r]];
                        for (int k = 0; k < r; ++k) s -= A[r * (size_t)n + k] * y[k];
                        y[r] = s / A[r * (size_t)n + r];
                    }
                    for (int r = n - 1; r >= 0; --r) {
                        double s = y[r];
                        for (int k = r + 1; k < n; ++k) s -= A[k * (size_t)n + r] * y[k];
                        y[r] = s / A[r * (size_t)n + r];
                    }
                    for (int r = 0; r < n; ++r) dp[perm[r]] = y[r];
                    for (int q = 0; q < nf; ++q) {
                        const int v = free_kf[q];
                        Tt[v] = se3_mul(se3_exp(&dp[6 * q]), T[v]);
                        for (int r = 0; r < 6; ++r) scale += dp[6 * q + r] * (lambda * dp[6 * q + r] + bp[6 * q + r]);
                    }
                    for (int j = 0; j < L; ++j) {
                        if (pt_edges[j].empty()) continue;
                        double rr[3] = {bl[3 * (size_t)j], bl[3 * (size_t)j + 1], bl[3 * (size_t)j + 2]};
                        for (int e : pt_edges[j]) {
                            const int f = fpos[ekf[e]];
                            if (f < 0) continue;
                            for (int c = 0; c < 3; ++c) {
                                double t = 0;
                                for (int r = 0; r < 6; ++r) t += Hpl[18 * (size_t)e + r * 3 + c] * dp[6 * f + r];
                                rr[c] -= t;
                            }
                        }
                        const double* d = &D[9 * (size_t)j];
                        for (int c = 0; c < 3; ++c) {
                            const double v = d[c * 3] * rr[0] + d[c * 3 + 1] * rr[1] + d[c * 3 + 2] * rr[2];
                            Xt[3 * (size_t)j + c] = X[3 * (size_t)j + c] + v;
                            scale += v * (lambda * v + bl[3 * (size_t)j + c]);
                        }
                    }
                    temp = chi2(Tt, Xt);
                } else {
                    ++failed;
                    scale = 0;
                }
                scale += 1e-3;
                rho = (cur - temp) / scale;
                if (rho > 0 && std::isfinite(temp)) {
                    double alpha = 1. - std::pow((2 * rho - 1), 3);
                    alpha = std::min(alpha, 2. / 3.);
                    lambda *= std::max(1. / 3., alpha); ni = 2; cur = temp;
                    T.swap(Tt); X.swap(Xt); accepted = 1;
                } else {
                    lambda *= ni; ni *= 2;
                }
                ++qmax;
                if (!(rho < 0 && qmax < 10)) break;
            }
            IterStats st{};
            st.chi2_before = before; st.chi2_after = cur; st.lambda = lambda; st.rho = rho; st.trials = qmax; st.accepted = accepted;
            st.terminate = (qmax == 10 || rho == 0) ? 1 : 0;
            if (st.terminate && failed == qmax) *status = 2;
            if (stats) stats[it] = st;
            if (trace) {
                double* tr = trace + (size_t)it * (7 * (size_t)N + 3 * (size_t)L);
                for (int v = 0; v < N; ++v) pose_out(T[v], tr + 7 * (size_t)v);
                for (size_t k = 0; k < 3 * (size_t)L; ++k) tr[7 * (size_t)N + k] = X[k];
            }
            ++done;
            if (st.terminate) break;
        }
        return done;
    }
};

}  // namespace

extern "C" {

// One window. Arrays as se2gpu_se3_ba takes them; poses [N*7], points [L*3], chi2 [E], outlier [E] out; stats
// [iterations], trace [iterations*(7N+3L)] may be NULL. Returns the number of LM iterations; *status 0 OK, 2 NOT_PD.
int se3_ba_oracle_run(int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O, const int* from, const int* to,
                      const float* measure, const float* info, int L, const float* xyz, int E, const int* ept, const int* ekf,
                      const float* uv, const float* w, const void* params, int rev_sums, int rev_order, void* stats,
                      double* poses, double* points, double* chi2, uint8_t* outlier, int* status, double* trace) {
    Window W;
    W.N = N; W.O = O; W.L = L; W.E = E; W.rev_sums = rev_sums; W.rev_order = rev_order;
    W.p = (const WParams*)params;
    W.from = from; W.to = to; W.ept = ept; W.ekf = ekf;
    W.T.resize(N); W.prior_meas.resize(N); W.prior_info.assign(36 * (size_t)N, 0.0); W.has_prior.assign(prior, prior + N);
    for (int v = 0; v < N; ++v) {
        W.T[v] = se3_from_f32(Tcw + 16 * (size_t)v);
        if (prior[v]) plane_motion_prior(W.T[v], W.p->Tbc, W.p->xrot, W.p->yrot, W.p->zinfo, &W.prior_meas[v], &W.prior_info[36 * (size_t)v]);
    }
    W.Z.resize(O); W.Om.resize(36 * (size_t)O);
    for (int o = 0; o < O; ++o) {
        W.Z[o] = se3_from_f32(measure + 16 * (size_t)o);
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {  // addEdgeSE3Expmap: [trans rot] -> [rot trans]
                const int sr = r < 3 ? r + 3 : r - 3, sc = c < 3 ? c + 3 : c - 3;
                W.Om[36 * (size_t)o + r * 6 + c] = (double)info[36 * (size_t)o + sr * 6 + sc];
            }
    }
    W.X.assign(xyz, xyz + 3 * (size_t)L);
    W.uv.assign(uv, uv + 2 * (size_t)E);
    W.w.assign(w, w + E);
    std::vector<uint8_t> active(prior, prior + N);
    for (int o = 0; o < O; ++o) active[from[o]] = active[to[o]] = 1;
    for (int e = 0; e < E; ++e) active[ekf[e]] = 1;
    W.fpos.assign(N, -1);
    for (int v = 0; v < N; ++v)
        if (active[v] && !fixed[v]) { W.fpos[v] = (int)W.free_kf.size(); W.free_kf.push_back(v); }
    const int nf = (int)W.free_kf.size();
    W.order.resize(nf);
    for (int q = 0; q < nf; ++q) W.order[q] = rev_order ? nf - 1 - q : q;
    W.pt_edges.assign(L, {});
    for (int e = 0; e < E; ++e) W.pt_edges[ept[e]].push_back(e);
    if (rev_sums)
        for (auto& v : W.pt_edges) std::reverse(v.begin(), v.end());
    const int done = W.optimize((IterStats*)stats, trace, status);
    for (int v = 0; v < N; ++v) pose_out(W.T[v], poses + 7 * (size_t)v);
    for (size_t k = 0; k < 3 * (size_t)L; ++k) points[k] = W.X[k];
    for (int e = 0; e < E; ++e) {
        double err[2];
        chi2[e] = W.proj(W.T[ekf[e]], &W.X[3 * (size_t)ept[e]], e, err, nullptr, nullptr);
        outlier[e] = chi2[e] > (double)W.p->chi2_cut ? 1 : 0;
    }
    return done;
}

}  // extern "C"
