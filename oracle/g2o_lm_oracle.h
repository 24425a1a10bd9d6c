// g2o's Levenberg-Marquardt control and the two Cholesky forms of the BA oracles — TEST INFRASTRUCTURE ONLY.
//
// OptimizationAlgorithmLevenberg::solve (g2o tag 20160424, not vendored; its published algorithm is restated) as every BA
// oracle runs it: lambda_0 = 1e-5 max|diag H| with nu = 2, rho = (chi2 - chi2_trial) / (scale + 1e-3), the (2 rho - 1)^3
// schedule, at most 10 trials, Terminate on 10 trials or rho == 0. Plain C++17: this restates g2o on its own and shares
// nothing with the product's solvers. Each oracle library is one translation unit, so everything here has internal
// linkage and only the oracles' extern "C" entry points are exported.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

namespace {

struct IterStats {  // must match se2gpu_ba_iter_stats (include/se2gpu.h)
    double chi2_before, chi2_after, lambda, rho;
    int trials, accepted, terminate, pad;
};
static_assert(sizeof(IterStats) == 48, "IterStats must match se2gpu_ba_iter_stats");

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg::solve per iteration; returns the iterations
// done. The problem supplies:
//   double start_chi2(int it, double carried)        chi2 at the start of iteration it. carried is the chi2 iteration it - 1
//                                                    ended with; it differs from the estimate's chi2 only after a failed
//                                                    trial passed the rho test (an infinite chi2 before it), when it is
//                                                    DBL_MAX. An oracle either carries it or evaluates the estimate.
//   void build()                                     the linear system at the current estimate
//   double max_diag()                                max |diag H| over every free vertex (computeLambdaInit)
//   bool trial(double lambda, double* chi2, double* scale)
//                                                    solve at lambda and form the trial estimate; false when the factorisation
//                                                    fails, leaving the estimate as it was, else its chi2 and computeScale's sum
//                                                    without the 1e-3
//   void accept() / void reject()                    keep the trial estimate / go back to the one before it; called only
//                                                    after a trial that was solved
//   void record(int it)                              the trace row of iteration it
// *not_pd is set when the last iteration terminated with every trial's factorisation failed. stop (may be NULL) is polled
// before each iteration and after each trial.
template <class Problem>
int lm_optimize(Problem& p, int iterations, IterStats* stats, bool* not_pd, const volatile uint8_t* stop = nullptr) {
    double lambda = 0, ni = 2, currentChi = 0;
    int done = 0;
    for (int it = 0; it < iterations && !(stop && *stop); ++it) {
        IterStats st{};
        currentChi = p.start_chi2(it, currentChi);
        st.chi2_before = currentChi;
        p.build();
        if (it == 0) { lambda = 1e-5 * p.max_diag(); ni = 2; }
        double rho = 0;
        int qmax = 0, failed = 0;
        do {
            double tempChi = std::numeric_limits<double>::max(), scale = 0;
            const bool solved = p.trial(lambda, &tempChi, &scale);
            if (!solved) {
                tempChi = std::numeric_limits<double>::max();
                scale = 0;
                ++failed;
            }
            rho = (currentChi - tempChi) / (scale + 1e-3);
            if (rho > 0 && std::isfinite(tempChi)) {  // a failed trial gets here from an infinite chi2
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha);
                ni = 2;
                currentChi = tempChi;
                if (solved) p.accept();
                st.accepted = 1;
            } else {
                lambda *= ni;
                ni *= 2;
                if (solved) p.reject();
            }
            qmax++;
        } while (rho < 0 && qmax < 10 && !(stop && *stop));
        st.chi2_after = currentChi; st.lambda = lambda; st.rho = rho; st.trials = qmax;
        st.terminate = (qmax == 10 || rho == 0) ? 1 : 0;
        if (st.terminate && failed == qmax) *not_pd = true;
        if (stats) stats[it] = st;
        p.record(it);
        ++done;
        if (st.terminate) break;
    }
    return done;
}

// Dense LL^T solve of the n x n system A x = b (A row-major, lower triangle read) with dot-product substitution: what
// CHOLMOD does on a small dense system. False when a pivot is not positive (CHOLMOD's minor != n).
bool dense_llt_solve(int n, const double* A, const double* b, double* x) {
    std::vector<double> L((size_t)n * n);
    for (int r = 0; r < n; ++r)
        for (int c = 0; c <= r; ++c) {
            double s = A[r * (size_t)n + c];
            for (int k = 0; k < c; ++k) s -= L[r * (size_t)n + k] * L[c * (size_t)n + k];
            if (c == r) {
                if (!(s > 0.0) || !std::isfinite(s)) return false;
                L[r * (size_t)n + r] = std::sqrt(s);
            } else {
                L[r * (size_t)n + c] = s / L[c * (size_t)n + c];
            }
        }
    for (int r = 0; r < n; ++r) {
        double s = b[r];
        for (int k = 0; k < r; ++k) s -= L[r * (size_t)n + k] * x[k];
        x[r] = s / L[r * (size_t)n + r];
    }
    for (int r = n - 1; r >= 0; --r) {
        double s = x[r];
        for (int k = r + 1; k < n; ++k) s -= L[k * (size_t)n + r] * x[k];
        x[r] = s / L[r * (size_t)n + r];
    }
    return true;
}

// Symmetric positive-definite matrix in lower skyline (profile) storage; the Cholesky stays in the profile and the back
// substitution runs by columns (axpy), so it sums in a different order from dense_llt_solve.
struct Skyline {
    int n = 0;
    std::vector<int> first;       // first stored column of row r
    std::vector<size_t> off;      // offset of row r's first stored entry
    std::vector<double> v;
    void build(int n_, const std::vector<int>& first_) {
        n = n_; first = first_; off.assign(n + 1, 0);
        for (int r = 0; r < n; ++r) off[r + 1] = off[r] + (size_t)(r - first[r] + 1);
        v.assign(off[n], 0.0);
    }
    inline double& at(int r, int c) { return v[off[r] + (c - first[r])]; }  // requires first[r] <= c <= r
    inline double get(int r, int c) const { if (c > r) std::swap(r, c); return c < first[r] ? 0.0 : v[off[r] + (c - first[r])]; }
    // in-place LL^T; false if not positive definite (CHOLMOD "minor != n")
    bool cholesky() {
        for (int r = 0; r < n; ++r) {
            double* Lr = &v[off[r]];
            for (int c = first[r]; c <= r; ++c) {
                const double* Lc = &v[off[c]];
                int k0 = std::max(first[r], first[c]);
                double s = Lr[c - first[r]];
                for (int k = k0; k < c; ++k) s -= Lr[k - first[r]] * Lc[k - first[c]];
                if (c == r) {
                    if (!(s > 0.0) || !std::isfinite(s)) return false;
                    Lr[c - first[r]] = std::sqrt(s);
                } else {
                    Lr[c - first[r]] = s / Lc[c - first[c]];
                }
            }
        }
        return true;
    }
    void solve(double* x) const {  // x := (L L^T)^-1 x
        for (int r = 0; r < n; ++r) {
            const double* Lr = &v[off[r]];
            double s = x[r];
            for (int k = first[r]; k < r; ++k) s -= Lr[k - first[r]] * x[k];
            x[r] = s / Lr[r - first[r]];
        }
        for (int r = n - 1; r >= 0; --r) {
            const double* Lr = &v[off[r]];
            x[r] /= Lr[r - first[r]];
            for (int k = first[r]; k < r; ++k) x[k] -= Lr[k - first[r]] * x[r];
        }
    }
};

}  // namespace
