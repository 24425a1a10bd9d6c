// g2o's OptimizationAlgorithmLevenberg control, stated once for every LM solver of the library: the windowed BA (ba.cu, both
// execution modes), the pose-only BA (pose_ba.cu), the feature-graph constraint (feat_edge.cu) and the global pose graph
// (global_ba.cu). The rules compile for host and device; tests/native/lm_host.cpp pins them on the host.
//
// Under nvcc the header also holds the numerics the three one-CTA solvers share (pose_ba.cu, feat_edge.cu, global_ba.cu): the
// fixed-order CTA sum and max, and the dense LL^T of a small SPD matrix with its triangular solve.
#pragma once
#include <cfloat>
#include <cmath>

#include "../../include/se2gpu.h"

#if defined(__CUDACC__)
#define SE2_HD __host__ __device__ __forceinline__
#else
#define SE2_HD inline
#endif

namespace se2gpu {

// OptimizationAlgorithmLevenberg::_maxTrialsAfterFailure: lambda trials per iteration before the iteration terminates
constexpr int kLmMaxTrials = 10;

// computeLambdaInit: lambda_0 = tau * max |diag H| over all free vertices, tau = 1e-5
SE2_HD void lm_lambda_init(double max_diag, double& lambda, double& ni) {
    lambda = 1e-5 * max_diag;
    ni = 2.0;
}

// The gain-ratio test and lambda schedule of one trial (OptimizationAlgorithmLevenberg::solve). tempChi: chi2 at the trial
// point, scale: the computeScale() sum; both are replaced by the values the test used (a failed solve rejects the trial).
// rho receives the gain ratio. Returns whether the trial was accepted, in which case chi_cur = tempChi and the caller makes
// the trial state current.
SE2_HD bool lm_gain_step(double& tempChi, double& scale, bool solve_ok, double& chi_cur, double& lambda, double& ni, double& rho) {
    if (!solve_ok) { tempChi = DBL_MAX; scale = 0.0; }
    scale += 1e-3;
    rho = (chi_cur - tempChi) / scale;
    if (rho > 0 && std::isfinite(tempChi)) {
        double alpha = 1. - pow((2 * rho - 1), 3);
        alpha = fmin(alpha, 2. / 3.);
        lambda *= fmax(1. / 3., alpha); ni = 2; chi_cur = tempChi;
        return true;
    }
    lambda *= ni; ni *= 2;
    return false;
}

// do { ... } while (rho < 0 && qmax < _maxTrialsAfterFailure): another trial in the same iteration (a NaN rho stops)
SE2_HD bool lm_retry(double rho, int trials) { return rho < 0 && trials < kLmMaxTrials; }

// the iteration returns Terminate: every trial used, or a zero gain ratio
SE2_HD bool lm_terminate(double rho, int trials) { return trials == kLmMaxTrials || rho == 0; }

// the statistics of one completed iteration
SE2_HD se2gpu_ba_iter_stats lm_iter_stats(double chi_before, double chi_after, double lambda, double rho, int trials, int accepted) {
    se2gpu_ba_iter_stats o;
    o.chi2_before = chi_before; o.chi2_after = chi_after; o.lambda = lambda; o.rho = rho;
    o.trials = trials; o.accepted = accepted; o.terminate = lm_terminate(rho, trials) ? 1 : 0; o.pad = 0;
    return o;
}

// NOT_PD: the iteration terminated and not one of its trials could solve the damped system
SE2_HD bool lm_not_pd(const se2gpu_ba_iter_stats& st, int failed_solves) { return st.terminate && failed_solves == st.trials; }

#if defined(__CUDACC__)

// Fixed-order sum over the CTA of N values per thread: an xor-shuffle tree in each warp, then the WARPS warp sums in index
// order from warp 0 by thread 0 into out. red is shared scratch; the barrier before it is written lets the previous sum
// still be reading it. The bytes do not depend on scheduling or on the CTA's position in a batch.
template <int N, int WARPS, int LD>
__device__ __forceinline__ void cta_sum(double* a, double (&red)[WARPS][LD], double* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], off);
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) red[warp][k] = a[k];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 0; k < N; ++k) {
            double s = red[0][k];
            for (int w = 1; w < WARPS; ++w) s += red[w][k];
            out[k] = s;
        }
}

// the same order for the maximum of one value per thread; the result is valid in thread 0
template <int WARPS, int LD>
__device__ __forceinline__ double cta_max(double v, double (&red)[WARPS][LD]) {
    for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][0] = v;
    __syncthreads();
    double s = red[0][0];
    for (int w = 1; w < WARPS; ++w) s = fmax(s, red[w][0]);
    return s;
}

// In-place dense LL^T of the SPD n x n matrix in the lower triangle of A (row stride ld); the upper triangle is not read
// or written. False when a pivot is not positive or not finite.
__device__ inline bool chol_factor(int n, int ld, double* A) {
    for (int r = 0; r < n; ++r)
        for (int c = 0; c <= r; ++c) {
            double s = A[r * ld + c];
            for (int k = 0; k < c; ++k) s -= A[r * ld + k] * A[c * ld + k];
            if (c == r) {
                if (!(s > 0.0) || !isfinite(s)) return false;
                A[r * ld + r] = sqrt(s);
            } else {
                A[r * ld + c] = s / A[c * ld + c];
            }
        }
    return true;
}

// x = (L L^T)^-1 b for the factor chol_factor left in L
__device__ inline void chol_solve(int n, int ld, const double* L, const double* b, double* x) {
    for (int r = 0; r < n; ++r) {
        double s = b[r];
        for (int k = 0; k < r; ++k) s -= L[r * ld + k] * x[k];
        x[r] = s / L[r * ld + r];
    }
    for (int r = n - 1; r >= 0; --r) {
        double s = x[r];
        for (int k = r + 1; k < n; ++k) s -= L[k * ld + r] * x[k];
        x[r] = s / L[r * ld + r];
    }
}

#endif  // __CUDACC__

}  // namespace se2gpu
