// The reduced solve over 6 x 6 pose blocks shared by the global pose graph (global_ba.cu) and the SE(3)-XYZ window BA
// (se3_ba.cu): the block-envelope Cholesky (LL^T, 6 x 6 pivots) in the order of global_ba_plan.h's symbolic phase, and its
// forward and back substitution. One CTA walks the pivot columns. A is any struct with the plan's arrays (nf, first,
// rowoff, col_ptr, col_rows) and the numeric ones: L [env blocks * 36] (factorised in place), b and x [nf * 6].
#pragma once
#include <cuda_runtime.h>

#include "lm.h"

namespace se2gpu {

template <class A>
__device__ inline const double* blkp(const double* M, const A& a, int p, int q) {
    return M + 36 * (size_t)(a.rowoff[p] + (q - a.first[p]));
}

// block-envelope Cholesky of L in place (lower blocks, row-major 6 x 6); false when a pivot block is not positive definite.
// Every thread of the CTA (THREADS of them) takes part; s_D is 36 doubles of shared memory, s_flag one shared int.
template <int THREADS, class A>
__device__ bool env_factor(const A& a, double* s_D, int* s_flag) {
    double* L = a.L;
    for (int k = 0; k < a.nf; ++k) {
        const int fk = a.first[k];
        if (threadIdx.x < 36) {  // the pivot block's Schur update
            const int r = threadIdx.x / 6, c = threadIdx.x % 6;
            double s = blkp(L, a, k, k)[r * 6 + c];
            for (int j = fk; j < k; ++j) {
                const double* Lkj = blkp(L, a, k, j);
                for (int t = 0; t < 6; ++t) s -= Lkj[r * 6 + t] * Lkj[c * 6 + t];
            }
            s_D[r * 6 + c] = s;
        }
        __syncthreads();
        if (threadIdx.x == 0) {  // dense 6 x 6 LL^T of the pivot
            const int ok = chol_factor(6, 6, s_D);
            double* Lkk = L + 36 * (size_t)(a.rowoff[k] + (k - fk));
            for (int r = 0; r < 6; ++r)
                for (int c = 0; c < 6; ++c) Lkk[r * 6 + c] = c <= r ? s_D[r * 6 + c] : 0.0;
            *s_flag = ok;
        }
        __syncthreads();
        if (!*s_flag) return false;
        const int r0 = a.col_ptr[k], nr = a.col_ptr[k + 1] - r0;
        for (int idx = threadIdx.x; idx < nr * 36; idx += THREADS) {  // the rows below: A_ik - sum_j L_ij L_kj^T
            const int i = a.col_rows[r0 + idx / 36], r = (idx % 36) / 6, c = idx % 6;
            double* Lik = L + 36 * (size_t)(a.rowoff[i] + (k - a.first[i]));
            double s = Lik[r * 6 + c];
            for (int j = max(a.first[i], fk); j < k; ++j) {
                const double* Lij = blkp(L, a, i, j);
                const double* Lkj = blkp(L, a, k, j);
                for (int t = 0; t < 6; ++t) s -= Lij[r * 6 + t] * Lkj[c * 6 + t];
            }
            Lik[r * 6 + c] = s;
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < nr * 6; idx += THREADS) {  // ... times L_kk^-T
            const int i = a.col_rows[r0 + idx / 6], r = idx % 6;
            double* row = L + 36 * (size_t)(a.rowoff[i] + (k - a.first[i])) + r * 6;
            for (int c = 0; c < 6; ++c) {
                double s = row[c];
                for (int t = 0; t < c; ++t) s -= row[t] * s_D[c * 6 + t];
                row[c] = s / s_D[c * 6 + c];
            }
        }
        __syncthreads();
    }
    return true;
}

// L L^T x = b by warp 0: forward over the rows of the envelope, back over its columns
template <class A>
__device__ void env_substitute(const A& a) {
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    double* x = a.x;
    for (int k = 0; k < a.nf; ++k) {
        if (lane < 6) {
            double s = a.b[6 * k + lane];
            for (int j = a.first[k]; j < k; ++j) {
                const double* Lkj = blkp(a.L, a, k, j);
                for (int t = 0; t < 6; ++t) s -= Lkj[lane * 6 + t] * x[6 * j + t];
            }
            x[6 * k + lane] = s;
        }
        __syncwarp();
        if (lane == 0) {
            const double* Lkk = blkp(a.L, a, k, k);
            for (int r = 0; r < 6; ++r) {
                double s = x[6 * k + r];
                for (int t = 0; t < r; ++t) s -= Lkk[r * 6 + t] * x[6 * k + t];
                x[6 * k + r] = s / Lkk[r * 6 + r];
            }
        }
        __syncwarp();
    }
    for (int k = a.nf - 1; k >= 0; --k) {
        if (lane < 6) {
            double s = x[6 * k + lane];
            for (int q = a.col_ptr[k]; q < a.col_ptr[k + 1]; ++q) {
                const int i = a.col_rows[q];
                const double* Lik = blkp(a.L, a, i, k);
                for (int t = 0; t < 6; ++t) s -= Lik[t * 6 + lane] * x[6 * i + t];
            }
            x[6 * k + lane] = s;
        }
        __syncwarp();
        if (lane == 0) {
            const double* Lkk = blkp(a.L, a, k, k);
            for (int r = 5; r >= 0; --r) {
                double s = x[6 * k + r];
                for (int t = r + 1; t < 6; ++t) s -= Lkk[t * 6 + r] * x[6 * k + t];
                x[6 * k + r] = s / Lkk[r * 6 + r];
            }
        }
        __syncwarp();
    }
}

}  // namespace se2gpu
