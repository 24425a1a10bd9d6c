// Assembly and solve of the reduced system over 6 x 6 pose blocks, shared by the global pose graph (global_ba.cu) and the
// SE(3)-XYZ window BA (se3_ba.cu), in the order of global_ba_plan.h's symbolic phase:
//  * assembly: the 120-double record of one SE(3) link (edge_record), the gathers of H's diagonal blocks with b
//    (gather_diag) and of its off-diagonal blocks (gather_off) from those records in the plan's fixed order, and the
//    damping of the pose diagonal (damp). Each takes the first index and the stride of its loop, so the one-CTA kernel
//    passes (threadIdx.x, threads) and a cooperative kernel its grid-wide (thread, stride);
//  * solve: the block-envelope Cholesky (LL^T, 6 x 6 pivots) and its forward and back substitution, one CTA walking the
//    pivot columns.
// A is any struct with the plan's arrays (nf, first, rowoff, col_ptr, col_rows, and for the gathers pH, pb, Hs, diag_ptr,
// diag_code, S, off_blk, off_ptr, off_code) and, for the solve, the numeric ones: L [env blocks * 36] (factorised in
// place), b and x [nf * 6].
#pragma once
#include <cuda_runtime.h>

#include "global_ba_plan.h"
#include "lm.h"

namespace se2gpu {

constexpr int kEdgeRec = 120;  // per link: H_ii, H_jj, H_ij (36 each), b_i, b_j (6 each)

// block (p, q) of an envelope matrix, first[p] <= q <= p
template <class T, class A>
__device__ inline T* blkp(T* M, const A& a, int p, int q) {
    return M + 36 * (size_t)(a.rowoff[p] + (q - a.first[p]));
}

// one link's record from its error e, information Om and Jacobians J[0] (i) and J[1] (j): H_ii = Ji^T Om Ji, H_jj,
// H_ij = Ji^T Om Jj, b_i = -Ji^T Om e, b_j
__device__ __forceinline__ void edge_record(const double* Om, const double* e, const double (&J)[2][36], double* out) {
    double Oe[6];
    for (int r = 0; r < 6; ++r) {
        double acc = 0;
        for (int c = 0; c < 6; ++c) acc += Om[r * 6 + c] * e[c];
        Oe[r] = acc;
    }
    for (int s = 0; s < 2; ++s) {
        double OJ[36];
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
                double acc = 0;
                for (int m = 0; m < 6; ++m) acc += Om[r * 6 + m] * J[s][m * 6 + c];
                OJ[r * 6 + c] = acc;
            }
        for (int r = 0; r < 6; ++r) {
            for (int c = 0; c < 6; ++c) {
                double acc = 0;
                for (int m = 0; m < 6; ++m) acc += J[s][m * 6 + r] * OJ[m * 6 + c];
                out[36 * s + r * 6 + c] = acc;  // s = 0: H_ii, s = 1: H_jj
                if (s == 1) {
                    double ij = 0;
                    for (int m = 0; m < 6; ++m) ij += J[0][m * 6 + r] * OJ[m * 6 + c];
                    out[72 + r * 6 + c] = ij;
                }
            }
            double acc = 0;
            for (int m = 0; m < 6; ++m) acc += J[s][m * 6 + r] * Oe[m];
            out[108 + 6 * s + r] = -acc;
        }
    }
}

// the diagonal blocks of H into Hs and b: entry rc of position p (rc < 36 the block, else b) is the prior's pH / pb entry,
// plus the records `rec` of the links in diag_code for which active(link) holds, in list order; then more(p, rc, s) adds
// what the caller gathers after the links
template <class A, class Active, class More>
__device__ __forceinline__ void gather_diag(const A& a, const double* rec, double* b, int start, int stride, Active active, More more) {
    for (int idx = start; idx < a.nf * 42; idx += stride) {
        const int p = idx / 42, rc = idx % 42;
        const bool isb = rc >= 36;
        double s = isb ? a.pb[6 * (size_t)p + rc - 36] : a.pH[36 * (size_t)p + rc];
        for (int q = a.diag_ptr[p]; q < a.diag_ptr[p + 1]; ++q) {
            const int code = a.diag_code[q], e = code >> 2, side = code & 3;
            if (!active(e)) continue;
            s += isb ? rec[kEdgeRec * (size_t)e + 108 + 6 * side + rc - 36] : rec[kEdgeRec * (size_t)e + 36 * side + rc];
        }
        s = more(p, rc, s);
        if (isb) b[6 * (size_t)p + rc - 36] = s;
        else blkp(a.Hs, a, p, p)[rc] = s;
    }
}

// the off-diagonal blocks of H into Hs: entry rc of nonzero block sl is the sum of H_ij (kOffDiag) or H_ij^T (kOffDiagT)
// over the links in off_code for which active(link) holds, in list order
template <class A, class Active>
__device__ __forceinline__ void gather_off(const A& a, const double* rec, int start, int stride, Active active) {
    for (int idx = start; idx < a.S * 36; idx += stride) {
        const int sl = idx / 36, rc = idx % 36, tr = (rc % 6) * 6 + rc / 6;
        double s = 0;
        for (int q = a.off_ptr[sl]; q < a.off_ptr[sl + 1]; ++q) {
            const int code = a.off_code[q], e = code >> 2;
            if (!active(e)) continue;
            s += rec[kEdgeRec * (size_t)e + 72 + ((code & 3) == gba::kOffDiag ? rc : tr)];
        }
        a.Hs[36 * (size_t)a.off_blk[sl] + rc] = s;
    }
}

// L + lambda I on the pose diagonal
template <class A>
__device__ __forceinline__ void damp(const A& a, double* L, double lambda, int start, int stride) {
    for (int idx = start; idx < a.nf * 6; idx += stride) blkp(L, a, idx / 6, idx / 6)[(idx % 6) * 7] += lambda;
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
            double* Lkk = L + 36 * (size_t)(a.rowoff[k] + (k - fk));  // blkp(L, a, k, k) with first[k] loaded before the barrier
            for (int r = 0; r < 6; ++r)
                for (int c = 0; c < 6; ++c) Lkk[r * 6 + c] = c <= r ? s_D[r * 6 + c] : 0.0;
            *s_flag = ok;
        }
        __syncthreads();
        if (!*s_flag) return false;
        const int r0 = a.col_ptr[k], nr = a.col_ptr[k + 1] - r0;
        for (int idx = threadIdx.x; idx < nr * 36; idx += THREADS) {  // the rows below: A_ik - sum_j L_ij L_kj^T
            const int i = a.col_rows[r0 + idx / 36], r = (idx % 36) / 6, c = idx % 6;
            double* Lik = blkp(L, a, i, k);
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
            double* row = blkp(L, a, i, k) + r * 6;
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
