// Partitioned block-band LDL^T of the reduced pose system S dx = b for windows whose reduced system does not fit one CTA's
// shared memory (BASELINE config 5: 2000 keyframes, n = 5997, block half-bandwidth 5). Replaces, at that scale, the
// single-CTA global-memory envelope factorisation (a chain of n/3 dependent block steps walking through L2) by a
// one-level substructuring (nested dissection of the band) that exposes p-way parallelism:
//
//   block columns:  [ I_0 | s_0 | I_1 | s_1 | ... | s_{p-2} | I_{p-1} ]      separators s_q are w blocks wide (w = block
//   half-bandwidth), so interiors I_k are mutually decoupled.
//   K1 band_part_factor   one CTA per partition, everything in shared memory: block LDL^T (3x3 pivots, the same pivot-warp
//                         look-ahead scheme as the small-window solver) of the interior band A_II, carrying along the
//                         coupling rows to both separators - the left separator's rows fill in over the whole interior
//                         (the "spike" U), the right separator's rows are ordinary band rows - and the right-hand side.
//                         What remains below the interior after the elimination is the partition's Schur contribution
//                         -C A_II^-1 C^T to the separator system, split in its left-left, right-right and right-left blocks.
//   K2 band_sep_solve     one CTA: assembles the separator system T (block tridiagonal in separators, band storage in shared
//                         memory) from S's own separator entries and the p contributions, factorises and solves it.
//   K3 band_part_back     one CTA per partition: back substitution of the interior given its two separators' solutions.
// Dependent chain: |I_k| + w (p-1) block steps instead of n/3 (config 5: 96 + 95 instead of 1999), all in shared memory.
// The factorisation order is a symmetric permutation of S, so "some pivot block not positive definite" is still exactly
// "S not positive definite" (CHOLMOD's minor != n): the trial is rejected.
// Every sum has a fixed order (no atomics): runs are bit-reproducible.
#include <algorithm>
#include <cmath>
#include <cstdio>

#include "ba_band.h"
#include "common.h"
#include "sym3.h"

namespace se2band {

namespace {

constexpr int THREADS = 512;

// ---- block LDL^T on a band-stored matrix in shared memory ----------------------------------------------------------
// Ab: nrows x BW1 (row r holds columns r-bw..r, bw = BW1-1); the first `npiv` 3x3 diagonal blocks are eliminated.
// Optional extra rows U [l3 x nrows] attached to every column (the left separator's coupling rows, dense after fill-in), with
// their own diagonal block Tll [l3 x l3] and right-hand side yl [l3]. y [nrows] is the right-hand side of the band rows.
// a_i = A[i][k..k+2] is left UNSCALED in place (L_ik = a_ik W_k), W [npiv x 9] = inverse pivot blocks.
// tb: 2 x 3 doubles (W_k u_k, double-buffered by step parity); ok: shared int, 0 when a pivot block is not positive definite.
__device__ void band_factor(double* __restrict__ Ab, int BW1, int nrows, int npiv, double* __restrict__ U, int l3,
                            double* __restrict__ Tll, double* __restrict__ y, double* __restrict__ yl, double* __restrict__ W,
                            double* __restrict__ tb, int* ok) {
    const int bw = BW1 - 1;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, wid = tid >> 5;
#define A_(r, c) Ab[(r) * BW1 + ((c) - (r) + bw)]
    auto invert_and_publish = [&](int j) {            // pivot block j (rows/cols 3j..3j+2, final), rhs y[3j..3j+2]
        const int r = 3 * j;
        const double a = A_(r, r), b = A_(r + 1, r), c = A_(r + 2, r), e = A_(r + 1, r + 1), f = A_(r + 2, r + 1), i2 = A_(r + 2, r + 2);
        const double u0 = y[r], u1 = y[r + 1], u2 = y[r + 2];
        const Sym3Inv inv = sym3_inverse(a, b, c, e, f, i2);
        const double w00 = inv.i00, w01 = inv.i01, w02 = inv.i02, w11 = inv.i11, w12 = inv.i12, w22 = inv.i22;
        if (lane == 0) {
            double* Wj = W + 9 * j;
            Wj[0] = w00; Wj[1] = w01; Wj[2] = w02; Wj[3] = w01; Wj[4] = w11; Wj[5] = w12; Wj[6] = w02; Wj[7] = w12; Wj[8] = w22;
            double* t = tb + 3 * (j & 1);
            t[0] = w00 * u0 + w01 * u1 + w02 * u2; t[1] = w01 * u0 + w11 * u1 + w12 * u2; t[2] = w02 * u0 + w12 * u1 + w22 * u2;
            if (!inv.pd) *ok = 0;
        }
    };
    if (wid == 0 && npiv > 0) invert_and_publish(0);
    __syncthreads();
    for (int j = 0; j < npiv; ++j) {
        if (!*ok) break;                               // written before the barrier that precedes this read: uniform
        const int k = 3 * j;
        const double* Wj = W + 9 * j;
        const double w00 = Wj[0], w01 = Wj[1], w02 = Wj[2], w11 = Wj[4], w12 = Wj[5], w22 = Wj[8];
        const double* t = tb + 3 * (j & 1);
        const double t0 = t[0], t1 = t[1], t2 = t[2];
        const int rmax = min(k + bw, nrows - 1);       // last row / column coupled to pivot block j
        const int R = rmax - (k + 3) + 1;              // trailing rows k+3 .. rmax
        if (wid == 0) {
            // look-ahead: rows k+3..k+5 (the next pivot block, or the first rows below the eliminated part) and their rhs
            if (R >= 3 && lane < 9) {
                const int q = lane;                    // 0..5: (ii,jj) = (0,0)(1,0)(1,1)(2,0)(2,1)(2,2); 6..8: rhs of row q-6
                const int ii = q < 1 ? 0 : (q < 3 ? 1 : (q < 6 ? 2 : q - 6));
                const int jj = q < 1 ? 0 : (q < 3 ? q - 1 : (q < 6 ? q - 3 : 0));
                const int i = k + 3 + ii, c = k + 3 + jj;
                const double a0 = A_(i, k), a1 = A_(i, k + 1), a2 = A_(i, k + 2);
                if (q < 6) {
                    const double b0 = A_(c, k), b1 = A_(c, k + 1), b2 = A_(c, k + 2);
                    const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                    A_(i, c) -= a0 * v0 + a1 * v1 + a2 * v2;
                } else {
                    y[i] -= a0 * t0 + a1 * t1 + a2 * t2;
                }
            }
            __syncwarp();
            if (j + 1 < npiv) invert_and_publish(j + 1);
        } else if (R > 0 || l3 > 0) {
            const int wk = tid - 32, nwk = nt - 32;
            // work items of this step: [0, R*R) band (row ii, col cc <= ii; rows ii < 3 belong to the look-ahead),
            // then l3*R spike entries, l3*l3 left-left entries (lower triangle), R + l3 right-hand-side entries
            const int Rp = R > 0 ? R : 0;
            const int n_band = Rp * Rp, n_spike = l3 * Rp, n_ll = l3 * l3, total = n_band + n_spike + n_ll + Rp + l3;
            for (int id = wk; id < total; id += nwk) {
                if (id < n_band) {
                    const int ii = id / Rp, cc = id - ii * Rp;
                    if (ii < 3 || cc > ii) continue;
                    const int i = k + 3 + ii, c = k + 3 + cc;
                    const double a0 = A_(i, k), a1 = A_(i, k + 1), a2 = A_(i, k + 2);
                    const double b0 = A_(c, k), b1 = A_(c, k + 1), b2 = A_(c, k + 2);
                    const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                    A_(i, c) -= a0 * v0 + a1 * v1 + a2 * v2;
                } else if (id < n_band + n_spike) {
                    const int e = id - n_band, tt = e / Rp, cc = e - tt * Rp;
                    const int c = k + 3 + cc;
                    const double* ur = U + (size_t)tt * nrows;
                    const double a0 = ur[k], a1 = ur[k + 1], a2 = ur[k + 2];
                    const double b0 = A_(c, k), b1 = A_(c, k + 1), b2 = A_(c, k + 2);
                    const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                    U[(size_t)tt * nrows + c] -= a0 * v0 + a1 * v1 + a2 * v2;
                } else if (id < n_band + n_spike + n_ll) {
                    const int e = id - n_band - n_spike, tt = e / l3, t2i = e - tt * l3;
                    if (t2i > tt) continue;
                    const double* ur = U + (size_t)tt * nrows; const double* uc = U + (size_t)t2i * nrows;
                    const double a0 = ur[k], a1 = ur[k + 1], a2 = ur[k + 2];
                    const double b0 = uc[k], b1 = uc[k + 1], b2 = uc[k + 2];
                    const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                    Tll[tt * l3 + t2i] -= a0 * v0 + a1 * v1 + a2 * v2;
                } else {
                    const int e = id - n_band - n_spike - n_ll;
                    if (e < Rp) {
                        if (e < 3) continue;           // look-ahead rows
                        const int i = k + 3 + e;
                        y[i] -= A_(i, k) * t0 + A_(i, k + 1) * t1 + A_(i, k + 2) * t2;
                    } else {
                        const int tt = e - Rp;
                        const double* ur = U + (size_t)tt * nrows;
                        yl[tt] -= ur[k] * t0 + ur[k + 1] * t1 + ur[k + 2] * t2;
                    }
                }
            }
        }
        __syncthreads();
    }
    __syncthreads();
#undef A_
}

// Back substitution x_k = W_k (z_k - sum_{i>k} a_ik^T x_i) for the first npiv blocks, axpy form: thread c owns the running
// z_c of column c (needs blockDim.x >= 3 npiv). z arrives in `z` with the contributions of all rows >= 3 npiv already
// subtracted; on return z holds x. xz: 2 x 3 doubles of exchange space.
__device__ void band_backsolve(const double* __restrict__ Ab, int BW1, int npiv, const double* __restrict__ W, double* __restrict__ z,
                               double* __restrict__ xz) {
    const int bw = BW1 - 1, c = threadIdx.x, n3 = 3 * npiv;
    double zc = c < n3 ? z[c] : 0.0;
    for (int kb = npiv - 1; kb >= 0; --kb) {
        const int k = 3 * kb;
        double* ex = xz + 3 * (kb & 1);
        if (c >= k && c < k + 3) ex[c - k] = zc;
        __syncthreads();
        const double* Wk = W + 9 * kb;
        const double z0 = ex[0], z1 = ex[1], z2 = ex[2];
        const double x0 = Wk[0] * z0 + Wk[1] * z1 + Wk[2] * z2, x1 = Wk[3] * z0 + Wk[4] * z1 + Wk[5] * z2, x2 = Wk[6] * z0 + Wk[7] * z1 + Wk[8] * z2;
        if (c < k) {
            // rows k..k+2 of column c, where inside the band
            const double a0 = (k - c <= bw) ? Ab[(size_t)k * BW1 + (c - k + bw)] : 0.0;
            const double a1 = (k + 1 - c <= bw) ? Ab[(size_t)(k + 1) * BW1 + (c - k - 1 + bw)] : 0.0;
            const double a2 = (k + 2 - c <= bw) ? Ab[(size_t)(k + 2) * BW1 + (c - k - 2 + bw)] : 0.0;
            zc -= a0 * x0 + a1 * x1 + a2 * x2;
        }
        zc = (c == k) ? x0 : (c == k + 1) ? x1 : (c == k + 2) ? x2 : zc;
    }
    if (c < n3) z[c] = zc;
    __syncthreads();
}

struct Sm {                              // carve-up of a partition's shared memory / workspace (doubles)
    int m3, r3, l3, nrows, BW1, m;
    size_t oAb, oU, oTll, oY, oYl, oW, total;
    __host__ __device__ Sm(int m_, int l3_, int r3_, int BW1_) {
        m = m_; m3 = 3 * m_; l3 = l3_; r3 = r3_; nrows = m3 + r3; BW1 = BW1_;
        oAb = 0; oU = oAb + (size_t)nrows * BW1; oTll = oU + (size_t)l3 * nrows; oY = oTll + (size_t)l3 * l3; oYl = oY + nrows;
        oW = oYl + l3; total = oW + (size_t)9 * m;
    }
};

__global__ void __launch_bounds__(THREADS) band_part_factor(const Part* __restrict__ parts, int BW1, const double* __restrict__ S,
                                                            const double* __restrict__ bs, double* __restrict__ work, int* __restrict__ okv) {
    extern __shared__ double sm[];
    __shared__ double tb[6];
    __shared__ int ok;
    const Part pt = parts[blockIdx.x];
    const Sm L(pt.a1 - pt.a0, pt.l3, pt.r3, BW1);
    const int bw = BW1 - 1, g0 = 3 * pt.a0;
    double *Ab = sm + L.oAb, *U = sm + L.oU, *Tll = sm + L.oTll, *y = sm + L.oY, *yl = sm + L.oYl, *W = sm + L.oW;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) ok = 1;
    // band rows: interior rows verbatim; right-separator rows keep only their coupling to the interior
    for (int e = tid; e < L.nrows * BW1; e += nt) {
        const int r = e / BW1, s = e - r * BW1, c = r + s - bw;          // local column
        double v = 0.0;
        if (r < L.m3 || c < L.m3) v = S[(size_t)(g0 + r) * BW1 + s];
        Ab[e] = v;
    }
    // spike rows: U[t][c] = S[g0 + c][g0 - l3 + t] for interior columns c close to the left separator, zero elsewhere
    for (int e = tid; e < L.l3 * L.nrows; e += nt) {
        const int t = e / L.nrows, c = e - t * L.nrows;
        const int gr = g0 + c, gc = g0 - L.l3 + t;
        U[e] = (c < L.m3 && gr - gc <= bw) ? S[(size_t)gr * BW1 + (gc - gr + bw)] : 0.0;
    }
    for (int e = tid; e < L.l3 * L.l3; e += nt) Tll[e] = 0.0;
    for (int e = tid; e < L.nrows; e += nt) y[e] = e < L.m3 ? bs[g0 + e] : 0.0;
    for (int e = tid; e < L.l3; e += nt) yl[e] = 0.0;
    __syncthreads();
    band_factor(Ab, BW1, L.nrows, L.m, U, L.l3, Tll, y, yl, W, tb, &ok);
    double* out = work + pt.ws;
    for (size_t e = tid; e < L.total; e += nt) out[e] = sm[e];
    if (tid == 0) okv[blockIdx.x] = ok;
}

// separator system: unknowns = the separators' scalars in order; band half-width bwT = l3 + r3 - 1 (two adjacent separators)
__global__ void __launch_bounds__(THREADS) band_sep_solve(const Part* __restrict__ parts, int p, int BW1, int w3, int nT, const double* __restrict__ S,
                                                          const double* __restrict__ bs, const double* __restrict__ work, int* __restrict__ okv,
                                                          double* __restrict__ dxp, int n, int* __restrict__ solve_ok) {
    extern __shared__ double sm[];
    __shared__ double tb[6], xz[6];
    __shared__ int ok;
    const int bw = BW1 - 1, BWT1 = 2 * w3, bwT = BWT1 - 1;
    double* T = sm;                               // nT x BWT1
    double* yT = T + (size_t)nT * BWT1;            // nT
    double* W = yT + nT;                           // (nT/3) x 9
    const int tid = threadIdx.x, nt = blockDim.x;
    int all_ok = 1;
    for (int k = 0; k < p; ++k) all_ok &= okv[k];
    if (tid == 0) ok = 1;
    for (int e = tid; e < nT * BWT1; e += nt) {
        const int r = e / BWT1, s = e - r * BWT1, c = r + s - bwT;       // separator-system row / column
        double v = 0.0;
        if (c >= 0) {
            const int q = r / w3, rr = r - q * w3, qc = c / w3, cc = c - qc * w3;      // separator index, offset inside it
            const Part pq = parts[q];                                   // partition left of separator q
            const Sm Lq(pq.a1 - pq.a0, pq.l3, pq.r3, BW1);
            const double* wq = work + pq.ws;
            if (qc == q) {
                // S's own entry + right-right part of partition q + left-left part of partition q+1
                const int gr = 3 * pq.a1 + rr, gc = 3 * pq.a1 + cc;
                if (gr - gc <= bw) v = S[(size_t)gr * BW1 + (gc - gr + bw)];
                const int lr = Lq.m3 + rr, lc = Lq.m3 + cc;
                if (lr - lc <= bw) v += wq[Lq.oAb + (size_t)lr * BW1 + (lc - lr + bw)];
                const Part pn = parts[q + 1];
                const Sm Ln(pn.a1 - pn.a0, pn.l3, pn.r3, BW1);
                v += work[pn.ws + Ln.oTll + (size_t)rr * Ln.l3 + cc];
            } else if (qc == q - 1) {
                // right-left part of partition q: rows = right separator (q), columns = left separator (q-1): U[cc][m3 + rr]
                v = wq[Lq.oU + (size_t)cc * Lq.nrows + (Lq.m3 + rr)];
            }
        }
        T[e] = v;
    }
    for (int r = tid; r < nT; r += nt) {
        const int q = r / w3, rr = r - q * w3;
        const Part pq = parts[q], pn = parts[q + 1];
        const Sm Lq(pq.a1 - pq.a0, pq.l3, pq.r3, BW1), Ln(pn.a1 - pn.a0, pn.l3, pn.r3, BW1);
        yT[r] = bs[3 * pq.a1 + rr] + work[pq.ws + Lq.oY + Lq.m3 + rr] + work[pn.ws + Ln.oYl + rr];
    }
    __syncthreads();
    if (all_ok) band_factor(T, BWT1, nT, nT / 3, nullptr, 0, nullptr, yT, nullptr, W, tb, &ok);
    __syncthreads();
    const int good = all_ok && ok;
    if (good) band_backsolve(T, BWT1, nT / 3, W, yT, xz);
    for (int r = tid; r < nT; r += nt) {
        const int q = r / w3, rr = r - q * w3;
        dxp[3 * parts[q].a1 + rr] = good ? yT[r] : 0.0;
    }
    if (tid == 0) { okv[p] = good; *solve_ok = good; }
    (void)n;
}

__global__ void __launch_bounds__(THREADS) band_part_back(const Part* __restrict__ parts, int p, int BW1, const double* __restrict__ work,
                                                          const int* __restrict__ okv, double* __restrict__ dxp) {
    extern __shared__ double sm[];
    __shared__ double xz[6];
    const Part pt = parts[blockIdx.x];
    const Sm L(pt.a1 - pt.a0, pt.l3, pt.r3, BW1);
    const int bw = BW1 - 1, g0 = 3 * pt.a0, tid = threadIdx.x, nt = blockDim.x;
    if (!okv[p]) {                                   // not positive definite: the trial is rejected, the step is zero
        for (int e = tid; e < L.m3; e += nt) dxp[g0 + e] = 0.0;
        return;
    }
    const double* in = work + pt.ws;
    for (size_t e = tid; e < L.total; e += nt) sm[e] = in[e];
    __shared__ double xs[2 * 96];                    // solutions of the left / right separator (<= 32 blocks wide each... see plan())
    for (int e = tid; e < L.l3; e += nt) xs[e] = dxp[g0 - L.l3 + e];
    for (int e = tid; e < L.r3; e += nt) xs[96 + e] = dxp[g0 + L.m3 + e];
    __syncthreads();
    double *Ab = sm + L.oAb, *U = sm + L.oU, *y = sm + L.oY, *W = sm + L.oW;
    // z_c = u_c - U[:, c]^T x_left - sum over right-separator rows inside the band of A[i][c] x_i
    for (int c = tid; c < L.m3; c += nt) {
        double zc = y[c];
        for (int t = 0; t < L.l3; ++t) zc -= U[(size_t)t * L.nrows + c] * xs[t];
        for (int i = L.m3; i < L.nrows && i - c <= bw; ++i) zc -= Ab[(size_t)i * BW1 + (c - i + bw)] * xs[96 + i - L.m3];
        y[c] = zc;
    }
    __syncthreads();
    band_backsolve(Ab, BW1, L.m, W, y, xz);
    for (int c = tid; c < L.m3; c += nt) dxp[g0 + c] = y[c];
}

}  // namespace

bool plan(Plan& pl, int nf, const std::vector<int>& bmax, int smem_optin) {
    release(pl);
    pl.active = false;
    int w = 0;
    for (int a = 0; a < nf; ++a) w = std::max(w, bmax[a] - a);
    if (w < 1 || w > 10 || nf < 4 * w + 4) return false;
    const int w3 = 3 * w, bw = 3 * w + 2, BW1 = bw + 1;
    const size_t budget = smem_optin > 4096 ? (size_t)smem_optin - 2048 : 46 * 1024;
    int best_p = 0; double best_cost = 1e300;
    for (int p = 2; p <= 64; ++p) {
        const int tot_int = nf - w * (p - 1);
        if (tot_int < p * std::max(w, 2)) break;
        const int m = (tot_int + p - 1) / p;                   // largest interior
        const int nT = w3 * (p - 1);
        if (3 * m > THREADS - 32 || nT > THREADS - 32) continue;   // one thread per column in the back substitutions
        const Sm L(m, w3, w3, BW1);
        const size_t smem_part = L.total * sizeof(double);
        const size_t smem_sep = ((size_t)nT * 2 * w3 + nT + 3 * (size_t)nT) * sizeof(double);
        if (smem_part > budget || smem_sep > budget) continue;
        const double cost = m + 1.15 * w * (p - 1);            // dependent block steps: interior chain + separator chain (wider band)
        if (cost < best_cost) { best_cost = cost; best_p = p; }
    }
    if (!best_p) return false;
    const int p = best_p;
    pl.n = 3 * nf; pl.nf = nf; pl.w = w; pl.bw = bw; pl.p = p; pl.nT = w3 * (p - 1); pl.bwT = 2 * w3 - 1;
    pl.band_elems = (size_t)pl.n * BW1;
    const int tot_int = nf - w * (p - 1), base = tot_int / p, extra = tot_int % p;
    pl.parts.clear();
    long long off = 0; int pos = 0; size_t smem_part = 0;
    for (int k = 0; k < p; ++k) {
        const int m = base + (k < extra ? 1 : 0);
        Part pt{};
        pt.a0 = pos; pt.a1 = pos + m; pt.l3 = k > 0 ? w3 : 0; pt.r3 = k < p - 1 ? w3 : 0;
        const Sm L(m, pt.l3, pt.r3, BW1);
        pt.ws = off; pt.ws_elems = (long long)L.total; off += (long long)((L.total + 31) & ~(size_t)31);
        smem_part = std::max(smem_part, L.total * sizeof(double));
        pl.max_m3 = std::max(pl.max_m3, 3 * m);
        pl.parts.push_back(pt);
        pos = pt.a1 + w;
    }
    pl.smem_part = smem_part;
    pl.smem_sep = ((size_t)pl.nT * 2 * w3 + pl.nT + 3 * (size_t)pl.nT) * sizeof(double);
    if (cudaMalloc((void**)&pl.d_parts, sizeof(Part) * p) != cudaSuccess || cudaMalloc((void**)&pl.d_work, sizeof(double) * (size_t)off) != cudaSuccess ||
        cudaMalloc((void**)&pl.d_ok, sizeof(int) * (p + 1)) != cudaSuccess ||
        cudaMemcpy(pl.d_parts, pl.parts.data(), sizeof(Part) * p, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaGetLastError(); release(pl); return false;
    }
    if (cudaFuncSetAttribute(band_part_factor, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget) != cudaSuccess ||
        cudaFuncSetAttribute(band_sep_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget) != cudaSuccess ||
        cudaFuncSetAttribute(band_part_back, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget) != cudaSuccess) {
        cudaGetLastError(); release(pl); return false;
    }
    pl.active = true;
    return true;
}

void release(Plan& pl) {
    if (pl.d_parts) cudaFree(pl.d_parts);
    if (pl.d_work) cudaFree(pl.d_work);
    if (pl.d_ok) cudaFree(pl.d_ok);
    pl.d_parts = nullptr; pl.d_work = nullptr; pl.d_ok = nullptr; pl.active = false;
}

int solve(const Plan& pl, const double* Sband, const double* bs, double* dxp, int* solve_ok, cudaStream_t s) {
    SE2_NVTX("se2gpu.ba.band_solve");
    const int BW1 = pl.bw + 1;
    SE2_LAUNCH(band_part_factor, pl.p, THREADS, pl.smem_part, s, pl.d_parts, BW1, Sband, bs, pl.d_work, pl.d_ok);
    SE2_LAUNCH(band_sep_solve, 1, THREADS, pl.smem_sep, s, pl.d_parts, pl.p, BW1, 3 * pl.w, pl.nT, Sband, bs, pl.d_work, pl.d_ok, dxp, pl.n, solve_ok);
    SE2_LAUNCH(band_part_back, pl.p, THREADS, pl.smem_part, s, pl.d_parts, pl.p, BW1, pl.d_work, pl.d_ok, dxp);
    return SE2GPU_OK;
}

}  // namespace se2band
