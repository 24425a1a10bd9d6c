// SE(2)-XYZ local bundle adjustment on sm_90a — kernels + C ABI (include/se2gpu.h).
//
// Replaces, for graphs made of VertexSE2 / VertexSBAPointXYZ / EdgeSE2XYZ / PreEdgeSE2, the work done
// inside SlamOptimizer::optimize (reference src/LocalMapper.cpp:259-260): per-edge error and analytic
// Jacobians (src/EdgeSE2XYZ.cpp:61-106, include/se2lam/EdgeSE2XYZ.h:62-102), Huber-weighted quadratic
// forms, Schur complement onto the pose block, the reduced solve, landmark back-substitution, the
// additive oplus update and g2o's Levenberg-Marquardt control (restated in SURVEY.md section 8a B6-B10).
//
// Design (DESIGN.md section 3): every accumulation is a GATHER with a fixed summation order, so a run is
// bit-reproducible and free of atomics. Two execution modes:
//   * ba_persistent (one GPU, reduced system <= 156 unknowns): the whole optimize() call is ONE cooperative kernel, the
//     phases separated by grid barriers, LM control evaluated redundantly by every CTA;
//   * one kernel per phase (large windows, sharded runs without peer exchange, set_mode(1)), the reduced system of a
//     sharded run summed through the all-reduce callback.
// ba_persistent's body is a template over the team of CTAs that runs one window (GridTeam / ClusterTeam):
// ba_persistent_cluster runs it on one thread-block cluster per window, many windows per launch (se2gpu_ba_optimize_batch).
// Both modes call the same LM phase functions (section "LM phase functions" below): pk_landmark (EdgeSE2XYZ error, Huber
// weighting, Hll/bl, Hpl/PH records), pk_odo (PreEdgeSE2), lm_damp (damping terms), pk_pose_item and pose_odo_gather
// (pose-side gather), schur_pairs / schur_odo / schur_pose_sweep (Schur gathers of ba_schur and pk_phase_schur_par),
// pose_oplus / pose_scale, diag_absmax and cta_max (lambda_0); the LM control is lm.h's, and sym3_inverse (sym3.h) is
// shared with the LDL^T solvers. pk_schur_item and the landmark back-substitution keep a copy per mode (see
// there: register allocation of ba_persistent). The multi-launch kernels:
//   ba_linearize<JAC>   per landmark (one thread, JAC) or robust chi2 only (!JAC, at x_trial); extra blocks do the
//                       PreEdgeSE2 odometry edges
//   ba_pose_reduce      one CTA per free pose -> Hpp diag, bp
//   ba_iter_begin       currentChi, lambda_0 at iteration 0 (ba_pose_diag_max: rank-summed pose diagonal, sharded runs)
//   ba_lm_prep          per landmark (Hll+lambda I)^-1, Y_e = Hpl_e Hll^-1, g_e = Hpl_e Hll^-1 bl
//   ba_schur            one CTA per non-zero 3x3 block of S gathers its (edge,edge) pair list
//   ba_chol_solve_smem / _gmem   one CTA: block LDL^T (3x3 pivots) of S inside its envelope + back substitution
//                       (large windows: the partitioned band solver, ba_band.cu)
//   ba_backsub_update   per landmark back-substitution, x_trial = x (+) dx, gain-ratio denominator partials
//   ba_decide           g2o's rho test / lambda schedule on device; host reads one small struct per trial
#include <cooperative_groups.h>
#include <cfloat>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <chrono>
#include <vector>
#include <algorithm>
#include <mutex>
#include <unordered_map>

#include "ba_context.h"
#include "lm.h"
#include "sym3.h"

using namespace se2ba;

namespace {

using se2gpu::fail;
using se2gpu::lm_gain_step;
using se2gpu::lm_iter_stats;
using se2gpu::lm_lambda_init;
using se2gpu::lm_retry;

constexpr int CHOL_THREADS = 512;

// A per-edge record is 96 bytes (three 32-byte sectors), 32-byte aligned: gathers read it with 16-byte loads - the record gathers of the
// Schur phase are bound by L1 wavefronts (every lane hits a different record), so halving the load instructions per record halves them.
__device__ __forceinline__ void load_rec10(const double* __restrict__ rec, double* v) {
    const double2* r2 = reinterpret_cast<const double2*>(rec);
#pragma unroll
    for (int q = 0; q < 5; ++q) { const double2 t = r2[q]; v[2 * q] = t.x; v[2 * q + 1] = t.y; }
}
__device__ __forceinline__ void load_rec12(const double* __restrict__ rec, double* v) {
    const double2* r2 = reinterpret_cast<const double2*>(rec);
#pragma unroll
    for (int q = 0; q < 6; ++q) { const double2 t = r2[q]; v[2 * q] = t.x; v[2 * q + 1] = t.y; }
}

// element (r, c), r >= c, of the reduced system
__device__ __forceinline__ size_t sidx(const Dev& d, int r, int c) {
    return d.sbw ? (size_t)r * (d.sbw + 1) + (size_t)(c - r + d.sbw) : (size_t)r * d.n + c;
}

__device__ __forceinline__ double normalize_theta(double theta) {
    if (theta >= -M_PI && theta < M_PI) return theta;
    double multiplier = floor(theta / (2 * M_PI));
    theta = theta - multiplier * 2 * M_PI;
    if (theta >= M_PI) theta -= 2 * M_PI;
    if (theta < -M_PI) theta += 2 * M_PI;
    return theta;
}

// EdgeSE2XYZ::computeError / linearizeOplus (EdgeSE2XYZ.cpp:61-106), closed form:
// lc = Rcb Rz(-theta) (lw - (x,y,0)) + tcb ; e = fx*(lc.xy/lc.z) + c - uv ; M = Jpi Rcw ;
// J_pose = [-M[:,0:2] | M (d.y,-d.x,0)^T] ; J_point = M
// EXPLICIT: the camera-frame point as the rounding sequence nvcc contracts it to when the camera is a kernel parameter
// (ba_persistent): fma(Rcw2, d2, fma(Rcw0, d0, Rcw1 * d1)) + tcb. ba_persistent_cluster reads the camera from shared memory;
// left to itself nvcc then hoists Rcb2 * d2 out of the edge loop and rounds it on its own in one copy, and the two kernels
// would differ in the last bits for a camera whose extrinsic products are inexact.
template <bool JAC, bool EXPLICIT = false>
__device__ __forceinline__ void edge_xyz(const Cam& cam, const double* __restrict__ ps, const double* __restrict__ lw,
                                         double u, double v, double* err, double* A, double* B) {
    double s, c;
    sincos(ps[2], &s, &c);
    double Rcw[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        Rcw[r * 3 + 0] = cam.Rcb[r * 3 + 0] * c - cam.Rcb[r * 3 + 1] * s;
        Rcw[r * 3 + 1] = cam.Rcb[r * 3 + 0] * s + cam.Rcb[r * 3 + 1] * c;
        Rcw[r * 3 + 2] = cam.Rcb[r * 3 + 2];
    }
    const double d0 = lw[0] - ps[0], d1 = lw[1] - ps[1], d2 = lw[2];
    double lc[3];
    if (EXPLICIT) {
#pragma unroll
        for (int r = 0; r < 3; ++r)
            lc[r] = __dadd_rn(__fma_rn(Rcw[r * 3 + 2], d2, __fma_rn(Rcw[r * 3], d0, __dmul_rn(Rcw[r * 3 + 1], d1))), cam.tcb[r]);
    } else {
#pragma unroll
        for (int r = 0; r < 3; ++r) lc[r] = Rcw[r * 3] * d0 + Rcw[r * 3 + 1] * d1 + Rcw[r * 3 + 2] * d2 + cam.tcb[r];
    }
    const double zi = 1.0 / lc[2];
    err[0] = lc[0] * zi * cam.fx + cam.cx - u;
    err[1] = lc[1] * zi * cam.fx + cam.cy - v;
    if (JAC) {
        const double zi2 = zi * zi;
        const double j00 = cam.fx * zi, j02 = -cam.fx * lc[0] * zi2, j12 = -cam.fx * lc[1] * zi2;
        double M[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            M[k] = j00 * Rcw[k] + j02 * Rcw[6 + k];
            M[3 + k] = j00 * Rcw[3 + k] + j12 * Rcw[6 + k];
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            A[r * 3 + 0] = -M[r * 3 + 0];
            A[r * 3 + 1] = -M[r * 3 + 1];
            A[r * 3 + 2] = M[r * 3 + 0] * d1 - M[r * 3 + 1] * d0;
            B[r * 3 + 0] = M[r * 3 + 0];
            B[r * 3 + 1] = M[r * 3 + 1];
            B[r * 3 + 2] = M[r * 3 + 2];
        }
    }
}

__device__ __forceinline__ double block_sum(double v, double* sh) {
    // deterministic: warp tree (xor shuffles) then warp 0 sums the per-warp values in order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double r = 0;
    if (w == 0) {
        r = l < nw ? sh[l] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    return r;  // valid in warp 0
}

// =================================================================================================
// LM phase functions. Both execution modes run the arithmetic of every phase through these: the multi-launch kernels with
// one thread per landmark (LANES = 1) and their own launch geometry, the persistent kernel with LPL lanes per landmark and
// its work split. What differs between the modes - the index mapping and the order of the final reductions - stays with
// the callers.
constexpr int LPL = 8;   // lanes per landmark in the persistent kernel

__device__ __forceinline__ double group_sum(double v) {   // sum over the LPL-lane group, fixed order
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// block-wide max, same order in every CTA; result broadcast to all threads
__device__ double cta_max(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double m = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, sh[w]);
    __syncthreads();
    return m;
}

// max |diagonal| of the symmetric 3x3 block j of a component-major array H [6][stride] (Hll or Hpp)
__device__ __forceinline__ double diag_absmax(const double* H, size_t stride, int j) {
    return fmax(fabs(H[j]), fmax(fabs(H[3 * stride + j]), fabs(H[5 * stride + j])));
}

// Damping-dependent terms of landmark j from its sums Hll = {h00 .. h22} and bl = {b0, b1, b2}: (Hll + lambda I)^-1, stored
// by lane 0, and for the landmark's edges beg+sub, beg+sub+lanes, ... the record Y_e = Hpl_e Hll^-1 | g_e = Hpl_e (Hll^-1 bl)
__device__ __forceinline__ void lm_damp(const Dev& d, int j, int beg, int end, int sub, int lanes, double lam, double h00, double h01,
                                        double h02, double h11, double h12, double h22, double b0, double b1, double b2) {
    const size_t L = d.L;
    const Sym3Inv inv = sym3_inverse(h00 + lam, h01, h02, h11 + lam, h12, h22 + lam);
    const double i00 = inv.i00, i01 = inv.i01, i02 = inv.i02, i11 = inv.i11, i12 = inv.i12, i22 = inv.i22;
    if (sub == 0) { d.HllInv[j] = i00; d.HllInv[L + j] = i01; d.HllInv[2 * L + j] = i02; d.HllInv[3 * L + j] = i11; d.HllInv[4 * L + j] = i12; d.HllInv[5 * L + j] = i22; }
    const double db0 = i00 * b0 + i01 * b1 + i02 * b2, db1 = i01 * b0 + i11 * b1 + i12 * b2, db2 = i02 * b0 + i12 * b1 + i22 * b2;
    for (int k = beg + sub; k < end; k += lanes) {
        if (d.e_hidx[k] < 0) continue;
        double hp[10], yv[12];
        load_rec10(d.Hpl + (size_t)k * EB, hp);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double g0 = hp[r * 3], g1 = hp[r * 3 + 1], g2 = hp[r * 3 + 2];
            yv[r * 3 + 0] = g0 * i00 + g1 * i01 + g2 * i02;
            yv[r * 3 + 1] = g0 * i01 + g1 * i11 + g2 * i12;
            yv[r * 3 + 2] = g0 * i02 + g1 * i12 + g2 * i22;
            yv[9 + r] = g0 * db0 + g1 * db1 + g2 * db2;
        }
        double2* y2 = reinterpret_cast<double2*>(d.Y + (size_t)k * EB);
#pragma unroll
        for (int q = 0; q < 6; ++q) y2[q] = make_double2(yv[2 * q], yv[2 * q + 1]);
    }
}

// One (landmark j, lane sub) slice of the linearisation (JAC) or of the robust chi2 evaluation (!JAC); the LANES lanes of a
// group call it together and take the landmark's edges in turn: e, J, Huber weighting, Hll / bl summed over the group, the
// per-edge Hpl and pose-side records. lam_fuse >= 0: the damping of the coming trial is already known, and the damping-
// dependent landmark terms are formed here from the sums every lane of the group holds (the persistent kernel saves its
// lm_prep phase and grid barrier that way). Returns the lane's share of the robust chi2.
template <bool JAC, int LANES, bool EXPLICIT = false>
__device__ __forceinline__ double pk_landmark(const Dev& d, const Cam& cam, const double* xp, const double* xl, int j, int sub, double lam_fuse) {
    static_assert(LANES == 1 || LANES == LPL, "group_sum sums over LPL lanes");
    double chi = 0, h00 = 0, h01 = 0, h02 = 0, h11 = 0, h12 = 0, h22 = 0, b0 = 0, b1 = 0, b2 = 0;
    int beg = 0, end = 0;
    if (j < d.L) { beg = d.lm_ptr[j]; end = d.lm_ptr[j + 1]; }
    if (end > beg) {
        const double lw[3] = {xl[3 * j], xl[3 * j + 1], xl[3 * j + 2]};
        const double dsqr = cam.delta * cam.delta;
        for (int e = beg + sub; e < end; e += LANES) {
            const int p = d.e_pose[e];
            const double ps[3] = {xp[3 * p], xp[3 * p + 1], xp[3 * p + 2]};
            double er[2], A[6], B[6];
            edge_xyz<JAC, EXPLICIT>(cam, ps, lw, d.e_u[e], d.e_v[e], er, A, B);
            const double w00 = d.e_w00[e], w01 = d.e_w01[e], w11 = d.e_w11[e];
            const double we0 = w00 * er[0] + w01 * er[1], we1 = w01 * er[0] + w11 * er[1];
            const double c2 = er[0] * we0 + er[1] * we1;
            double rho1 = 1.0;
            if (c2 <= dsqr) chi += c2;
            else { const double sq = sqrt(c2); chi += 2 * sq * cam.delta - dsqr; rho1 = cam.delta / sq; }
            if (JAC) {
                const double W00 = rho1 * w00, W01 = rho1 * w01, W11 = rho1 * w11;
                const double r0 = -rho1 * we0, r1 = -rho1 * we1;
                double BtW[6], AtW[6];
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    BtW[r * 2] = B[r] * W00 + B[3 + r] * W01; BtW[r * 2 + 1] = B[r] * W01 + B[3 + r] * W11;
                    AtW[r * 2] = A[r] * W00 + A[3 + r] * W01; AtW[r * 2 + 1] = A[r] * W01 + A[3 + r] * W11;
                }
                h00 += BtW[0] * B[0] + BtW[1] * B[3]; h01 += BtW[0] * B[1] + BtW[1] * B[4]; h02 += BtW[0] * B[2] + BtW[1] * B[5];
                h11 += BtW[2] * B[1] + BtW[3] * B[4]; h12 += BtW[2] * B[2] + BtW[3] * B[5]; h22 += BtW[4] * B[2] + BtW[5] * B[5];
                b0 += B[0] * r0 + B[3] * r1; b1 += B[1] * r0 + B[4] * r1; b2 += B[2] * r0 + B[5] * r1;
                if (d.e_hidx[e] >= 0) {
                    double hv[10], pv[10];            // the two 96-byte records, written with 16-byte stores
#pragma unroll
                    for (int r = 0; r < 3; ++r)
#pragma unroll
                        for (int c = 0; c < 3; ++c) hv[r * 3 + c] = AtW[r * 2] * B[c] + AtW[r * 2 + 1] * B[3 + c];
                    hv[9] = 0.0;
                    pv[0] = AtW[0] * A[0] + AtW[1] * A[3]; pv[1] = AtW[0] * A[1] + AtW[1] * A[4];
                    pv[2] = AtW[0] * A[2] + AtW[1] * A[5]; pv[3] = AtW[2] * A[1] + AtW[3] * A[4];
                    pv[4] = AtW[2] * A[2] + AtW[3] * A[5]; pv[5] = AtW[4] * A[2] + AtW[5] * A[5];
                    pv[6] = A[0] * r0 + A[3] * r1; pv[7] = A[1] * r0 + A[4] * r1; pv[8] = A[2] * r0 + A[5] * r1; pv[9] = 0.0;
                    double2* h2 = reinterpret_cast<double2*>(d.Hpl + (size_t)e * EB);
                    double2* p2 = reinterpret_cast<double2*>(d.PH + (size_t)e * EB);
#pragma unroll
                    for (int q = 0; q < 5; ++q) { h2[q] = make_double2(hv[2 * q], hv[2 * q + 1]); p2[q] = make_double2(pv[2 * q], pv[2 * q + 1]); }
                }
            }
        }
    }
    if (JAC) {
        if (LANES > 1) {
            h00 = group_sum(h00); h01 = group_sum(h01); h02 = group_sum(h02); h11 = group_sum(h11); h12 = group_sum(h12); h22 = group_sum(h22);
            b0 = group_sum(b0); b1 = group_sum(b1); b2 = group_sum(b2);
        }
        if (sub == 0 && end > beg) {
            const size_t L = d.L;
            d.Hll[j] = h00; d.Hll[L + j] = h01; d.Hll[2 * L + j] = h02; d.Hll[3 * L + j] = h11; d.Hll[4 * L + j] = h12; d.Hll[5 * L + j] = h22;
            d.bl[j] = b0; d.bl[L + j] = b1; d.bl[2 * L + j] = b2;
        }
        if (lam_fuse >= 0.0 && end > beg) lm_damp(d, j, beg, end, sub, LANES, lam_fuse, h00, h01, h02, h11, h12, h22, b0, b1, b2);
    }
    return chi;
}

// PreEdgeSE2 (EdgeSE2XYZ.h:68-99) for one odometry edge: e = [Ri^T (rj-ri) - m_xy ; thj - thi - m_th], no robust kernel.
// JAC: the blocks A_ii, A_ij, A_jj and b_i, b_j. Returns the edge's chi2.
template <bool JAC>
__device__ __forceinline__ double pk_odo(const Dev& d, const double* xp, int o) {
    const size_t O = d.O;
    const int pi = d.o_i[o], pj = d.o_j[o];
    double s, c;
    sincos(xp[3 * pi + 2], &s, &c);
    const double dx = xp[3 * pj] - xp[3 * pi], dy = xp[3 * pj + 1] - xp[3 * pi + 1];
    const double e0 = c * dx + s * dy - d.o_m[o], e1 = -s * dx + c * dy - d.o_m[O + o];
    const double e2 = xp[3 * pj + 2] - xp[3 * pi + 2] - d.o_m[2 * O + o];
    const double w0 = d.o_w[o], w1 = d.o_w[O + o], w2 = d.o_w[2 * O + o], w3 = d.o_w[3 * O + o], w4 = d.o_w[4 * O + o], w5 = d.o_w[5 * O + o];
    const double W[9] = {w0, w1, w2, w1, w3, w4, w2, w4, w5};
    const double we[3] = {W[0] * e0 + W[1] * e1 + W[2] * e2, W[3] * e0 + W[4] * e1 + W[5] * e2, W[6] * e0 + W[7] * e1 + W[8] * e2};
    if (JAC) {
        const double rx = -dy, ry = dx;
        const double Ai[9] = {-c, -s, -(c * rx + s * ry), s, -c, -(-s * rx + c * ry), 0, 0, -1};
        const double Aj[9] = {c, s, 0, -s, c, 0, 0, 0, 1};
        double AiW[9], AjW[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                AiW[r * 3 + k] = Ai[r] * W[k] + Ai[3 + r] * W[3 + k] + Ai[6 + r] * W[6 + k];
                AjW[r * 3 + k] = Aj[r] * W[k] + Aj[3 + r] * W[3 + k] + Aj[6 + r] * W[6 + k];
            }
        const int u6[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            const int r = u6[q][0], cc = u6[q][1];
            d.oAii[q * O + o] = AiW[r * 3] * Ai[cc] + AiW[r * 3 + 1] * Ai[3 + cc] + AiW[r * 3 + 2] * Ai[6 + cc];
            d.oAjj[q * O + o] = AjW[r * 3] * Aj[cc] + AjW[r * 3 + 1] * Aj[3 + cc] + AjW[r * 3 + 2] * Aj[6 + cc];
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) d.oAij[(r * 3 + cc) * O + o] = AiW[r * 3] * Aj[cc] + AiW[r * 3 + 1] * Aj[3 + cc] + AiW[r * 3 + 2] * Aj[6 + cc];
            d.obi[r * O + o] = -(Ai[r] * we[0] + Ai[3 + r] * we[1] + Ai[6 + r] * we[2]);
            d.obj[r * O + o] = -(Aj[r] * we[0] + Aj[3 + r] * we[1] + Aj[6 + r] * we[2]);
        }
    }
    return e0 * we[0] + e1 * we[1] + e2 * we[2];
}

// ph[0..8] += the pose-side terms (Hpp 6 unique, bp 3) of pose a's odometry edges k0, k0+stride, ... of its list
__device__ __forceinline__ void pose_odo_gather(const Dev& d, int a, int k0, int stride, double* ph) {
    const size_t O = d.O;
    for (int k = d.pose_odo_ptr[a] + k0; k < d.pose_odo_ptr[a + 1]; k += stride) {
        const int code = d.pose_odo[k], o = code >> 1;
        const double* H = (code & 1) ? d.oAjj : d.oAii;
        const double* b = (code & 1) ? d.obj : d.obi;
#pragma unroll
        for (int q = 0; q < 6; ++q) ph[q] += H[q * O + o];
#pragma unroll
        for (int q = 0; q < 3; ++q) ph[6 + q] += b[q * O + o];
    }
}

// pose a: Hpp diagonal block (6 unique) + bp from its edges (list in `edges`, shared or global) and odometry edges, by the
// whole CTA (any size). Summation order: thread-strided partials, warp xor-tree, then the per-warp sums in warp order.
__device__ void pk_pose_item(const Dev& d, int a, const int* edges, int ne, double* sh9 /*[warps][9]*/) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double acc[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) acc[q] = 0;
    for (int k = threadIdx.x; k < ne; k += blockDim.x) {
        double rec[10];
        load_rec10(d.PH + (size_t)edges[k] * EB, rec);
#pragma unroll
        for (int q = 0; q < 9; ++q) acc[q] += rec[q];
    }
    pose_odo_gather(d, a, threadIdx.x, blockDim.x, acc);
#pragma unroll
    for (int q = 0; q < 9; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int q = 0; q < 9; ++q) sh9[wid * 9 + q] = acc[q];
    __syncthreads();
    if (threadIdx.x < 9) {
        double v = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += sh9[w * 9 + threadIdx.x];
        if (threadIdx.x < 6) d.Hpp[threadIdx.x * (size_t)d.nf + a] = v;
        else d.bp[3 * a + threadIdx.x - 6] = v;
    }
}

// Gathers of one 3x3 block (a >= b) of the reduced system S_ab = [a==b](Hpp_aa + lambda I) + sum(odo blocks) - sum Y_e1 Hpl_e2^T,
// bs_a = bp_a - sum_e g_e, into acc[0..8] (S) and acc[9..11] (bs); each loop takes the items k0, k0+stride, ... of its list.
// pairs: pair k is the edges (e1[k ps], e2[k ps])
__device__ __forceinline__ void schur_pairs(const Dev& d, const int* e1, const int* e2, int ps, int np, int k0, int stride, double* acc) {
    for (int k = k0; k < np; k += stride) {
        double y[10], h[10];
        load_rec10(d.Y + (size_t)e1[k * ps] * EB, y); load_rec10(d.Hpl + (size_t)e2[k * ps] * EB, h);
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[r * 3 + c] -= y[r * 3] * h[c * 3] + y[r * 3 + 1] * h[c * 3 + 1] + y[r * 3 + 2] * h[c * 3 + 2];
    }
}
// odometry blocks A_ij (or A_ij^T) of block blk
__device__ __forceinline__ void schur_odo(const Dev& d, int blk, int k0, int stride, double* acc) {
    const size_t O = d.O;
    for (int k = d.blk_odo_ptr[blk] + k0; k < d.blk_odo_ptr[blk + 1]; k += stride) {
        const int code = d.blk_odo[k], o = code >> 1;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[r * 3 + c] += (code & 1) ? d.oAij[(c * 3 + r) * O + o] : d.oAij[(r * 3 + c) * O + o];
    }
}
// diagonal block: one sweep over the pose's edges for the g terms and, unless ph is null, the pose-side sums ph[0..8] (Hpp, bp)
__device__ __forceinline__ void schur_pose_sweep(const Dev& d, const int* edges, int ne, int k0, int stride, double* acc, double* ph) {
    for (int k = k0; k < ne; k += stride) {
        const double2* yr2 = reinterpret_cast<const double2*>(d.Y + (size_t)edges[k] * EB);
        const double2 g01 = yr2[4], g2 = yr2[5];        // doubles 8..11 of the record: Y[8], g[0], g[1], g[2]
        acc[9] -= g01.y; acc[10] -= g2.x; acc[11] -= g2.y;
        if (ph) {
            double rec[10];
            load_rec10(d.PH + (size_t)edges[k] * EB, rec);
#pragma unroll
            for (int q = 0; q < 9; ++q) ph[q] += rec[q];
        }
    }
}

// pose t's trial point x (+) dx: additive, angle re-normalised; a fixed pose is copied
__device__ __forceinline__ void pose_oplus(const Dev& d, int t, const double* xp, double* xpt) {
    const int a = d.hidx[t];
    if (a >= 0) {
        xpt[3 * t] = xp[3 * t] + d.dxp[3 * a]; xpt[3 * t + 1] = xp[3 * t + 1] + d.dxp[3 * a + 1];
        xpt[3 * t + 2] = normalize_theta(xp[3 * t + 2] + d.dxp[3 * a + 2]);
    } else {
        xpt[3 * t] = xp[3 * t]; xpt[3 * t + 1] = xp[3 * t + 1]; xpt[3 * t + 2] = xp[3 * t + 2];
    }
}
// computeScale term dx_a^T (lambda dx_a + bp_a) of free pose a
__device__ __forceinline__ double pose_scale(const Dev& d, int a, double lam) {
    const double p0 = d.dxp[3 * a], p1 = d.dxp[3 * a + 1], p2 = d.dxp[3 * a + 2];
    return p0 * (lam * p0 + d.bp[3 * a]) + p1 * (lam * p1 + d.bp[3 * a + 1]) + p2 * (lam * p2 + d.bp[3 * a + 2]);
}

// =================================================================================================
// Multi-launch kernels: one kernel per phase, the phase functions above with one thread per landmark / edge / item.

// linearise (JAC) or evaluate robust chi2 only (!JAC) at x[xi].  blocks [0,nb_lm): landmarks;
// blocks [nb_lm, nb_lm+nb_odo): PreEdgeSE2 edges.  part_chi[block] = partial activeRobustChi2.
template <bool JAC>
__global__ void __launch_bounds__(LM_THREADS) ba_linearize(Dev d, Cam cam, int use_trial) {
    __shared__ double sh[32];
    const int xi = use_trial ? (d.st->cur ^ 1) : d.st->cur;
    const double* __restrict__ xp = d.xp[xi];
    const double* __restrict__ xl = d.xl[xi];
    double chi = 0.0;
    if ((int)blockIdx.x < d.nb_lm) {
        chi = pk_landmark<JAC, 1>(d, cam, xp, xl, blockIdx.x * LM_THREADS + threadIdx.x, 0, -1.0);
    } else {
        const int o = (blockIdx.x - d.nb_lm) * LM_THREADS + threadIdx.x;
        if (o < d.O) chi = pk_odo<JAC>(d, xp, o);
    }
    const double tot = block_sum(chi, sh);
    if (threadIdx.x == 0) d.part_chi[blockIdx.x] = tot;
}

// one CTA (POSE_THREADS threads) per free pose: Hpp diagonal block (6 unique) and bp from its edges (+ its odometry edges)
constexpr int POSE_THREADS = 256;
__global__ void __launch_bounds__(POSE_THREADS) ba_pose_reduce(Dev d) {
    __shared__ double sh[(POSE_THREADS / 32) * 9];
    const int a = blockIdx.x;
    pk_pose_item(d, a, d.pose_edges + d.pose_ptr[a], d.pose_ptr[a + 1] - d.pose_ptr[a], sh);
}

// start of an LM iteration: currentChi from the linearisation partials; lambda init at iteration 0
// (lm_lambda_init over the max |diag H| of all free vertices).
// In sharded mode the host has all-reduced scal[0] (chi) and scal[1] (max diag) before `finish` runs.
__global__ void __launch_bounds__(256) ba_iter_begin(Dev d, int iter, int phase /*0: local partials -> scal, 1: consume scal*/, int itg /*g2o iteration number: lambda is initialised at 0 only*/) {
    __shared__ double sh[32];
    if (phase == 0) {
        double chi = 0;
        for (int b = threadIdx.x; b < d.nb_lm + d.nb_odo; b += blockDim.x) chi += d.part_chi[b];
        chi = block_sum(chi, sh);
        double m = 0;
        if (itg == 0) {
            for (int j = threadIdx.x; j < d.L; j += blockDim.x)
                if (d.lm_ptr[j + 1] > d.lm_ptr[j]) m = fmax(m, diag_absmax(d.Hll, d.L, j));
            // pose diagonal is only final after the cross-rank sum; in sharded mode it is handled by the host
            if (d.world == 1)
                for (int a = threadIdx.x; a < d.nf; a += blockDim.x) m = fmax(m, diag_absmax(d.Hpp, d.nf, a));
            m = cta_max(m, sh);
        }
        if (threadIdx.x == 0) { d.scal[0] = chi; d.scal[1] = m; }
    }
    if (phase == 1 || d.world == 1) {
        __syncthreads();
        if (threadIdx.x == 0) {
            LMState& s = *d.st;
            s.chi_cur = d.scal[0]; s.chi_before = s.chi_cur;
            if (itg == 0) { s.max_diag = d.scal[1]; lm_lambda_init(s.max_diag, s.lambda, s.ni); }
            s.trials = 0; s.accepted = 0; s.terminate = 0; s.retry = 0; s.iter = iter; s.rho = 0;
        }
    }
}

// sharded runs, iteration 0: out = max(out, max |diagonal| of the rank-summed pose blocks hpp [6][nf])
__global__ void __launch_bounds__(256) ba_pose_diag_max(const double* hpp, int nf, double* out) {
    __shared__ double sh[8];
    double m = 0;
    for (int a = threadIdx.x; a < nf; a += blockDim.x) m = fmax(m, diag_absmax(hpp, nf, a));
    m = cta_max(m, sh);
    if (threadIdx.x == 0) *out = fmax(*out, m);
}

// per landmark: (Hll + lambda I)^-1, Y_e = Hpl_e Hll^-1, g_e = Hpl_e (Hll^-1 bl)
__global__ void __launch_bounds__(LM_THREADS) ba_lm_prep(Dev d) {
    const int j = blockIdx.x * LM_THREADS + threadIdx.x;
    if (j >= d.L) return;
    const int beg = d.lm_ptr[j], end = d.lm_ptr[j + 1];
    if (end <= beg) return;
    const size_t L = d.L;
    lm_damp(d, j, beg, end, 0, 1, d.st->lambda, d.Hll[j], d.Hll[L + j], d.Hll[2 * L + j], d.Hll[3 * L + j], d.Hll[4 * L + j],
            d.Hll[5 * L + j], d.bl[j], d.bl[L + j], d.bl[2 * L + j]);
}

// one CTA (SCHUR_THREADS threads) per stored 3x3 block (a >= b) of the reduced pose Hessian; a diagonal block adds Hpp_aa
// from ba_pose_reduce (and lambda on rank 0 only: the damping is added once across shards)
constexpr int SCHUR_THREADS = 128;
__global__ void __launch_bounds__(SCHUR_THREADS) ba_schur(Dev d) {
    __shared__ double sh[SCHUR_THREADS / 32][12];
    const int blk = blockIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int a = d.blk_a[blk], b = d.blk_b[blk];
    double acc[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) acc[q] = 0;
    const int p0 = d.blk_pair_ptr[blk];
    schur_pairs(d, d.pair_e1 + p0, d.pair_e2 + p0, 1, d.blk_pair_ptr[blk + 1] - p0, threadIdx.x, SCHUR_THREADS, acc);
    schur_odo(d, blk, threadIdx.x, SCHUR_THREADS, acc);
    if (a == b) schur_pose_sweep(d, d.pose_edges + d.pose_ptr[a], d.pose_ptr[a + 1] - d.pose_ptr[a], threadIdx.x, SCHUR_THREADS, acc, nullptr);
#pragma unroll
    for (int q = 0; q < 12; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    if (lane == 0)
#pragma unroll
        for (int q = 0; q < 12; ++q) sh[wid][q] = acc[q];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < 12; ++q) { double v = 0; for (int w = 0; w < SCHUR_THREADS / 32; ++w) v += sh[w][q]; acc[q] = v; }
        const size_t nf = d.nf;
        if (a == b) {
            const double lam = (d.rank == 0) ? d.st->lambda : 0.0;   // damping is added once across shards
            const double H[9] = {d.Hpp[a], d.Hpp[nf + a], d.Hpp[2 * nf + a], d.Hpp[nf + a], d.Hpp[3 * nf + a], d.Hpp[4 * nf + a],
                                 d.Hpp[2 * nf + a], d.Hpp[4 * nf + a], d.Hpp[5 * nf + a]};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    if (c <= r || !d.sbw) d.S[sidx(d, 3 * a + r, 3 * b + c)] = acc[r * 3 + c] + H[r * 3 + c] + (r == c ? lam : 0.0);
                d.bs[3 * a + r] = d.bp[3 * a + r] + acc[9 + r];
            }
        } else {
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) d.S[sidx(d, 3 * a + r, 3 * b + c)] = acc[r * 3 + c];
        }
    }
}

// Reduced solve, one CTA: block LDL^T with 3x3 pivot blocks (one pose per block) restricted to the envelope of S.
//   S = L D L^T, D block diagonal, L unit block lower. Per block step k: W = D_k^-1 (closed-form symmetric inverse; the
//   leading principal minors double as the positive-definiteness test == CHOLMOD's "not PD"), every trailing entry
//   A[i][j] -= a_i . (W a_j) with a_i = A[i][k..k+2] left UNSCALED in place, the right-hand side rides along as an
//   extra column. One block barrier per pose (n/3 barriers instead of n), a short FP64 dependency chain per step
//   (dependent DFMAs, one 1/x, shared-memory loads and one barrier).
// Back substitution: x_k = W_k (u_k - sum_{i>k} a_i^T x_i), warp 0 only, warp-synchronous.
// SMEM=true indexes the dynamic shared array directly (LDS, no generic-address conversion in the loops);
// SMEM=false works in place in global memory (reduced systems too large for one CTA's shared memory).
#ifdef SE2_SOLVE_STAMPS
__device__ long long g_stamps[128];  // tools/solve_bench.cu: clock64 stamps of thread 0 of CTAs 0 / 1 (plain stores, no read-modify-write)
#define STAMP(i) do { if (threadIdx.x == 0) g_stamps[(blockIdx.x & 1) * 64 + (i)] = clock64(); } while (0)
#else
#define STAMP(i) do { } while (0)
#endif
#if defined(SE2_SOLVE_STAMPS) && SE2_SOLVE_STAMPS >= 2
// per-step stamps of one steady-state step, written by ALL lanes of a warp to one shared word (a thread-0-only stamp makes
// thread 0 diverge from its warp and distorts what it measures)
__device__ long long g_wstamps[16 * 16];
#define WSTAMP_DECL __shared__ long long s_wst[16 * 16];
#define WSTAMP(kbv, i) do { if ((kbv) == 10) s_wst[(threadIdx.x >> 5) * 16 + (i)] = clock64(); } while (0)
#define WSTAMP_DUMP do { __syncthreads(); if (threadIdx.x < 256) g_wstamps[threadIdx.x] = s_wst[threadIdx.x]; } while (0)
#else
#define WSTAMP_DECL
#define WSTAMP(kbv, i) do { } while (0)
#define WSTAMP_DUMP do { } while (0)
#endif

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier helpers: stage the reduced system into shared memory
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
// the same address as an opaque register value: nvcc otherwise RE-MATERIALISES the window base at every use inside the solve's
// loops (S2UR SR_CgaCtaId + ULEA in front of the LDS of every row pass, on the critical path of every pivot step)
__device__ __forceinline__ unsigned smem_u32_pinned(const void* p) { unsigned a = smem_u32(p); asm volatile("mov.b32 %0, %0;" : "+r"(a)); return a; }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    asm volatile("fence.proxy.async;" ::: "memory");   // order earlier generic-proxy accesses before the async-proxy copy
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// explicit 32-bit shared-window loads / stores: the address register is derived ONCE from the dynamic shared array, so the
// hot loops contain no generic->shared conversions (nvcc otherwise re-derives the window base from SR_CgaCtaId, an
// S2UR in front of many LDS, which dominated the per-pivot latency of the first versions of this solve)
struct SmemIO {
    static __device__ __forceinline__ double ld(unsigned a) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a)); return v; }
    static __device__ __forceinline__ void st(unsigned a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
    static __device__ __forceinline__ int ldi(unsigned a) { int v; asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
    static __device__ __forceinline__ void sti(unsigned a, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
    // 16-byte / 8-byte pairs (a must be aligned accordingly): one shared-memory instruction instead of two
    static __device__ __forceinline__ void ld2(unsigned a, double& x, double& y) { asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x), "=d"(y) : "r"(a)); }
    static __device__ __forceinline__ void st2(unsigned a, double x, double y) { asm volatile("st.shared.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(x), "d"(y) : "memory"); }
    static __device__ __forceinline__ void ldi2(unsigned a, int& x, int& y) { asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(x), "=r"(y) : "r"(a)); }
    static __device__ __forceinline__ void sti2(unsigned a, int x, int y) { asm volatile("st.shared.v2.s32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory"); }
};
struct GmemIO {   // same interface on byte offsets from a global base (reduced systems that do not fit one CTA's shared memory)
    static __device__ __forceinline__ double ld(unsigned long long a) { return *reinterpret_cast<const volatile double*>(a); }
    static __device__ __forceinline__ void st(unsigned long long a, double v) { *reinterpret_cast<volatile double*>(a) = v; }
    static __device__ __forceinline__ int ldi(unsigned long long a) { return *reinterpret_cast<const volatile int*>(a); }
    static __device__ __forceinline__ void sti(unsigned long long a, int v) { *reinterpret_cast<volatile int*>(a) = v; }
    static __device__ __forceinline__ void ld2(unsigned long long a, double& x, double& y) { x = ld(a); y = ld(a + 8); }
    static __device__ __forceinline__ void st2(unsigned long long a, double x, double y) { st(a, x); st(a + 8, y); }
    static __device__ __forceinline__ void ldi2(unsigned long long a, int& x, int& y) { x = ldi(a); y = ldi(a + 4); }
    static __device__ __forceinline__ void sti2(unsigned long long a, int x, int y) { sti(a, x); sti(a + 4, y); }
};

// Block LDL^T of the reduced system (see "Reduced solve, one CTA" above for the algorithm).
//   ADDR = unsigned (shared window) or unsigned long long (global); aA, aY, aW, aC, aT are the byte addresses of
//   A [n*n], y [n] (= row n of A when the two are adjacent), W records [8 per pose, 16-byte aligned inside a 9-per-pose area],
//   cmax (int) [n], scratch {3 unused, ok (int), 2 x 3 back-substitution exchange slots}.
// Slices of the block LDL^T for the two-sided ("twisted") solve; the defaults reproduce the plain full solve.
struct LdltOpt {
    int ld = 0;                 // leading dimension of A in elements (0: n)
    int kb0 = 0, kb1 = -1;      // pivot blocks [kb0, kb1) are eliminated by this call (-1: all)
    bool init = true;           // load y from bs (when given) and reset the positive-definiteness flag
    bool backsolve = true;      // run the back substitution and write the outputs
    int npiv = -1;              // back substitution: blocks >= npiv take their solution from xinj (-1: all blocks are pivots)
    const double* xinj = nullptr;
    // back substitution hook of the twisted solve: once blocks >= pub_kb are solved their owners write x mirrored to pub and count in
    double* pub = nullptr; unsigned* pub_cnt = nullptr; int pub_kb = 0;
    unsigned* okword = nullptr; unsigned okval = 0;     // thread 0 writes okval | ok right after the factorisation
};
constexpr int TW_XM = 3 * TW_MAX_W * (3 * TW_MAX_W + 1) + 16;
constexpr int TW_BUF_DOUBLES = TW_XM + 3 * TW_MAX_W + 16;

template <class IO, class ADDR>
__device__ void ldlt_block_solve_impl(ADDR aA, ADDR aY, ADDR aW, ADDR aC, ADDR aT, int n, const double* bs, double* dxp, LMState* st, const LdltOpt opt = LdltOpt()) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    const ADDR aOK = aT + 24;
    WSTAMP_DECL
    const int ld = opt.ld > 0 ? opt.ld : n;      // leading dimension of A
#define A_(r, c) (aA + (ADDR)(((r) * ld + (c)) * 8))
#define Y_(i) (aY + (ADDR)((i) * 8))
    // per-block record, 64 bytes at a 16-byte aligned address: W = D_kb^-1 packed [w00 w01 | w02 w11 | w12 w22] and {pd, m} (ints):
    // pd = pivot block positive definite, m = trailing rows/cols of the block's envelope. One 8-byte + three 16-byte shared loads
    // per warp and step: the step is bound by the shared-memory instruction queue (16 warps re-reading the same words), not by
    // arithmetic.
    const ADDR aWr = (aW + (ADDR)15) & ~(ADDR)15;
#define R_(kb) (aWr + (ADDR)((kb) * 64))
    // the right-hand side is row n of the matrix: y_i -= a_i . (W u_k) = u_k . (W a_i) is the update of entry (n, i) with
    // a_n = u_k = y[k..k+2], the same formula as every other trailing entry (no separate code path, no published W u)
    auto rowaddr = [&](int i) -> ADDR { return i == n ? aY : aA + (ADDR)i * (ADDR)(ld * 8); };
    STAMP(0);
    if (opt.init) {
        if (tid == 0) IO::sti(aOK, 1);
        if (bs) for (int i = tid; i < n; i += nt) IO::st(Y_(i), bs[i]);
    }
    __syncthreads();
    const int nb = n / 3;                                           // blocks of the matrix (rows below the eliminated part are updated too)
    const int kb0 = opt.kb0, kb1 = opt.kb1 < 0 ? nb : opt.kb1;      // pivot blocks eliminated by this call
    STAMP(1);
    // The pivot-block inverse is the serial chain of the factorisation: warp 0 ("pivot warp") updates the NEXT pivot block and
    // its right-hand-side entries first, inverts it and publishes the record of block k+1 before the step's barrier, while the
    // other warps update the rest of the trailing envelope. After the barrier everybody just reads the record.
    auto invert_and_publish = [&](int kb, int r) {     // pivot block at rows/cols r..r+2 (already final)
        const double a = IO::ld(A_(r, r)), b = IO::ld(A_(r + 1, r)), c = IO::ld(A_(r + 2, r));
        const double e = IO::ld(A_(r + 1, r + 1)), f = IO::ld(A_(r + 2, r + 1)), i2 = IO::ld(A_(r + 2, r + 2));
        const int mnext = IO::ldi(aC + (ADDR)((r + 2) * 4)) - (r + 2);
        WSTAMP(kb - 1, 4);
        const Sym3Inv w = sym3_inverse(a, b, c, e, f, i2);
        WSTAMP(kb - 1, 5);
        if (lane == 0) {
            const ADDR rec = R_(kb);
            IO::st2(rec, w.i00, w.i01); IO::st2(rec + 16, w.i02, w.i11); IO::st2(rec + 32, w.i12, w.i22); IO::sti2(rec + 48, w.pd ? 1 : 0, mnext);
            if (!w.pd) IO::sti(aOK, 0);
        }
        WSTAMP(kb - 1, 6);
    };
    const bool go = IO::ldi(aOK) != 0;                               // a continuation slice of a system already found indefinite does nothing
    if (wid == 0 && kb0 < kb1 && go) invert_and_publish(kb0, 3 * kb0);
    __syncthreads();
    STAMP(2);
    for (int kb = go ? kb0 : kb1; kb < kb1; ++kb) {
        WSTAMP(kb, 0);
        int pdk, m;                                              // m: trailing rows/cols k+3 .. k+2+m
        IO::ldi2(R_(kb) + 48, pdk, m);
        if (!pdk) break;                                         // uniform: published before the barrier that precedes this read
        const int k = 3 * kb;
        WSTAMP(kb, 1);
        if (wid == 0) {
            double w00, w01, w02, w11, w12, w22;
            IO::ld2(R_(kb), w00, w01); IO::ld2(R_(kb) + 16, w02, w11); IO::ld2(R_(kb) + 32, w12, w22);
            // next pivot block: rows k+3..k+5 (ii = 0..2), cols jj <= ii (lanes 0..5), and the right-hand side of those columns
            // (row n, lanes 6..8)
            if (kb + 1 < nb && lane < 9) {
                const int q = lane;                 // 0..5: (ii,jj) = (0,0)(1,0)(1,1)(2,0)(2,1)(2,2); 6..8: (n, q-6)
                const bool rhs = q >= 6;
                const int ii = q < 1 ? 0 : (q < 3 ? 1 : 2);
                const int jj = q < 1 ? 0 : (q < 3 ? q - 1 : (q < 6 ? q - 3 : q - 6));
                if ((rhs ? jj : ii) < m) {          // rows / columns beyond the envelope of this block column are structurally untouched
                    const int j = k + 3 + jj;
                    const ADDR ra = rowaddr(rhs ? n : k + 3 + ii), dst = ra + (ADDR)(j * 8), rb = A_(j, k);
                    const double a0 = IO::ld(ra + (ADDR)(k * 8)), a1 = IO::ld(ra + (ADDR)(k * 8 + 8)), a2 = IO::ld(ra + (ADDR)(k * 8 + 16));
                    const double b0 = IO::ld(rb), b1 = IO::ld(rb + 8), b2 = IO::ld(rb + 16);
                    const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                    IO::st(dst, IO::ld(dst) - (a0 * v0 + a1 * v1 + a2 * v2));
                }
            }
            WSTAMP(kb, 2);
            if (kb + 1 < kb1) {
                __syncwarp();                       // the 6 freshly updated values are in memory: re-read, invert, publish
                WSTAMP(kb, 3);
                invert_and_publish(kb + 1, k + 3);
            }
            WSTAMP(kb, 7);
        } else if (m > 63 || (wid & 3) != 0) {
            // rows ii >= 3 of the trailing envelope and the right-hand side (pseudo row ii == m, columns >= 3): lanes over the columns.
            // A narrow envelope has rows of <= 16 (8) columns: 2 (4) rows share one warp pass, which halves (quarters) the
            // shared-memory instructions of the step. Warps are dealt to the 4 SM sub-partitions by warp id mod 4: for a narrow
            // envelope the warps that share the pivot warp's sub-partition sit the step out, so the pivot chain never waits for an
            // issue slot.
            const bool quiet = m <= 63;
            const int rank = quiet ? wid - (wid >> 2) - 1 : wid - 1, nwk = quiet ? nw - ((nw + 3) >> 2) : nw - 1;
            const int lg = m <= 8 ? 3 : (m <= 16 ? 4 : 5), rpp = 32 >> lg, col = lane & ((1 << lg) - 1), sub = lane >> lg;
            const int nrows = m - 2;
            if (rank * rpp < nrows) {
                double w00, w01, w02, w11, w12, w22;
                IO::ld2(R_(kb), w00, w01); IO::ld2(R_(kb) + 16, w02, w11); IO::ld2(R_(kb) + 32, w12, w22);
                for (int s0 = rank * rpp; s0 < nrows; s0 += nwk * rpp) {
                    const int ii = 3 + s0 + sub;
                    if (ii > m) continue;
                    const bool rhs = ii == m;
                    const ADDR ra = rowaddr(rhs ? n : k + 3 + ii);
                    const int jlo = rhs ? 3 : 0, jhi = rhs ? m - 1 : ii;
                    const double a0 = IO::ld(ra + (ADDR)(k * 8)), a1 = IO::ld(ra + (ADDR)(k * 8 + 8)), a2 = IO::ld(ra + (ADDR)(k * 8 + 16));
                    for (int jj = col; jj <= jhi; jj += 1 << lg) {
                        if (jj < jlo) continue;
                        const int j = k + 3 + jj;
                        const ADDR dst = ra + (ADDR)(j * 8), rb = A_(j, k);
                        const double b0 = IO::ld(rb), b1 = IO::ld(rb + 8), b2 = IO::ld(rb + 16);
                        const double v0 = w00 * b0 + w01 * b1 + w02 * b2, v1 = w01 * b0 + w11 * b1 + w12 * b2, v2 = w02 * b0 + w12 * b1 + w22 * b2;
                        IO::st(dst, IO::ld(dst) - (a0 * v0 + a1 * v1 + a2 * v2));
                    }
                }
            }
            WSTAMP(kb, 7);
        }
        __syncthreads();
        WSTAMP(kb, 8);
    }
    __syncthreads();
    STAMP(3);
    WSTAMP_DUMP;
    const int ok = IO::ldi(aOK);
    if (!opt.backsolve) return;                                    // factorisation slice only (twisted solve: the driver continues)
    if (opt.okword && tid == 0) { *reinterpret_cast<volatile unsigned*>(opt.okword) = opt.okval | (unsigned)ok; __threadfence(); }
    const int npiv = opt.npiv < 0 ? nb : opt.npiv;                 // blocks >= npiv take their solution from opt.xinj
    if (ok) {
        if (n <= 160 && nt >= 160) {
            // Back substitution, axpy form on 5 warps: thread c < n owns the accumulator z_c = u_c - sum(a^T x) of column c in
            // a register. Per block step (descending) the three owners of block kb publish their finished accumulators,
            // one named barrier later every thread forms x_kb = W_kb z_kb redundantly and subtracts row block kb of the
            // factor times x_kb from its own column: no reduction tree, ~40 instructions per warp and step. (A single warp
            // issues one instruction every ~4 cycles, so the dot-product form below - ~200 instructions per step on one
            // warp - costs ~800 cycles per step whatever the latencies are.)
            if (tid < 160) {
                const int c = tid;
                double z = c < n ? IO::ld(Y_(c)) : 0.0;
                const int cm = c < n ? IO::ldi(aC + (ADDR)(c * 4)) : -1;
                for (int kb = nb - 1; kb >= 0; --kb) {
                    const int k = 3 * kb;
                    const ADDR xz = aT + (ADDR)(32 + 24 * (kb & 1));        // double-buffered exchange slots
                    if (c >= k && c < k + 3) IO::st(xz + (ADDR)((c - k) * 8), z);
                    const bool in = c < k && cm >= k + 2;                  // row block kb inside this column's envelope
                    const double a0 = in ? IO::ld(A_(k, c)) : 0.0, a1 = in ? IO::ld(A_(k + 1, c)) : 0.0, a2 = in ? IO::ld(A_(k + 2, c)) : 0.0;
                    double w00, w01, w02, w11, w12, w22;
                    IO::ld2(R_(kb), w00, w01); IO::ld2(R_(kb) + 16, w02, w11); IO::ld2(R_(kb) + 32, w12, w22);
                    asm volatile("bar.sync 1, 160;" ::: "memory");
                    const double z0 = IO::ld(xz), z1 = IO::ld(xz + 8), z2 = IO::ld(xz + 16);
                    double x0 = w00 * z0 + w01 * z1 + w02 * z2, x1 = w01 * z0 + w11 * z1 + w12 * z2, x2 = w02 * z0 + w12 * z1 + w22 * z2;
                    if (kb >= npiv) { x0 = opt.xinj[3 * (kb - npiv)]; x1 = opt.xinj[3 * (kb - npiv) + 1]; x2 = opt.xinj[3 * (kb - npiv) + 2]; }
                    z -= a0 * x0 + a1 * x1 + a2 * x2;
                    z = (c == k) ? x0 : (c == k + 1) ? x1 : (c == k + 2) ? x2 : z;
                    if (opt.pub && kb == opt.pub_kb && c >= k && c < n) { opt.pub[n - 1 - c] = z; __threadfence(); atomicAdd(opt.pub_cnt, 1u); }
                }
                if (c < n) IO::st(Y_(c), z);
            }
        } else if (wid == 0) {
            // lanes = 3 columns x 8 row slots; each 8-lane group sums its column's dot product with an xor tree
            const int c = lane >> 3, rs = lane & 7;
            for (int kb = nb - 1; kb >= 0; --kb) {
                const int k = 3 * kb, m = IO::ldi(aC + (ADDR)((k + 2) * 4)) - (k + 2);
                double sdot = 0;
                if (c < 3)
                    for (int ii = rs; ii < m; ii += 8) sdot += IO::ld(A_(k + 3 + ii, k + c)) * IO::ld(Y_(k + 3 + ii));
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 4);
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 2);
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 1);
                const double rc = (c < 3) ? IO::ld(Y_(k + c)) - sdot : 0.0;
                const double r0 = __shfl_sync(0xffffffffu, rc, 0), r1 = __shfl_sync(0xffffffffu, rc, 8), r2 = __shfl_sync(0xffffffffu, rc, 16);
                if (lane < 3) {     // row `lane` of the symmetric W from its packed upper triangle [00 01 02 11 12 22]
                    const int q0 = lane, q1 = lane == 0 ? 1 : (lane == 1 ? 3 : 4), q2 = lane == 0 ? 2 : (lane == 1 ? 4 : 5);
                    IO::st(Y_(k + lane), IO::ld(R_(kb) + (ADDR)(q0 * 8)) * r0 + IO::ld(R_(kb) + (ADDR)(q1 * 8)) * r1 + IO::ld(R_(kb) + (ADDR)(q2 * 8)) * r2);
                }
                __syncwarp();
            }
        }
        __syncthreads();
        STAMP(4);
        if (dxp) for (int i = tid; i < n; i += nt) dxp[i] = IO::ld(Y_(i));
    } else {
        if (dxp) for (int i = tid; i < n; i += nt) dxp[i] = 0.0;
    }
    if (tid == 0 && st) st->solve_ok = ok;
    STAMP(5);
#undef A_
#undef Y_
#undef R_
}

template <bool SMEM>
__device__ void ldlt_block_solve(double* G, double* ywork, int n, const int* colmax_g, const double* bs, double* dxp, LMState* st) {
    if (SMEM) {
        extern __shared__ double sm[];
        // layout: A [n*n] | y [n] | W records [3n + 2] | cmax (int) [n] | scratch
        const unsigned sA = smem_u32_pinned(sm);
        const unsigned sY = sA + (unsigned)n * n * 8, sW = sY + (unsigned)n * 8, sC = sW + (unsigned)(3 * n + 2) * 8;
        const unsigned sT = (sC + (unsigned)n * 4 + 15u) & ~15u;
        ldlt_block_solve_impl<SmemIO, unsigned>(sA, sY, sW, sC, sT, n, bs, dxp, st);
    } else {
        // global layout: A = G; ywork holds y [n] | W [3n] | scratch [4]; the envelope stays where it is
        const unsigned long long gA = (unsigned long long)G, gY = (unsigned long long)ywork, gW = gY + (unsigned long long)n * 8;
        const unsigned long long gT = gW + (unsigned long long)(3 * n) * 8;
        ldlt_block_solve_impl<GmemIO, unsigned long long>(gA, gY, gW, (unsigned long long)colmax_g, gT, n, bs, dxp, st);
    }
}

// S (n*n doubles, rounded up to 16 B: the tail lands in y, which is initialised afterwards) and the envelope -> shared
// memory. One elected thread issues a single bulk copy; everybody waits on the mbarrier phase `parity`.
__device__ __forceinline__ void ldlt_stage(const Dev& d, const double* S, unsigned long long* bar, unsigned parity) {
    extern __shared__ double sm[];
    const int n = d.n;
    int* cmax = reinterpret_cast<int*>(sm + (size_t)n * n + n + 3 * (size_t)n + 2);
    const unsigned bytes = (unsigned)(((size_t)n * n * 8 + 15) & ~(size_t)15);
    if (bytes) {
        if (threadIdx.x == 0) bulk_g2s(sm, S, bytes, bar);
        for (int t = threadIdx.x; t < n; t += blockDim.x) cmax[t] = d.colmax[t];
        mbar_wait(bar, parity);
    }
    __syncthreads();
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// The CTAs that run one window in the persistent kernel ("team"): the cooperative grid (ba_persistent) or one thread-block
// cluster (ba_persistent_cluster). rank() / size() are the CTA's place among the window's CTAs and their number; sync() ends a
// phase. Phase functions read them through the type, as unsigned like blockIdx.x / gridDim.x, so that the grid instantiation
// compiles to the code the grid-only kernel had.
namespace cg = cooperative_groups;
struct GridTeam {
    static constexpr bool kExplicitFma = false;   // camera in parameter space: edge_xyz as written (see there)
    cg::grid_group g;
    __device__ __forceinline__ GridTeam() : g(cg::this_grid()) {}
    static __device__ __forceinline__ unsigned rank() { return blockIdx.x; }
    static __device__ __forceinline__ unsigned size() { return gridDim.x; }
    __device__ __forceinline__ void sync() { g.sync(); }
};
// Cluster barrier: barrier.cluster.arrive.release + wait.acquire, which sm_90a compiles to MEMBAR.ALL.GPU, UCGABAR_ARV,
// UCGABAR_WAIT and CCTL.IVALL - the L1 invalidation lets plain loads after it see what the other CTAs of the cluster stored
// before it. Cluster scope is enough: everything one phase hands to the next (part_*, S / bs, tw_buf / tw_flag, the LM state
// and the per-landmark and per-edge arrays) belongs to the window, and only the window's own CTAs read it.
struct ClusterTeam {
    static constexpr bool kExplicitFma = true;    // camera in shared memory: edge_xyz's contraction spelled out (see there)
    static __device__ __forceinline__ unsigned rank() { return cg::this_cluster().block_rank(); }
    static __device__ __forceinline__ unsigned size() { return cg::this_cluster().num_blocks(); }
    __device__ __forceinline__ void sync() { cg::this_cluster().sync(); }
};

// Two-sided solve of the reduced system on CTAs 0 and 1 of the persistent kernel (both resident: cooperative launch, or
// one cluster, whose CTAs the hardware co-schedules).
// The pivot chain - one dependent 3x3 inverse per pose block - is the critical path of the single-CTA solve; the envelope of a
// local window is a narrow band, so the blocks split into top [0, m0), separator [m0, m0 + w) and bottom [m0 + w, nb) with no
// top-bottom coupling. CTA 0 eliminates the top blocks of S[0 : 3(m0+w)) in place; CTA 1 eliminates the bottom blocks on the
// index-reversed copy A1[r'][c'] = S[n-1-c'][n-1-r'] (lower triangle -> lower triangle, same code); its separator update goes to
// CTA 0 through tw_buf, CTA 0 finishes the separator blocks, back-substitutes and hands the separator solution back as soon as it
// exists. Chain length max(m0, nb - m0 - w) + w instead of nb. `seq` counts the solves of this launch from 1.
template <class Team>
__device__ void ldlt_twisted_solve(const Dev& d, const double* S, const double* bs, unsigned long long* bar, unsigned parity, unsigned seq) {
    extern __shared__ double sm[];
    __shared__ double xs[3 * TW_MAX_W];
    const int n = d.n, nb = n / 3, m0 = d.tw_m0, w = d.tw_w, m1 = nb - m0 - w, w3 = 3 * w;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* T = d.tw_buf;
    if (Team::rank() == 0) {
        const int n0 = 3 * (m0 + w);
        // layout: A [n0 rows, leading dimension n] | y [n0] | W [3 n0] | pad [2] | cmax (int) [n0] | scratch
        double* y = sm + (size_t)n0 * n;
        int* cm = reinterpret_cast<int*>(y + 4 * (size_t)n0 + 2);
        const unsigned sA = smem_u32_pinned(sm), sY = sA + (unsigned)n0 * n * 8, sW = sY + (unsigned)n0 * 8, sC = sY + (unsigned)(4 * n0 + 2) * 8, sT = (sC + (unsigned)n0 * 4 + 15u) & ~15u;
        const unsigned bytes = (unsigned)(((size_t)n0 * n * 8 + 15) & ~(size_t)15);
        STAMP(50);
        if (tid == 0) bulk_g2s(sm, S, bytes, bar);
        for (int t = tid; t < n0; t += nt) cm[t] = min(d.colmax[t], n0 - 1);
        mbar_wait(bar, parity);
        __syncthreads();
        STAMP(51);
        LdltOpt o;
        o.ld = n; o.kb0 = 0; o.kb1 = m0; o.backsolve = false;
        ldlt_block_solve_impl<SmemIO, unsigned>(sA, sY, sW, sC, sT, n0, bs, nullptr, nullptr, o);
        STAMP(52);
        if (tid == 0) while (ld_acquire_u32(d.tw_flag) < seq) { }
        __syncthreads();
        STAMP(53);
        for (int q = tid; q < w3 * w3 + w3; q += nt) {
            if (q < w3 * w3) {
                const int i = q / w3, j = q - i * w3;
                if (j <= i) sm[(size_t)(3 * m0 + i) * n + 3 * m0 + j] += __ldcg(T + (w3 - 1 - j) * w3 + (w3 - 1 - i));
            } else {
                const int i = q - w3 * w3;
                y[3 * m0 + i] += __ldcg(T + w3 * w3 + (w3 - 1 - i));
            }
        }
        if (tid == 0 && __ldcg(T + w3 * w3 + w3) == 0.0) SmemIO::sti(sT + 24, 0);
        __syncthreads();
        STAMP(54);
        o.kb0 = m0; o.kb1 = m0 + w; o.init = false; o.backsolve = true;
        o.pub = T + TW_XM; o.pub_cnt = d.tw_flag + 1; o.pub_kb = m0; o.okword = d.tw_flag + 2; o.okval = seq << 1;
        ldlt_block_solve_impl<SmemIO, unsigned>(sA, sY, sW, sC, sT, n0, nullptr, d.dxp, d.st, o);
        if (tid == 0 && !SmemIO::ldi(sT + 24)) atomicAdd(d.tw_flag + 1, (unsigned)w3);      // not positive definite: nothing was published
        STAMP(55);
    } else {
        const int n1 = 3 * (m1 + w);
        // layout: A1 [n1 * n1] | y [n1] | W [3 n1] | pad [2] | cmax (int) [n1] | scratch
        double* y = sm + (size_t)n1 * n1;
        int* cm = reinterpret_cast<int*>(y + 4 * (size_t)n1 + 2);
        const unsigned sA = smem_u32_pinned(sm), sY = sA + (unsigned)n1 * n1 * 8, sW = sY + (unsigned)n1 * 8, sC = sY + (unsigned)(4 * n1 + 2) * 8, sT = (sC + (unsigned)n1 * 4 + 15u) & ~15u;
        STAMP(50);
#pragma unroll 4
        for (int q = tid; q < n1 * n1; q += nt) {
            const int c = q / n1, r = q - c * n1;              // r fastest: consecutive threads read consecutive (descending) columns of one row of S
            if (r >= c && r <= d.tw_cmax1[c]) sm[(size_t)r * n1 + c] = (c >= 3 * m1) ? 0.0 : S[(size_t)(n - 1 - c) * n + (n - 1 - r)];
        }
        for (int t = tid; t < n1; t += nt) { cm[t] = d.tw_cmax1[t]; y[t] = t < 3 * m1 ? bs[n - 1 - t] : 0.0; }
        __syncthreads();
        STAMP(51);
        LdltOpt o;
        o.ld = n1; o.kb0 = 0; o.kb1 = m1; o.backsolve = false;
        ldlt_block_solve_impl<SmemIO, unsigned>(sA, sY, sW, sC, sT, n1, nullptr, nullptr, nullptr, o);
        STAMP(52);
        for (int q = tid; q < w3 * w3 + w3; q += nt) {
            if (q < w3 * w3) {
                const int i = q / w3, j = q - i * w3;
                if (j <= i) T[q] = sm[(size_t)(3 * m1 + i) * n1 + 3 * m1 + j];
            } else {
                T[q] = y[3 * m1 + q - w3 * w3];
            }
        }
        if (tid == 0) T[w3 * w3 + w3] = SmemIO::ldi(sT + 24) ? 1.0 : 0.0;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            st_release_u32(d.tw_flag, seq);
            STAMP(53);
            while (ld_acquire_u32(d.tw_flag + 1) < seq * (unsigned)w3) { }
        }
        __syncthreads();
        const bool ok = (__ldcg(d.tw_flag + 2) & 1u) != 0;
        if (tid < w3) xs[tid] = __ldcg(T + TW_XM + tid);
        __syncthreads();
        STAMP(54);
        if (ok) {
            o.kb0 = m1; o.kb1 = m1; o.init = false; o.backsolve = true; o.npiv = m1; o.xinj = xs;
            ldlt_block_solve_impl<SmemIO, unsigned>(sA, sY, sW, sC, sT, n1, nullptr, nullptr, nullptr, o);
            __syncthreads();
            for (int c = tid; c < 3 * m1; c += nt) d.dxp[n - 1 - c] = y[c];
        } else {
            for (int c = tid; c < 3 * m1; c += nt) d.dxp[n - 1 - c] = 0.0;
        }
        STAMP(55);
    }
}

__global__ void __launch_bounds__(CHOL_THREADS) ba_chol_solve_smem(Dev d) {
    __shared__ __align__(8) unsigned long long bar;
    if (threadIdx.x == 0) mbar_init(&bar, 1);
    __syncthreads();
    ldlt_stage(d, d.S, &bar, 0);
    ldlt_block_solve<true>(nullptr, nullptr, d.n, nullptr, d.bs, d.dxp, d.st);
}

__global__ void __launch_bounds__(CHOL_THREADS) ba_chol_solve_gmem(Dev d, double* ywork) {
    ldlt_block_solve<false>(d.S, ywork, d.n, d.colmax, d.bs, d.dxp, d.st);
}

constexpr int MAX_PEERS = 8;

// back-substitution + oplus into the trial buffers + partial sums of computeScale(). The landmark part is the same arithmetic
// as pk_phase_backsub's with a different summation order (c = bl - sum there is (0 - sum) + bl); it is not shared because
// a shared helper makes ptxas spill more of ba_persistent.
__global__ void __launch_bounds__(LM_THREADS) ba_backsub_update(Dev d) {
    __shared__ double sh[32];
    const int t = blockIdx.x * LM_THREADS + threadIdx.x;
    const int cur = d.st->cur;
    const double lam = d.st->lambda;
    const double lam_pose = (d.rank == 0) ? lam : 0.0;
    double sc = 0.0;
    if (t < d.L) {
        const int j = t;
        const int beg = d.lm_ptr[j], end = d.lm_ptr[j + 1];
        const size_t L = d.L;
        double dl0 = 0, dl1 = 0, dl2 = 0;
        if (end > beg) {
            double c0 = d.bl[j], c1 = d.bl[L + j], c2 = d.bl[2 * L + j];
            for (int k = beg; k < end; ++k) {
                const int a = d.e_hidx[k];
                if (a < 0) continue;
                const double p0 = d.dxp[3 * a], p1 = d.dxp[3 * a + 1], p2 = d.dxp[3 * a + 2];
                c0 -= d.Hpl[(size_t)k * EB + (0)] * p0 + d.Hpl[(size_t)k * EB + (3)] * p1 + d.Hpl[(size_t)k * EB + (6)] * p2;
                c1 -= d.Hpl[(size_t)k * EB + (1)] * p0 + d.Hpl[(size_t)k * EB + (4)] * p1 + d.Hpl[(size_t)k * EB + (7)] * p2;
                c2 -= d.Hpl[(size_t)k * EB + (2)] * p0 + d.Hpl[(size_t)k * EB + (5)] * p1 + d.Hpl[(size_t)k * EB + (8)] * p2;
            }
            const double i00 = d.HllInv[j], i01 = d.HllInv[L + j], i02 = d.HllInv[2 * L + j], i11 = d.HllInv[3 * L + j], i12 = d.HllInv[4 * L + j], i22 = d.HllInv[5 * L + j];
            dl0 = i00 * c0 + i01 * c1 + i02 * c2; dl1 = i01 * c0 + i11 * c1 + i12 * c2; dl2 = i02 * c0 + i12 * c1 + i22 * c2;
            sc += dl0 * (lam * dl0 + d.bl[j]) + dl1 * (lam * dl1 + d.bl[L + j]) + dl2 * (lam * dl2 + d.bl[2 * L + j]);
        }
        const double* xl = d.xl[cur];
        double* xlt = d.xl[cur ^ 1];
        d.dxl[3 * j] = dl0; d.dxl[3 * j + 1] = dl1; d.dxl[3 * j + 2] = dl2;
        xlt[3 * j] = xl[3 * j] + dl0; xlt[3 * j + 1] = xl[3 * j + 1] + dl1; xlt[3 * j + 2] = xl[3 * j + 2] + dl2;
    }
    if (t < d.P) {
        pose_oplus(d, t, d.xp[cur], d.xp[cur ^ 1]);
        const int a = d.hidx[t];
        if (a >= 0) sc += pose_scale(d, a, lam_pose);
    }
    const double tot = block_sum(sc, sh);
    if (threadIdx.x == 0) d.part_scale[blockIdx.x] = tot;
}

// the LM decision of one trial (lm_gain_step) on the device.
// phase 0 sums the local partials into scal[0..1]; phase 1 (or single GPU) consumes them.
__global__ void __launch_bounds__(256) ba_decide(Dev d, int nb_scale, int phase, se2gpu_ba_iter_stats* stats_dev, int stop_local) {
    __shared__ double sh[32];
    if (phase == 0) {
        double chi = 0, sc = 0;
        for (int b = threadIdx.x; b < d.nb_lm + d.nb_odo; b += blockDim.x) chi += d.part_chi[b];
        for (int b = threadIdx.x; b < nb_scale; b += blockDim.x) sc += d.part_scale[b];
        chi = block_sum(chi, sh);
        sc = block_sum(sc, sh);
        // scal[2]: this rank's view of the abort flag; summed with the other two scalars, so every rank acts on the same value
        if (threadIdx.x == 0) { d.scal[0] = chi; d.scal[1] = sc; d.scal[2] = stop_local ? 1.0 : 0.0; }
    }
    if (phase == 1 || d.world == 1) {
        __syncthreads();
        if (threadIdx.x == 0) {
            LMState& s = *d.st;
            s.stop_all = d.scal[2] > 0.0 ? 1 : 0;
            double tempChi = d.scal[0], scale = d.scal[1], rho;
            if (lm_gain_step(tempChi, scale, s.solve_ok, s.chi_cur, s.lambda, s.ni, rho)) { s.cur ^= 1; s.accepted = 1; }
            s.chi_trial = tempChi; s.scale = scale; s.rho = rho;
            s.trials += 1;
            s.retry = (lm_retry(rho, s.trials) && !s.stop_all) ? 1 : 0;
            if (!s.retry) {
                const se2gpu_ba_iter_stats o = lm_iter_stats(s.chi_before, s.chi_cur, s.lambda, rho, s.trials, s.accepted);
                s.terminate = o.terminate;
                if (stats_dev) stats_dev[s.iter] = o;
            }
        }
    }
}

// =================================================================================================
// Persistent cooperative variant: the WHOLE optimize() call is one kernel launch. All CTAs are co-resident (one per
// SM, cooperative launch); phases are separated by grid-wide barriers instead of kernel boundaries, and the LM
// control (rho test, lambda schedule, accept/reject, termination) is evaluated redundantly and identically by every
// CTA from the same fixed-order partial sums, so no host round trip happens inside an optimize() call.
// Per-landmark work is spread over LPL lanes (edges strided over the lanes, xor-tree over the lane group).
constexpr int FALLBACK_CLOCK_KHZ = 1980000;   // H100 SXM maximum SM clock: cycle <-> time conversion if the device does not report one

struct PKArgs {
    int max_iters;
    int first_iter;           // iteration number of the first LM iteration of this call (g2o's solve(iteration): lambda is
                              // initialised at iteration 0 only; > 0 continues the lambda / nu schedule of the previous call)
    se2gpu_ba_iter_stats* stats;
    double* trace_p;          // [max_iters][3P] or null
    double* trace_l;          // [max_iters][3L] or null
    const volatile int* abort_host;   // mapped pinned word written by the host watcher
    int* abort_dev;           // [2] published copies (slot 0: written in phase A, slot 1: in phase F; read by all CTAs after the
                              // grid barrier that ends the phase - two slots so that a CTA running ahead into the next phase
                              // never overwrites a word a slower CTA has yet to read)
    double* part_chi;         // [2][team size]: row 0 = phase A (linearisation at x_cur), row 1 = phase F (chi2 at the trial point)
    double* part_scale;       // [team size]
    double* part_max;         // [team size]
    long long* phase_cycles;  // [8] SM cycles CTA 0 spent per phase incl. the barrier that ends it (profiling aid)
    int dyn_smem_bytes;       // dynamic shared memory of the launch (arena size of the non-zero CTAs)
    long long* cta_work;      // [team size][10] per-CTA busy cycles per phase (debug aid, null = off)
};

// Multi-GPU hooks of the persistent kernel (sharded runs on one NVLink node, se2gpu_ba_peer_import / _peer_attach_local): every
// rank runs the same cooperative kernel on its own landmarks; twice per lambda-trial the ranks exchange through peer memory
//   (1) the partial reduced systems [S | b_s]: after its Schur phase a rank publishes "epoch e complete" in a flag word of its
//       exchange block; when all flags are in, ALL CTAs of every rank sum the ranks' buffers slice by slice in rank order (own
//       buffer through the local pointer, the others over NVLink, every peer's load in flight at once: one round trip) into a
//       local buffer that the solve then stages - identical sums on every rank, so the replicated solves stay bit-identical;
//   (2) the scalars [chi2, scale, abort] (+ at iteration 0 the landmark-diagonal maximum and the pose diagonal for lambda_0):
//       same flags, a few doubles per rank.
// Only CTA 0 polls the peers (bounded spin); it hands the verdict to the other CTAs through a local word, so a missing peer
// makes every CTA of the rank leave the kernel with an error instead of hanging or trapping.
struct PKShard {
    int world, rank;
    const double* red[MAX_PEERS];      // partial [S | bs] of every rank
    const double* xch[MAX_PEERS];      // exchange block of every rank
    double* my_xch;                    // own exchange block
    double* ssum;                      // local: summed [S | bs]
    long long* go;                     // local [2]: epoch CTA 0 has seen complete on all peers (S, scalars); -1 = peer timeout
    long long epoch0, timeout_cycles;
    int xslot;                         // doubles per scalar slot
    const int* env_idx;                // linear indices (into [S | bs]) of the entries inside the envelope of S, then of bs
    int nenv;
};
// what one cluster of ba_persistent_cluster optimises (8-byte multiple: copied as 64-bit words)
struct PKWindow {
    Dev d;
    Cam cam;
    PKArgs pa;
};
static_assert(sizeof(PKWindow) % 8 == 0, "PKWindow is copied in 8-byte words");
constexpr int XCH_HDR = 16;            // doubles: [0] S flag, [1] scalar flag (as long long), rest padding

__device__ __forceinline__ void pk_publish(const PKShard& sh, int which, long long epoch) {     // CTA 0, thread 0, after a grid barrier
    __threadfence_system();
    *reinterpret_cast<volatile long long*>(sh.my_xch + which) = epoch;
    __threadfence_system();
}
// all threads of all CTAs; returns false on peer timeout (uniform across the grid)
template <class Team>
__device__ bool pk_wait_peers(const PKShard& sh, int which, long long epoch) {
    __shared__ long long s_go;
    if (Team::rank() == 0) {
        int ok = 1;
        if ((int)threadIdx.x < sh.world && (int)threadIdx.x != sh.rank) {
            const volatile long long* f = reinterpret_cast<const volatile long long*>(sh.xch[threadIdx.x] + which);
            const long long t0 = clock64();
            while (*f < epoch)
                if (clock64() - t0 > sh.timeout_cycles) { ok = 0; break; }
        }
        ok = __syncthreads_and(ok);
        if (threadIdx.x == 0) {
            __threadfence_system();
            *reinterpret_cast<volatile long long*>(sh.go + which) = ok ? epoch : -1;
            __threadfence();
        }
    }
    if (threadIdx.x == 0) {
        long long v;
        do { v = *reinterpret_cast<volatile long long*>(sh.go + which); } while (v >= 0 && v < epoch);
        __threadfence_system();
        s_go = v;
    }
    __syncthreads();
    const bool good = s_go >= 0;
    __syncthreads();
    return good;
}
// every CTA: ssum[e] = sum over ranks of red[r][e], rank order, for the entries e inside the envelope of the reduced system
// (the lower triangle within colmax[] - everything the Schur phase can write - and the right-hand side): a few percent of the
// dense n x n array for a local window, so the exchange moves kilobytes, not the whole buffer. ssum stays zero elsewhere.
template <class Team>
__device__ void pk_sum_partials(const PKShard& sh) {
    const int gtid = Team::rank() * blockDim.x + threadIdx.x, gthreads = Team::size() * blockDim.x;
    for (int v = gtid; v < sh.nenv; v += gthreads) {
        const int e = sh.env_idx[v];
        double t[MAX_PEERS];
#pragma unroll
        for (int r = 0; r < MAX_PEERS; ++r)
            if (r < sh.world) t[r] = (r == sh.rank) ? sh.red[r][e] : __ldcv(sh.red[r] + e);
        double acc = 0.0;
#pragma unroll
        for (int r = 0; r < MAX_PEERS; ++r)
            if (r < sh.world) acc += t[r];
        sh.ssum[e] = acc;
    }
}

// block-wide sum of a global array, same order in every CTA; result broadcast to all threads
__device__ double cta_sum_array(const double* a, int n, double* sh) {
    double v = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) v += a[i];
    const double r = block_sum(v, sh);
    __syncthreads();
    if (threadIdx.x == 0) sh[0] = r;
    __syncthreads();
    const double out = sh[0];
    __syncthreads();
    return out;
}
// Landmark work of the persistent kernel: lane groups (LPL lanes per landmark) are dealt to the CTAs round-robin, so every
// SM gets L / Team::size() landmarks on its first warps instead of the first CTAs running all 16 warps while the rest
// idle (the phases are FP64-issue bound per SM). Whole warps iterate together (the lane-group shuffles need them): the
// loop bound is the warp's first landmark; landmarks >= L are skipped inside the bodies.
template <class Team>
struct PKLmIter {
    int j, sub, step, j_warp;
    // In a sharded run only the landmarks j % world == rank carry work on this rank: the lane groups are dealt over THOSE (the
    // k-th owned landmark is j = k * world + rank), otherwise the owned landmarks alias onto a subset of the CTAs (world = 2
    // and an even grid: all of them on the even CTAs) and sharding buys no time per phase.
    __device__ __forceinline__ PKLmIter(const Dev& d) {
        const int lg = threadIdx.x / LPL;                       // lane group inside the CTA
        sub = threadIdx.x % LPL;
        j = (lg * Team::size() + Team::rank()) * d.world + d.rank;
        j_warp = ((threadIdx.x / 32) * (32 / LPL) * Team::size() + Team::rank()) * d.world + d.rank;
        step = (blockDim.x / LPL) * Team::size() * d.world;
    }
    __device__ __forceinline__ bool more(int L) const { return j_warp < L; }
    __device__ __forceinline__ void next() { j += step; j_warp += step; }
};

template <class Team, bool JAC>
__device__ void pk_phase_linearize(const Dev& d, const Cam& cam, int xi, double* part, double* sh, double lam_fuse = -1.0) {
    const double* xp = d.xp[xi];
    const double* xl = d.xl[xi];
    double chi = 0;
    for (PKLmIter<Team> it(d); it.more(d.L); it.next()) chi += pk_landmark<JAC, LPL, Team::kExplicitFma>(d, cam, xp, xl, it.j, it.sub, lam_fuse);
    // PreEdgeSE2 edges: one per CTA on the first lane of the last warp (idle unless a CTA holds > 60 landmarks), so that no CTA
    // serialises all of them behind its landmark work (they used to sit on CTA 0 and made it the slowest of the phase)
    if (threadIdx.x == blockDim.x - 32)
        for (int o = Team::rank(); o < d.O; o += Team::size()) chi += pk_odo<JAC>(d, xp, o);
    const double tot = block_sum(chi, sh);
    if (threadIdx.x == 0) part[Team::rank()] = tot;
}

// Static work lists of a persistent CTA, cached once per optimize() in its (otherwise unused) dynamic shared memory:
// the (edge, edge) pair lists of the blocks of S it owns and, for diagonal blocks, the pose's edge list. This removes
// the dependent L2 round trips for index data from every Schur / pose-gather phase (only the payload is gathered).
struct PKOwn { int blk, a, b, p0, np, e0, ne; };

// block (a >= b) of the reduced system; pairs interleaved (e1,e2) in `pairs` (shared) or null -> global lists at gp0.
// Its gather loops are written out rather than calling schur_pairs / schur_odo / schur_pose_sweep: with the shared loops here
// ptxas spills more of ba_persistent (sm_90a, CUDA 12.9: 372 B instead of 356 B of spill stores).
// A diagonal block also gathers the pose-side sums of its pose in the same sweep over the pose's edge list (Hpp_aa, b_p;
// the stand-alone pose gather of phase B is only needed at iteration 0, before lambda_0 exists) and stores them for
// the gain-ratio denominator. Summation order: thread-strided partials, warp xor-tree, per-warp sums in warp order.
__device__ void pk_schur_item(const Dev& d, double lam, int blk, int a, int b, const int* pairs, int gp0, int np, const int* edges, int ne,
                              double* shr /*[warps][21]*/) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t O = d.O, n = d.n, nf = d.nf;
    double acc[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) acc[q] = 0;
    for (int k = threadIdx.x; k < np; k += blockDim.x) {
        const int e1 = pairs ? pairs[2 * k] : d.pair_e1[gp0 + k], e2 = pairs ? pairs[2 * k + 1] : d.pair_e2[gp0 + k];
        double y[10], h[10];
        load_rec10(d.Y + (size_t)e1 * EB, y); load_rec10(d.Hpl + (size_t)e2 * EB, h);
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[r * 3 + c] -= y[r * 3] * h[c * 3] + y[r * 3 + 1] * h[c * 3 + 1] + y[r * 3 + 2] * h[c * 3 + 2];
    }
    for (int k = d.blk_odo_ptr[blk] + threadIdx.x; k < d.blk_odo_ptr[blk + 1]; k += blockDim.x) {
        const int code = d.blk_odo[k], o = code >> 1;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[r * 3 + c] += (code & 1) ? d.oAij[(c * 3 + r) * O + o] : d.oAij[(r * 3 + c) * O + o];
    }
    const bool diag = a == b;      // block-uniform
    double ph[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) ph[q] = 0;
    if (diag) {
        for (int k = threadIdx.x; k < ne; k += blockDim.x) {
            const double2* yr2 = reinterpret_cast<const double2*>(d.Y + (size_t)edges[k] * EB);
            const double2 g01 = yr2[4], g2 = yr2[5];        // doubles 8..11 of the record: Y[8], g[0], g[1], g[2]
            double rec[10];
            load_rec10(d.PH + (size_t)edges[k] * EB, rec);
            acc[9] -= g01.y; acc[10] -= g2.x; acc[11] -= g2.y;
#pragma unroll
            for (int q = 0; q < 9; ++q) ph[q] += rec[q];
        }
        for (int k = d.pose_odo_ptr[a] + threadIdx.x; k < d.pose_odo_ptr[a + 1]; k += blockDim.x) {
            const int code = d.pose_odo[k], o = code >> 1;
            const double* H = (code & 1) ? d.oAjj : d.oAii;
            const double* bb = (code & 1) ? d.obj : d.obi;
#pragma unroll
            for (int q = 0; q < 6; ++q) ph[q] += H[q * O + o];
#pragma unroll
            for (int q = 0; q < 3; ++q) ph[6 + q] += bb[q * O + o];
        }
    }
#pragma unroll
    for (int q = 0; q < 12; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    if (diag) {
#pragma unroll
        for (int q = 0; q < 9; ++q)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ph[q] += __shfl_xor_sync(0xffffffffu, ph[q], o);
    }
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 12; ++q) shr[wid * 21 + q] = acc[q];
        if (diag) {
#pragma unroll
            for (int q = 0; q < 9; ++q) shr[wid * 21 + 12 + q] = ph[q];
        }
    }
    __syncthreads();
    const int nwarp = (int)(blockDim.x >> 5);
    if (threadIdx.x < 12) {
        double v = 0;
        for (int w = 0; w < nwarp; ++w) v += shr[w * 21 + threadIdx.x];
        const int q = threadIdx.x;
        if (q < 9) {
            const int r = q / 3, c = q % 3;
            if (diag) {
                const int u6[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
                double hsum = 0;
                for (int w = 0; w < nwarp; ++w) hsum += shr[w * 21 + 12 + u6[r][c]];
                if (c >= r) d.Hpp[u6[r][c] * nf + a] = hsum;
                v += hsum + (r == c ? lam : 0.0);
            }
            d.S[(3 * a + r) * n + 3 * b + c] = v;
        } else if (diag) {
            double bsum = 0;
            for (int w = 0; w < nwarp; ++w) bsum += shr[w * 21 + 12 + 6 + (q - 9)];
            d.bp[3 * a + q - 9] = bsum;
            d.bs[3 * a + q - 9] = bsum + v;
        }
    }
}

// work split of the gather phases: CTA 0 runs the reduced solve and owns no blocks when the grid has other CTAs
struct PKWork {
    int first, stride;     // this CTA's blocks: first, first+stride, ... ; first < 0 -> none
    int n_own;             // of which the first n_own are cached in shared memory
    const PKOwn* own;
    const int* arena;
};

__device__ void pk_phase_pose_reduce(const Dev& d, const PKWork& w, double* sh9) {
    if (w.first < 0) return;
    int i = 0;
    for (int pos = w.first; pos < d.nord; pos += w.stride, ++i) {
        if (i < w.n_own) {
            const PKOwn o = w.own[i];
            if (o.a == o.b) pk_pose_item(d, o.a, w.arena + o.e0, o.ne, sh9);
        } else {
            const int blk = d.blk_order[pos];
            if (blk < 0) break;
            const int a = d.blk_a[blk];
            if (a == d.blk_b[blk]) pk_pose_item(d, a, d.pose_edges + d.pose_ptr[a], d.pose_ptr[a + 1] - d.pose_ptr[a], sh9);
        }
    }
}

__device__ void pk_phase_schur(const Dev& d, double lam, const PKWork& w, double* sh12) {
    if (w.first < 0) return;
    int i = 0;
    for (int pos = w.first; pos < d.nord; pos += w.stride, ++i) {
        if (i < w.n_own) {
            const PKOwn o = w.own[i];
            pk_schur_item(d, lam, o.blk, o.a, o.b, w.arena + o.p0, 0, o.np, w.arena + o.e0, o.ne, sh12);
        } else {
            const int blk = d.blk_order[pos];
            if (blk < 0) break;
            const int a = d.blk_a[blk], b = d.blk_b[blk];
            pk_schur_item(d, lam, blk, a, b, nullptr, d.blk_pair_ptr[blk], d.blk_pair_ptr[blk + 1] - d.blk_pair_ptr[blk],
                          d.pose_edges + d.pose_ptr[a], a == b ? d.pose_ptr[a + 1] - d.pose_ptr[a] : 0, sh12);
        }
    }
}

// Concurrent variant of pk_phase_schur: all blocks a CTA owns are processed at once, each by its own group of warps
// (plan_w0[i] = first warp, plan_nw[i] = number of warps of owned item i, proportional to the item's pair/edge count;
// built once per launch). One block barrier for the whole phase instead of two per block, and no warp idles while a
// 40-pair block is reduced. Summation order per block: lane-strided partials over the item's warps, warp xor-tree, the
// item's warps in rank order - fixed, so runs stay bit-reproducible.
__device__ void pk_phase_schur_par(const Dev& d, double lam, const PKWork& w, const unsigned char* plan_w0, const unsigned char* plan_nw, double* shr /*[warps][21]*/, double* red /*[warps][21][33]*/, long long* tdbg = nullptr) {
    if (w.first < 0) return;
    const long long t_in = tdbg ? clock64() : 0;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int it = -1, rk = 0, nwi = 1, w0 = 0;
    for (int i = 0; i < w.n_own; ++i)
        if (wid >= plan_w0[i] && wid < plan_w0[i] + plan_nw[i]) { it = i; w0 = plan_w0[i]; rk = wid - w0; nwi = plan_nw[i]; }
    PKOwn o{};
    bool diag = false;
    if (it >= 0) {
        o = w.own[it];
        diag = o.a == o.b;
        double acc[12], ph[9];
#pragma unroll
        for (int q = 0; q < 12; ++q) acc[q] = 0;
#pragma unroll
        for (int q = 0; q < 9; ++q) ph[q] = 0;
        const int* pairs = w.arena + o.p0;
        schur_pairs(d, pairs, pairs + 1, 2, o.np, rk * 32 + lane, nwi * 32, acc);
        if (rk == 0) schur_odo(d, o.blk, lane, 32, acc);
        if (diag) {
            schur_pose_sweep(d, w.arena + o.e0, o.ne, rk * 32 + lane, nwi * 32, acc, ph);
            if (rk == 0) pose_odo_gather(d, o.a, lane, 32, ph);
        }
        if (tdbg && threadIdx.x == 0) tdbg[8] += clock64() - t_in;      // gather loops of warp 0
        // warp reduction of the 21 partials through shared memory: every lane parks its values in a [21][33] tile (padded rows:
        // conflict-free), then lanes 0..20 each add one row in lane order - 21 stores + 32 loads per lane instead of 105
        // double-precision shuffle steps (210 SHFL + 105 DADD)
        double* sc = red + (size_t)wid * (21 * 33);
#pragma unroll
        for (int q = 0; q < 12; ++q) sc[q * 33 + lane] = acc[q];
#pragma unroll
        for (int q = 0; q < 9; ++q) sc[(12 + q) * 33 + lane] = ph[q];
        __syncwarp();
        if (lane < 21) {
            double v = 0;
#pragma unroll 8
            for (int i = 0; i < 32; ++i) v += sc[lane * 33 + i];
            shr[wid * 21 + lane] = v;
        }
        if (tdbg && threadIdx.x == 0) tdbg[9] += clock64() - t_in;      // ... + its reduction
    }
    __syncthreads();
    if (it >= 0 && rk == 0 && lane < 12) {
        const size_t n = d.n, nf = d.nf;
        const int q = lane;
        double v = 0;
        for (int r = 0; r < nwi; ++r) v += shr[(w0 + r) * 21 + q];
        if (q < 9) {
            const int r3 = q / 3, c3 = q % 3;
            if (diag) {
                const int u6[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
                double hsum = 0;
                for (int r = 0; r < nwi; ++r) hsum += shr[(w0 + r) * 21 + 12 + u6[r3][c3]];
                if (c3 >= r3) d.Hpp[u6[r3][c3] * nf + o.a] = hsum;
                v += hsum + (r3 == c3 ? lam : 0.0);
            }
            d.S[(3 * o.a + r3) * n + 3 * o.b + c3] = v;
        } else if (diag) {
            double bsum = 0;
            for (int r = 0; r < nwi; ++r) bsum += shr[(w0 + r) * 21 + 12 + 6 + (q - 9)];
            d.bp[3 * o.a + q - 9] = bsum;
            d.bs[3 * o.a + q - 9] = bsum + v;
        }
    }
}

template <class Team>
__device__ void pk_phase_lm_prep(const Dev& d, double lam) {
    const size_t L = d.L;
    for (PKLmIter<Team> it(d); it.more(d.L); it.next()) {
        const int j = it.j;
        if (j >= d.L) continue;
        const int beg = d.lm_ptr[j], end = d.lm_ptr[j + 1];
        if (end <= beg) continue;
        lm_damp(d, j, beg, end, it.sub, LPL, lam, d.Hll[j], d.Hll[L + j], d.Hll[2 * L + j], d.Hll[3 * L + j], d.Hll[4 * L + j],
                d.Hll[5 * L + j], d.bl[j], d.bl[L + j], d.bl[2 * L + j]);
    }
}

// E + F in one phase: back-substitution, oplus into the trial buffers, computeScale partial (returned) AND the robust chi2 at the
// trial point (*chi_out), with no grid barrier in between. The chi2 of a landmark's edges needs the landmark's trial point (formed
// by the same lane group a few instructions earlier) and the trial POSES: every CTA forms all of them itself first (P is a few
// dozen; all CTAs store identical values, and a CTA reads back only what it stored itself before its block barrier).
template <class Team>
__device__ double pk_phase_backsub(const Dev& d, const Cam& cam, int cur, double lam, double lam_pose, double* chi_out) {
    const double* xp = d.xp[cur];
    const double* xl = d.xl[cur];
    double* xpt = d.xp[cur ^ 1];
    double* xlt = d.xl[cur ^ 1];
    const size_t L = d.L;
    double sc = 0, chi = 0;
    for (int t = threadIdx.x; t < d.P; t += blockDim.x) pose_oplus(d, t, xp, xpt);
    __syncthreads();
    for (PKLmIter<Team> it(d); it.more(d.L); it.next()) {
        const int j = it.j, sub = it.sub;
        int beg = 0, end = 0;
        if (j < d.L) { beg = d.lm_ptr[j]; end = d.lm_ptr[j + 1]; }
        double c0 = 0, c1 = 0, c2 = 0;
        for (int k = beg + sub; k < end; k += LPL) {
            const int a = d.e_hidx[k];
            if (a < 0) continue;
            const double p0 = d.dxp[3 * a], p1 = d.dxp[3 * a + 1], p2 = d.dxp[3 * a + 2];
            double hp[10];
            load_rec10(d.Hpl + (size_t)k * EB, hp);
            c0 -= hp[0] * p0 + hp[3] * p1 + hp[6] * p2;
            c1 -= hp[1] * p0 + hp[4] * p1 + hp[7] * p2;
            c2 -= hp[2] * p0 + hp[5] * p1 + hp[8] * p2;
        }
        c0 = group_sum(c0); c1 = group_sum(c1); c2 = group_sum(c2);
        if (sub == 0 && j < d.L) {
            double dl0 = 0, dl1 = 0, dl2 = 0;
            if (end > beg) {
                c0 += d.bl[j]; c1 += d.bl[L + j]; c2 += d.bl[2 * L + j];
                const double i00 = d.HllInv[j], i01 = d.HllInv[L + j], i02 = d.HllInv[2 * L + j], i11 = d.HllInv[3 * L + j], i12 = d.HllInv[4 * L + j], i22 = d.HllInv[5 * L + j];
                dl0 = i00 * c0 + i01 * c1 + i02 * c2; dl1 = i01 * c0 + i11 * c1 + i12 * c2; dl2 = i02 * c0 + i12 * c1 + i22 * c2;
                sc += dl0 * (lam * dl0 + d.bl[j]) + dl1 * (lam * dl1 + d.bl[L + j]) + dl2 * (lam * dl2 + d.bl[2 * L + j]);
            }
            d.dxl[3 * j] = dl0; d.dxl[3 * j + 1] = dl1; d.dxl[3 * j + 2] = dl2;
            xlt[3 * j] = xl[3 * j] + dl0; xlt[3 * j + 1] = xl[3 * j + 1] + dl1; xlt[3 * j + 2] = xl[3 * j + 2] + dl2;
        }
        __syncwarp();                                           // the group's other lanes read the trial point back
        chi += pk_landmark<false, LPL, Team::kExplicitFma>(d, cam, xpt, xlt, j, sub, -1.0);
    }
    // pose terms of computeScale and the PreEdgeSE2 chi2: one item per CTA on the first lane of the last warp (see pk_phase_linearize)
    if (threadIdx.x == blockDim.x - 32) {
        for (int t = Team::rank(); t < d.P; t += Team::size()) {
            const int a = d.hidx[t];
            if (a >= 0) sc += pose_scale(d, a, lam_pose);
        }
        for (int o = Team::rank(); o < d.O; o += Team::size()) chi += pk_odo<false>(d, xpt, o);
    }
    *chi_out = chi;
    return sc;
}

// The whole optimize() of one window on the CTAs of `team` (see GridTeam / ClusterTeam). The LM arguments are taken by value:
// bound by reference to ba_persistent's parameter they cost it spill traffic (ptxas, sm_90a, CUDA 12.9).
template <class Team>
__device__ __forceinline__ void pk_optimize(Team& team, const Dev& d, const Cam& cam, const PKArgs pa, const PKShard& shd) {
    __shared__ double sh[32];
    __shared__ double shv[(PK_THREADS / 32) * 21];
    __shared__ __align__(8) unsigned long long stage_bar;
    unsigned stage_parity = 0;
    if (threadIdx.x == 0) mbar_init(&stage_bar, 1);
    // ---- static work lists of this CTA -> shared memory (CTA 0 keeps its shared memory for the reduced solve)
    extern __shared__ double sm[];
    __shared__ PKOwn own[PK_MAXOWN];
    __shared__ int s_nown, s_plan_ok;
    __shared__ unsigned char plan_w0[PK_MAXOWN], plan_nw[PK_MAXOWN];   // warp groups of the concurrent Schur phase
    constexpr int RED_SCRATCH_BYTES = PK_RED_SCRATCH_BYTES;
    double* red_scratch = sm + (pa.dyn_smem_bytes - RED_SCRATCH_BYTES) / 8;      // worker CTAs only (CTA 0 keeps its arena for the solve)
    PKWork work;
    {
        const int G = Team::size();
        const int nsolve = d.tw_m0 > 0 ? 2 : 1;             // CTAs that keep their shared memory for the reduced solve
        work.stride = G > 1 ? G - nsolve : 1;
        work.first = G > 1 ? (int)Team::rank() - nsolve : 0;  // < 0 for the solver CTAs of a multi-CTA grid
        work.own = own;
        work.arena = reinterpret_cast<const int*>(sm);
        int* arena = reinterpret_cast<int*>(sm);
        const int arena_ints = (G > 1 && work.first >= 0) ? (pa.dyn_smem_bytes - RED_SCRATCH_BYTES) / 4 : 0;   // the top of the arena is the reduction scratch
        if (threadIdx.x == 0) {
            int off = 0, no = 0;
            if (work.first >= 0)
                for (int pos = work.first; pos < d.nord && no < PK_MAXOWN; pos += work.stride) {
                    const int blk = d.blk_order[pos];
                    if (blk < 0) break;                     // holes only trail a worker's list
                    const int a = d.blk_a[blk], b = d.blk_b[blk];
                    const int np = d.blk_pair_ptr[blk + 1] - d.blk_pair_ptr[blk];
                    const int ne = (a == b) ? d.pose_ptr[a + 1] - d.pose_ptr[a] : 0;
                    if (off + 2 * np + ne > arena_ints) break;
                    own[no] = PKOwn{blk, a, b, off, np, off + 2 * np, ne};
                    off += 2 * np + ne; ++no;
                }
            s_nown = no;
            // concurrent Schur plan: possible when every owned block is cached; one warp per block, the spare warps go
            // one by one to the block with the most work per warp
            int total = 0;
            if (work.first >= 0) for (int pos = work.first; pos < d.nord; pos += work.stride) if (d.blk_order[pos] >= 0) ++total;
            const int nwarp = (int)(blockDim.x >> 5);
            s_plan_ok = (no == total && no > 0 && no <= nwarp) ? 1 : 0;
            if (s_plan_ok) {
                int wt[PK_MAXOWN], nwv[PK_MAXOWN];
                for (int i2 = 0; i2 < no; ++i2) { wt[i2] = own[i2].np + own[i2].ne + 8; nwv[i2] = 1; }
                for (int spare = nwarp - no; spare > 0; --spare) {
                    int best = 0;
                    for (int i2 = 1; i2 < no; ++i2) if ((long long)wt[i2] * nwv[best] > (long long)wt[best] * nwv[i2]) best = i2;
                    if (wt[best] <= 32 * nwv[best]) break;      // everybody already has a lane per work unit
                    ++nwv[best];
                }
                int at = 0;
                for (int i2 = 0; i2 < no; ++i2) { plan_w0[i2] = (unsigned char)at; plan_nw[i2] = (unsigned char)nwv[i2]; at += nwv[i2]; }
            }
        }
        __syncthreads();
        work.n_own = s_nown;
        for (int i = 0; i < work.n_own; ++i) {
            const PKOwn o = own[i];
            const int g0 = d.blk_pair_ptr[o.blk];
            for (int k = threadIdx.x; k < o.np; k += blockDim.x) { arena[o.p0 + 2 * k] = d.pair_e1[g0 + k]; arena[o.p0 + 2 * k + 1] = d.pair_e2[g0 + k]; }
            const int q0 = d.pose_ptr[o.a];
            for (int k = threadIdx.x; k < o.ne; k += blockDim.x) arena[o.e0 + k] = d.pose_edges[q0 + k];
        }
    }
    __syncthreads();
    const int n = d.n, nparts = Team::size();
    const bool shard = shd.world > 1;
    const double* Ssrc = shard ? shd.ssum : d.S;                   // what the solve stages: the rank-summed system in sharded runs
    const double* bsrc = shard ? shd.ssum + (size_t)n * n : d.bs;
    double lambda = d.st->lambda, ni = d.st->ni, chi_cur = d.st->chi_cur;   // continued from the previous call when first_iter > 0
    long long epoch = shd.epoch0;
    unsigned tw_seq = 0;
    if (d.tw_m0 > 0 && Team::rank() == 0 && threadIdx.x == 0) { d.tw_flag[0] = 0; d.tw_flag[1] = 0; d.tw_flag[2] = 0; }   // first use is several grid barriers away
    int cur = d.st->cur, done = 0;
    bool stop = false, peer_err = false;
    // scalar exchange of a sharded run: CTA 0 fills this rank's slot `epoch & 1` with v[0..nv) (+ the pose diagonal when
    // asked), publishes, everybody waits for the peers and reads all ranks' slots back in rank order
    auto xslot_of = [&](int r, long long e) { return shd.xch[r] + XCH_HDR + (size_t)(e & 1) * shd.xslot; };
    // phase timers live in shared memory and are touched by thread 0 only (keeps them out of the register budget)
    __shared__ long long tacc[8], wacc[10], tprev_s, wprev_s;
    if (threadIdx.x == 0) { for (int g = 0; g < 8; ++g) tacc[g] = 0; for (int g = 0; g < 10; ++g) wacc[g] = 0; tprev_s = wprev_s = clock64(); }
#define PK_TICK(g) do { if (threadIdx.x == 0) { const long long _t = clock64(); tacc[g] += _t - tprev_s; tprev_s = _t; wprev_s = _t; } } while (0)
#define PK_WORK(g) do { if (threadIdx.x == 0) { const long long _t = clock64(); wacc[g] += _t - wprev_s; wprev_s = _t; } } while (0)
    for (int it = 0; it < pa.max_iters && !stop; ++it) {
        const int itg = pa.first_iter + it;                       // g2o's iteration number
        // ---- A: linearise at x_cur (computeActiveErrors + buildSystem). For itg > 0 the damping of the first trial is already
        // known, so the damping-dependent landmark terms are formed in the same pass (no phase B, one grid barrier less).
        pk_phase_linearize<Team, true>(d, cam, cur, pa.part_chi, sh, itg > 0 ? lambda : -1.0);
        if (Team::rank() == 0 && threadIdx.x == 0) pa.abort_dev[0] = *pa.abort_host;
        PK_WORK(0);
        team.sync();
        PK_TICK(0);
        if (!shard && pa.abort_dev[0]) break;                      // sharded runs take the abort decision collectively (below)
        if (itg == 0) {
            // ---- B (first iteration only): pose-side gather and landmark diagonal maximum for lambda_0 = 1e-5 max|diag H|
            pk_phase_pose_reduce(d, work, shv);
            double m = 0;
            for (int j = Team::rank() * blockDim.x + threadIdx.x; j < d.L; j += Team::size() * blockDim.x)
                if (d.lm_ptr[j + 1] > d.lm_ptr[j]) m = fmax(m, diag_absmax(d.Hll, d.L, j));
            m = cta_max(m, sh);
            if (threadIdx.x == 0) pa.part_max[Team::rank()] = m;
            PK_WORK(1);
            team.sync();
            PK_TICK(1);
        }
        if (!shard || it == 0) chi_cur = cta_sum_array(pa.part_chi, nparts, sh);   // sharded: afterwards the accepted trial's global chi2 is carried
        if (itg == 0) {
            double m = 0;
            for (int i = threadIdx.x; i < nparts; i += blockDim.x) m = fmax(m, pa.part_max[i]);
            const size_t nf = d.nf;
            if (!shard) {
                for (int a = threadIdx.x; a < d.nf; a += blockDim.x) m = fmax(m, diag_absmax(d.Hpp, nf, a));
                m = cta_max(m, sh);
            } else {
                // lambda_0 needs the maximum over ALL landmarks and over the rank-SUMMED pose diagonal; chi2 and the abort flag ride along
                m = cta_max(m, sh);
                ++epoch;
                if (Team::rank() == 0) {
                    double* slot = shd.my_xch + XCH_HDR + (size_t)(epoch & 1) * shd.xslot;
                    if (threadIdx.x == 0) { slot[0] = chi_cur; slot[1] = 0.0; slot[2] = pa.abort_dev[0] ? 1.0 : 0.0; slot[3] = m; }
                    for (int a = threadIdx.x; a < d.nf; a += blockDim.x) { slot[8 + 3 * a] = d.Hpp[a]; slot[8 + 3 * a + 1] = d.Hpp[3 * nf + a]; slot[8 + 3 * a + 2] = d.Hpp[5 * nf + a]; }
                    __syncthreads();
                    if (threadIdx.x == 0) pk_publish(shd, 1, epoch);
                }
                if (!pk_wait_peers<Team>(shd, 1, epoch)) { peer_err = true; break; }
                double chi = 0, ab = 0, mm = 0;
                for (int r = 0; r < shd.world; ++r) { const double* sl = xslot_of(r, epoch); chi += __ldcv(sl); ab += __ldcv(sl + 2); mm = fmax(mm, __ldcv(sl + 3)); }
                for (int q = threadIdx.x; q < 3 * d.nf; q += blockDim.x) {
                    double v = 0;
                    for (int r = 0; r < shd.world; ++r) v += __ldcv(xslot_of(r, epoch) + 8 + q);
                    mm = fmax(mm, fabs(v));
                }
                m = cta_max(mm, sh);
                chi_cur = chi;
                if (ab > 0.0) break;
            }
            lm_lambda_init(m, lambda, ni);
        } else if (shard && it == 0) {
            // continuation call of a sharded run: this rank's chi2 partial -> global (one scalar exchange)
            ++epoch;
            if (Team::rank() == 0 && threadIdx.x == 0) {
                double* slot = shd.my_xch + XCH_HDR + (size_t)(epoch & 1) * shd.xslot;
                slot[0] = chi_cur; slot[1] = 0.0; slot[2] = pa.abort_dev[0] ? 1.0 : 0.0; slot[3] = 0.0;
                pk_publish(shd, 1, epoch);
            }
            if (!pk_wait_peers<Team>(shd, 1, epoch)) { peer_err = true; break; }
            double chi = 0, ab = 0;
            for (int r = 0; r < shd.world; ++r) { const double* sl = xslot_of(r, epoch); chi += __ldcv(sl); ab += __ldcv(sl + 2); }
            chi_cur = chi;
            if (ab > 0.0) break;
        }
        const double chi_before = chi_cur;
        const double lam_pose_mask = (d.rank == 0) ? 1.0 : 0.0;     // the damping of the pose block is added once across shards
        int trials = 0, accepted = 0;
        double rho = 0;
        do {
            // ---- P: damping-dependent per-landmark terms (first trial of itg > 0: already formed in phase A)
            PK_TICK(6);
            if (itg == 0 || trials > 0) {
                pk_phase_lm_prep<Team>(d, lambda);
                PK_WORK(2);
                team.sync();
            }
            PK_TICK(2);
            // ---- C: Schur complement gather
            if (s_plan_ok) pk_phase_schur_par(d, lambda * lam_pose_mask, work, plan_w0, plan_nw, shv, red_scratch, pa.cta_work ? wacc : nullptr);
            else pk_phase_schur(d, lambda * lam_pose_mask, work, shv);
            PK_WORK(3);
            team.sync();
            PK_TICK(3);
            if (shard) {
                // ---- X1: the all-reduce of the reduced system, inside the kernel: publish, wait for the peers, sum the ranks' buffers
                ++epoch;
                if (Team::rank() == 0 && threadIdx.x == 0) pk_publish(shd, 0, epoch);
                if (!pk_wait_peers<Team>(shd, 0, epoch)) { peer_err = true; break; }
                pk_sum_partials<Team>(shd);
                team.sync();
                PK_TICK(1);
            }
            // ---- D: reduced solve (one CTA; S staged into its shared memory)
            if (d.tw_m0 > 0) {
                ++tw_seq;
                if (Team::rank() < 2) ldlt_twisted_solve<Team>(d, Ssrc, bsrc, &stage_bar, stage_parity, tw_seq);
                stage_parity ^= 1;
            } else if (Team::rank() == 0) {
                ldlt_stage(d, Ssrc, &stage_bar, stage_parity);
                stage_parity ^= 1;
                PK_TICK(7);
                ldlt_block_solve<true>(nullptr, nullptr, n, nullptr, bsrc, d.dxp, d.st);
            }
            PK_WORK(4);
            team.sync();
            PK_TICK(4);
            const int solve_ok = d.st->solve_ok;
            // ---- E: back-substitution, oplus into the trial buffers, computeScale partials
            //      + F: robust chi2 at the trial point (same phase, see pk_phase_backsub)
            {
                double chi_part;
                const double sc = pk_phase_backsub<Team>(d, cam, cur, lambda, lambda * lam_pose_mask, &chi_part);
                const double tot = block_sum(sc, sh);
                if (threadIdx.x == 0) pa.part_scale[Team::rank()] = tot;
                const double totc = block_sum(chi_part, sh);
                if (threadIdx.x == 0) pa.part_chi[nparts + Team::rank()] = totc;
            }
            if (Team::rank() == 0 && threadIdx.x == 0) pa.abort_dev[1] = *pa.abort_host;
            PK_WORK(5);
            team.sync();
            PK_TICK(5);
            // ---- LM decision (identical in every CTA, and in every rank)
            double tempChi = cta_sum_array(pa.part_chi + nparts, nparts, sh);
            double scale = cta_sum_array(pa.part_scale, nparts, sh);
            double ab = pa.abort_dev[1] ? 1.0 : 0.0;
            if (shard) {
                // ---- X2: [chi2, scale, abort] summed over the ranks
                ++epoch;
                if (Team::rank() == 0 && threadIdx.x == 0) {
                    double* slot = shd.my_xch + XCH_HDR + (size_t)(epoch & 1) * shd.xslot;
                    slot[0] = tempChi; slot[1] = scale; slot[2] = ab; slot[3] = 0.0;
                    pk_publish(shd, 1, epoch);
                }
                if (!pk_wait_peers<Team>(shd, 1, epoch)) { peer_err = true; break; }
                tempChi = 0; scale = 0; ab = 0;
                for (int r = 0; r < shd.world; ++r) { const double* sl = xslot_of(r, epoch); tempChi += __ldcv(sl); scale += __ldcv(sl + 1); ab += __ldcv(sl + 2); }
            }
            if (lm_gain_step(tempChi, scale, solve_ok, chi_cur, lambda, ni, rho)) { cur ^= 1; accepted = 1; }
            ++trials;
            stop = ab > 0.0;
        } while (lm_retry(rho, trials) && !stop);
        if (peer_err) break;
        const se2gpu_ba_iter_stats o = lm_iter_stats(chi_before, chi_cur, lambda, rho, trials, accepted);
        if (Team::rank() == 0 && threadIdx.x == 0 && pa.stats) pa.stats[it] = o;
        if (pa.trace_p) for (int i = Team::rank() * blockDim.x + threadIdx.x; i < 3 * d.P; i += Team::size() * blockDim.x) pa.trace_p[(size_t)it * 3 * d.P + i] = d.xp[cur][i];
        if (pa.trace_l) for (int i = Team::rank() * blockDim.x + threadIdx.x; i < 3 * d.L; i += Team::size() * blockDim.x) pa.trace_l[(size_t)it * 3 * d.L + i] = d.xl[cur][i];
        ++done;
        if (o.terminate) stop = true;
    }
    PK_TICK(6);
#undef PK_TICK
#undef PK_WORK
    if (pa.cta_work && threadIdx.x == 0) for (int g = 0; g < 10; ++g) pa.cta_work[Team::rank() * 10 + g] = wacc[g];
    if (Team::rank() == 0 && threadIdx.x == 0) {
        LMState& s = *d.st;
        s.cur = cur; s.lambda = lambda; s.ni = ni; s.chi_cur = chi_cur; s.iter = done; s.epoch = epoch; s.error = peer_err ? 1 : 0;
        if (pa.phase_cycles) for (int g = 0; g < 8; ++g) pa.phase_cycles[g] += tacc[g];
    }
}

__global__ void __launch_bounds__(PK_THREADS, 1) ba_persistent(Dev d, Cam cam, PKArgs pa, PKShard shd) {
    GridTeam team;
    pk_optimize(team, d, cam, pa, shd);
}

// One window per thread-block cluster: cluster k optimises window k of the launch. The descriptor is copied once into shared
// memory from a device array the host fills per call (a parameter block would bound the batch by the 32 KB parameter limit:
// a descriptor is about 0.8 KB); the phases then read it as ba_persistent reads its parameters.
__global__ void __launch_bounds__(PK_THREADS, 1) ba_persistent_cluster(const PKWindow* __restrict__ windows) {
    __shared__ PKWindow w;
    const PKWindow* src = windows + blockIdx.x / ClusterTeam::size();
    for (int i = threadIdx.x; i < (int)(sizeof(PKWindow) / 8); i += blockDim.x)
        reinterpret_cast<unsigned long long*>(&w)[i] = reinterpret_cast<const unsigned long long*>(src)[i];
    __syncthreads();
    ClusterTeam team;
    const PKShard shd{};    // world 0: the batch runs unsharded windows only
    pk_optimize(team, w.d, w.cam, w.pa, shd);
}

// Map::optimizeLocalGraph write-back (Map.cpp:768-779): KeyFrame::setPose(Se2(vp(0), vp(1), vp(2))) narrows the pose to float
// and re-normalises the float angle (Se2::Se2, Config.cpp:194-195); MapPoint::setPos(toCvPt3f(...)) narrows the point.
__global__ void __launch_bounds__(256) ba_writeback_f32(const double* __restrict__ xp, int P, const double* __restrict__ xl, int L,
                                                        float* __restrict__ poses, float* __restrict__ points) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P && poses) {
        poses[3 * i] = (float)xp[3 * i]; poses[3 * i + 1] = (float)xp[3 * i + 1];
        poses[3 * i + 2] = (float)normalize_theta((double)(float)xp[3 * i + 2]);
    }
    if (i < L && points) { points[3 * i] = (float)xl[3 * i]; points[3 * i + 1] = (float)xl[3 * i + 1]; points[3 * i + 2] = (float)xl[3 * i + 2]; }
}

}  // namespace

// =================================================================================================
namespace {

// the only place the BA reads the environment
Switches read_switches() {
    Switches sw;
    if (const char* g = getenv("SE2GPU_BA_PK_GRID")) sw.pk_grid_limit = atoi(g);
    if (const char* t = getenv("SE2GPU_BA_PEER_TIMEOUT_S")) { if (atof(t) > 0) sw.peer_timeout_s = atof(t); }
    sw.debug = getenv("SE2GPU_BA_DEBUG") != nullptr;
    sw.no_band = getenv("SE2GPU_BA_NO_BAND") != nullptr;
    sw.no_twist = getenv("SE2GPU_BA_NO_TWIST") != nullptr;
    if (const char* c = getenv("SE2GPU_BA_BATCH_CLUSTER")) { const int v = atoi(c); if (v == 2 || v == 4 || v == 8) sw.batch_cluster = v; }
    return sw;
}

}  // namespace

extern "C" {

se2gpu_ba* se2gpu_ba_create(int max_poses, int max_points, int max_edges, int max_odo, int device) {
    if (max_poses <= 0 || max_points <= 0 || max_edges <= 0 || max_odo < 0) { fail(SE2GPU_ERR_INVALID, "bad capacities"); return nullptr; }
    if (se2gpu::select_device(device) != SE2GPU_OK) return nullptr;
    const size_t maxN = 3 * (size_t)max_poses;
    if (maxN * maxN * 8 > (size_t)8 << 30) { fail(SE2GPU_ERR_CAPACITY, "dense reduced system for %d poses exceeds this build's limit", max_poses); return nullptr; }
    se2gpu_ba* h = new se2gpu_ba;
    h->sw = read_switches();
    h->device = device; h->maxP = max_poses; h->maxL = max_points; h->maxE = max_edges; h->maxO = max_odo; h->maxN = (int)maxN;
    const size_t P = max_poses, L = max_points, E = max_edges, O = max_odo ? max_odo : 1;
    int rc = SE2GPU_OK;
    Dev& d = h->d;
    auto A = [&](auto** p, size_t c) {
        if (rc == SE2GPU_OK && h->bufs.alloc(p, c) != cudaSuccess) rc = fail(SE2GPU_ERR_CUDA, "cudaMalloc of %zu bytes failed", c * sizeof **p);
    };
    A(&d.xp[0], 3 * P); A(&d.xp[1], 3 * P); A(&d.xl[0], 3 * L); A(&d.xl[1], 3 * L); A(&d.st, 1);
    A(&d.e_pose, E); A(&d.e_hidx, E); A(&d.lm_ptr, L + 1); A(&d.hidx, P);
    A(&d.e_u, E); A(&d.e_v, E); A(&d.e_w00, E); A(&d.e_w01, E); A(&d.e_w11, E);
    A(&d.o_i, O); A(&d.o_j, O); A(&d.o_m, 3 * O); A(&d.o_w, 6 * O);
    A(&d.Hpl, EB * E); A(&d.PH, EB * E); A(&d.Y, EB * E);
    A(&d.Hll, 6 * L); A(&d.bl, 3 * L); A(&d.HllInv, 6 * L);
    A(&d.oAii, 6 * O); A(&d.oAij, 9 * O); A(&d.oAjj, 6 * O); A(&d.obi, 3 * O); A(&d.obj, 3 * O);
    A(&d.pose_ptr, P + 1); A(&d.pose_edges, E); A(&d.pose_odo_ptr, P + 1); A(&d.pose_odo, 2 * O);
    A(&d.Hpp, 6 * P); A(&d.bp, 3 * P);
    A(&h->red, maxN * maxN + maxN + 8); A(&h->ywork, 4 * maxN + 32); A(&d.colmax, maxN); A(&d.tw_cmax1, maxN); A(&d.tw_buf, TW_BUF_DOUBLES); A(&d.tw_flag, 4); A(&d.dxp, maxN); A(&d.dxl, 3 * L);
    const size_t nb = (L + LM_THREADS - 1) / LM_THREADS + (O + LM_THREADS - 1) / LM_THREADS + (P + LM_THREADS - 1) / LM_THREADS + 4;
    A(&d.part_chi, nb); A(&d.part_scale, nb);
    A(&h->stats_dev, h->max_stats);
    A(&h->xp0, 3 * P); A(&h->xl0, 3 * L); A(&h->wb32, 3 * P + 8 + 3 * L);
    A(&h->pk_part_chi, 2048); A(&h->pk_part_scale, 1024); A(&h->pk_part_max, 1024); A(&h->abort_dev, 2); A(&h->phase_cycles, 8); A(&h->cta_work, 1024 * 10);
    if (rc == SE2GPU_OK && cudaMallocHost((void**)&h->st_host, sizeof(LMState)) != cudaSuccess) rc = fail(SE2GPU_ERR_CUDA, "cudaMallocHost failed");
    if (rc == SE2GPU_OK) {
        cudaFuncSetAttribute(ba_chol_solve_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ldlt_smem_bytes(SMEM_CHOL_MAX_N));
    }
    if (rc == SE2GPU_OK) {
        // persistent cooperative kernel: one CTA per SM, all co-resident
        const int smem_max = (int)ldlt_smem_bytes(SMEM_CHOL_MAX_N);
        int coop = 0, nsm = 0, occ = 0;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device);
        cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device);
        cudaDeviceGetAttribute(&h->clock_khz, cudaDevAttrClockRate, device);
        cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        cudaMemset(h->phase_cycles, 0, 8 * sizeof(long long));
        if (coop && cudaFuncSetAttribute(ba_persistent, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max) == cudaSuccess &&
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ba_persistent, PK_THREADS, smem_max) == cudaSuccess && occ >= 1)
            h->pk_grid = std::min(nsm, 1024);
        if (h->sw.pk_grid_limit >= 2 && h->sw.pk_grid_limit < h->pk_grid) h->pk_grid = h->sw.pk_grid_limit;
        cudaGetLastError();
        if (cudaHostAlloc((void**)&h->abort_host, sizeof(int), cudaHostAllocMapped) != cudaSuccess ||
            cudaHostGetDevicePointer((void**)&h->abort_host_dev, h->abort_host, 0) != cudaSuccess) { h->pk_grid = 0; cudaGetLastError(); }
        else *h->abort_host = 0;
    }
    if (rc != SE2GPU_OK) { se2gpu_ba_destroy(h); return nullptr; }
    return h;
}

void se2gpu_ba_destroy(se2gpu_ba* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->abort_host) cudaFreeHost(h->abort_host);
    se2band::release(h->band);
    for (void* m : h->peer_opened) if (m) cudaIpcCloseMemHandle(m);
    // the peer exchange buffers are separate allocations (peer_alloc: a rank exports them by IPC handle); h->bufs frees the rest
    if (h->xch) cudaFree(h->xch);
    if (h->ssum) cudaFree(h->ssum);
    if (h->go) cudaFree(h->go);
    if (h->st_host) cudaFreeHost(h->st_host);
    if (h->dl.sc_host) cudaFreeHost(h->dl.sc_host);
    delete h;
}

static int peer_alloc(se2gpu_ba* h) {
    if (h->xch) return SE2GPU_OK;
    SE2_CUDA(cudaSetDevice(h->device));
    h->xslot = (8 + 3 * h->maxP + 7) & ~7;
    const size_t xd = XCH_HDR + 2 * (size_t)h->xslot;
    SE2_CUDA(cudaMalloc((void**)&h->xch, sizeof(double) * xd));
    SE2_CUDA(cudaMemset(h->xch, 0, sizeof(double) * xd));
    SE2_CUDA(cudaMalloc((void**)&h->ssum, sizeof(double) * ((size_t)SMEM_CHOL_MAX_N * SMEM_CHOL_MAX_N + SMEM_CHOL_MAX_N + 8)));
    SE2_CUDA(cudaMemset(h->ssum, 0, sizeof(double) * ((size_t)SMEM_CHOL_MAX_N * SMEM_CHOL_MAX_N + SMEM_CHOL_MAX_N + 8)));
    SE2_CUDA(cudaMalloc((void**)&h->go, 2 * sizeof(long long)));
    SE2_CUDA(cudaMemset(h->go, 0, 2 * sizeof(long long)));
    return SE2GPU_OK;
}

int se2gpu_ba_peer_export(se2gpu_ba* h, void* handle_out) {
    if (!h || !handle_out) return fail(SE2GPU_ERR_INVALID, "null argument");
    int rc = peer_alloc(h);
    if (rc != SE2GPU_OK) return rc;
    cudaIpcMemHandle_t hs[2];
    SE2_CUDA(cudaIpcGetMemHandle(&hs[0], h->red));
    SE2_CUDA(cudaIpcGetMemHandle(&hs[1], h->xch));
    static_assert(sizeof(hs) == SE2GPU_BA_PEER_HANDLE_BYTES, "handle size");
    memcpy(handle_out, hs, sizeof hs);
    return SE2GPU_OK;
}

int se2gpu_ba_peer_import(se2gpu_ba* h, const void* handles, int world) {
    if (!h || !handles) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (world != h->world || world < 2 || world > MAX_PEERS) return fail(SE2GPU_ERR_INVALID, "peer exchange needs 2..%d ranks matching se2gpu_ba_set_shard", MAX_PEERS);
    if (!h->xch) return fail(SE2GPU_ERR_INVALID, "call se2gpu_ba_peer_export first");
    SE2_CUDA(cudaSetDevice(h->device));
    const cudaIpcMemHandle_t* hs = static_cast<const cudaIpcMemHandle_t*>(handles);
    for (int r = 0; r < world; ++r) {
        if (r == h->rank) { h->peer_red[r] = h->red; h->peer_xch[r] = h->xch; continue; }
        void *pr = nullptr, *pf = nullptr;
        if (cudaIpcOpenMemHandle(&pr, hs[2 * r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess ||
            cudaIpcOpenMemHandle(&pf, hs[2 * r + 1], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            const cudaError_t e = cudaGetLastError();
            if (pr) cudaIpcCloseMemHandle(pr);
            return fail(SE2GPU_ERR_CUDA, "cudaIpcOpenMemHandle for rank %d failed: %s", r, cudaGetErrorString(e));
        }
        h->peer_red[r] = static_cast<const double*>(pr); h->peer_xch[r] = static_cast<const double*>(pf);
        for (void*& slot : h->peer_opened) if (!slot) { slot = pr; break; }
        for (void*& slot : h->peer_opened) if (!slot) { slot = pf; break; }
    }
    h->peer_on = true;
    return SE2GPU_OK;
}

int se2gpu_ba_peer_attach_local(se2gpu_ba** hs, int world) {
    if (!hs || world < 2 || world > MAX_PEERS) return fail(SE2GPU_ERR_INVALID, "peer exchange needs 2..%d contexts", MAX_PEERS);
    for (int r = 0; r < world; ++r) {
        if (!hs[r] || hs[r]->world != world || hs[r]->rank != r) return fail(SE2GPU_ERR_INVALID, "context %d is not rank %d of %d (se2gpu_ba_set_shard)", r, r, world);
        int rc = peer_alloc(hs[r]);
        if (rc != SE2GPU_OK) return rc;
    }
    for (int r = 0; r < world; ++r)
        for (int q = 0; q < world; ++q) {
            if (q != r && hs[q]->device != hs[r]->device) {      // same process, different GPUs: direct peer access
                SE2_CUDA(cudaSetDevice(hs[r]->device));
                int can = 0;
                SE2_CUDA(cudaDeviceCanAccessPeer(&can, hs[r]->device, hs[q]->device));
                if (!can) return fail(SE2GPU_ERR_CUDA, "device %d cannot access device %d", hs[r]->device, hs[q]->device);
                const cudaError_t e = cudaDeviceEnablePeerAccess(hs[q]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(SE2GPU_ERR_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
                cudaGetLastError();
            }
            hs[r]->peer_red[q] = hs[q]->red; hs[r]->peer_xch[q] = hs[q]->xch;
        }
    for (int r = 0; r < world; ++r) hs[r]->peer_on = true;
    return SE2GPU_OK;
}

int se2gpu_ba_set_stream(se2gpu_ba* h, void* stream) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    h->stream = (cudaStream_t)stream;
    return SE2GPU_OK;
}

int se2gpu_ba_set_shard(se2gpu_ba* h, int rank, int world, se2gpu_allreduce_fn allreduce, void* user) {
    if (!h || world < 1 || rank < 0 || rank >= world) return fail(SE2GPU_ERR_INVALID, "bad shard %d/%d", rank, world);
    if (world > 1 && !allreduce) return fail(SE2GPU_ERR_INVALID, "sharded BA needs an allreduce callback");
    h->rank = rank; h->world = world; h->allreduce = allreduce; h->ar_user = user;
    return SE2GPU_OK;
}

}  // extern "C"

namespace {

int ar(se2gpu_ba* h, double* buf, size_t count, int op) {
    if (h->world == 1) return SE2GPU_OK;
    int rc = h->allreduce(h->ar_user, buf, count, op, (void*)h->stream);
    if (rc != 0) return fail(SE2GPU_ERR_CUDA, "allreduce callback failed (%d)", rc);
    return SE2GPU_OK;
}

int launch_linearize(se2gpu_ba* h) {
    SE2_NVTX("se2gpu.ba.linearize");
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    h->prof.begin(0, s);
    if (d.nb_lm + d.nb_odo > 0) SE2_LAUNCH(ba_linearize<true>, d.nb_lm + d.nb_odo, LM_THREADS, 0, s, d, h->cam, 0);
    h->prof.end(s);
    h->prof.begin(1, s);
    if (d.nf > 0) SE2_LAUNCH(ba_pose_reduce, d.nf, POSE_THREADS, 0, s, d);
    h->prof.end(s);
    return SE2GPU_OK;
}

// elements of S as stored: dense for small windows, the band for large ones
size_t stored_S_elems(const se2gpu_ba* h) { return h->band.active ? h->band.band_elems : (size_t)h->d.n * h->d.n; }

// damping-dependent landmark terms at the current lambda, then this rank's reduced system [S | bs]
int launch_schur(se2gpu_ba* h) {
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    h->prof.begin(2, s);
    if (d.nb_lm > 0) SE2_LAUNCH(ba_lm_prep, d.nb_lm, LM_THREADS, 0, s, d);
    h->prof.end(s);
    // the global-memory Cholesky factorises S in place (fill-in outside the block list): re-zero it
    if (d.n > SMEM_CHOL_MAX_N) SE2_CUDA(cudaMemsetAsync(d.S, 0, sizeof(double) * stored_S_elems(h), s));
    h->prof.begin(3, s);
    if (d.nblk > 0) SE2_LAUNCH(ba_schur, d.nblk, SCHUR_THREADS, 0, s, d);
    h->prof.end(s);
    return SE2GPU_OK;
}

// S dx_p = bs by the solver the window's size and envelope selected
int launch_reduced_solve(se2gpu_ba* h) {
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    int rc = SE2GPU_OK;
    h->prof.begin(4, s);
    if (d.n <= SMEM_CHOL_MAX_N) SE2_LAUNCH(ba_chol_solve_smem, 1, CHOL_THREADS, ldlt_smem_bytes(d.n), s, d);   // n == 0: trivially ok
    else if (h->band.active) { if ((rc = se2band::solve(h->band, d.S, d.bs, d.dxp, &d.st->solve_ok, s)) != SE2GPU_OK) return rc; }
    else SE2_LAUNCH(ba_chol_solve_gmem, 1, CHOL_THREADS, 0, s, d, h->ywork);
    h->prof.end(s);
    return SE2GPU_OK;
}

int launch_solve(se2gpu_ba* h) {
    SE2_NVTX("se2gpu.ba.schur_solve");
    int rc = launch_schur(h);
    if (rc != SE2GPU_OK) return rc;
    if ((rc = ar(h, h->d.S, stored_S_elems(h) + h->d.n, 0)) != SE2GPU_OK) return rc;     // the message is the stored pattern
    return launch_reduced_solve(h);
}

}  // namespace

extern "C" {

int se2gpu_ba_optimize(se2gpu_ba* h, int max_iters, const volatile unsigned char* stop_flag, se2gpu_ba_iter_stats* stats,
                       double* trace_poses, double* trace_points) {
    return se2gpu_ba_optimize_from(h, 0, max_iters, stop_flag, stats, trace_poses, trace_points);
}

int se2gpu_ba_optimize_from(se2gpu_ba* h, int first_iteration, int max_iters, const volatile unsigned char* stop_flag,
                            se2gpu_ba_iter_stats* stats, double* trace_poses, double* trace_points) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    SE2_NVTX("se2gpu.ba.optimize");
    if (max_iters < 0 || first_iteration < 0) return fail(SE2GPU_ERR_INVALID, "negative iteration count");
    if (max_iters > h->max_stats) return fail(SE2GPU_ERR_CAPACITY, "max_iters > %d", h->max_stats);
    SE2_CUDA(cudaSetDevice(h->device));
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    const bool can_persist = (h->world == 1 || h->peer_on) && h->pk_grid > 0 && d.n <= SMEM_CHOL_MAX_N;
    if (h->mode == 2 && !can_persist) return fail(SE2GPU_ERR_INVALID, "persistent mode unavailable (sharded run without peer exchange, %d unknowns > %d, or no cooperative launch)", d.n, SMEM_CHOL_MAX_N);
    if (can_persist && h->mode != 1) {
        if (max_iters == 0) return 0;
        if (h->world == 1 && stop_flag && *stop_flag) return 0;      // sharded: the kernel takes the decision collectively
        // the whole optimize() is ONE cooperative launch; the host only forwards the abort flag while it runs
        // (a trace buffer that is replaced is idle: the launch that wrote it was waited for before optimize returned)
        if (trace_poses && h->trace_cap_p < (size_t)max_iters * 3 * h->P) {
            h->trace_cap_p = 0;
            SE2_CUDA(h->bufs.regrow(&h->trace_p, (size_t)max_iters * 3 * h->P));
            h->trace_cap_p = (size_t)max_iters * 3 * h->P;
        }
        if (trace_points && h->trace_cap_l < (size_t)max_iters * 3 * h->L) {
            h->trace_cap_l = 0;
            SE2_CUDA(h->bufs.regrow(&h->trace_l, (size_t)max_iters * 3 * h->L));
            h->trace_cap_l = (size_t)max_iters * 3 * h->L;
        }
        if (const int rc = plan_for_grid(h, h->pk_grid)) return rc;     // after a batched optimize the plan was made for a cluster
        *h->abort_host = (stop_flag && *stop_flag) ? 1 : 0;
        PKShard shd{};
        shd.world = h->world; shd.rank = h->rank;
        if (h->world > 1) {
            for (int r = 0; r < h->world; ++r) { shd.red[r] = h->peer_red[r]; shd.xch[r] = h->peer_xch[r]; }
            shd.my_xch = h->xch; shd.ssum = h->ssum; shd.go = h->go; shd.epoch0 = h->peer_epoch; shd.xslot = h->xslot;
            shd.env_idx = h->env_idx; shd.nenv = h->nenv;
            shd.timeout_cycles = (long long)(h->sw.peer_timeout_s * 1e3 * (double)(h->clock_khz > 0 ? h->clock_khz : FALLBACK_CLOCK_KHZ));
            SE2_CUDA(cudaMemsetAsync(h->go, 0, 2 * sizeof(long long), s));
        }
        PKArgs pa{max_iters, first_iteration, h->stats_dev, trace_poses ? h->trace_p : nullptr, trace_points ? h->trace_l : nullptr,
                  h->abort_host_dev, h->abort_dev, h->pk_part_chi, h->pk_part_scale, h->pk_part_max, h->prof.on ? h->phase_cycles : nullptr, 0, h->sw.debug ? h->cta_work : nullptr};
        if (h->prof.on) h->pk_launches++;
        const size_t smem = pk_dyn_smem_bytes(d.n);      // worker CTAs: pair lists + 87 KB of reduction scratch
        pa.dyn_smem_bytes = (int)smem;
        void* args[] = {(void*)&d, (void*)&h->cam, (void*)&pa, (void*)&shd};
        h->prof.begin(7, s);
        SE2_CUDA(cudaLaunchCooperativeKernel((void*)ba_persistent, dim3(h->pk_grid), dim3(PK_THREADS), args, smem, s));
        se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
        h->prof.end(s);
        SE2_CUDA(cudaMemcpyAsync(h->st_host, d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
        if (stop_flag) {
            while (cudaStreamQuery(s) == cudaErrorNotReady) if (*stop_flag) *(volatile int*)h->abort_host = 1;
        }
        SE2_CUDA(cudaStreamSynchronize(s));
        const int done = h->st_host->iter;
        if (h->world > 1) {
            h->peer_epoch = h->st_host->epoch;
            if (h->st_host->error) return fail(SE2GPU_ERR_CUDA, "sharded BA: a peer rank did not reach the exchange within %.1f s (rank %d of %d)", h->sw.peer_timeout_s, h->rank, h->world);
        }
        if (pa.cta_work) {   // SE2GPU_BA_DEBUG=1: per-phase busy cycles of every CTA (max / mean / who) to stderr
            std::vector<long long> w((size_t)h->pk_grid * 10);
            cudaMemcpy(w.data(), h->cta_work, w.size() * sizeof(long long), cudaMemcpyDeviceToHost);
            const char* names[10] = {"linearize", "pose+prep", "lm_prep", "schur", "solve", "backsub", "-", "chi2", "schur:gather", "schur:+shfl"};
            for (int g = 0; g < 10; ++g) {
                long long mx = 0, sum = 0; int who = 0;
                for (int c = 0; c < h->pk_grid; ++c) { const long long v = w[(size_t)c * 10 + g]; sum += v; if (v > mx) { mx = v; who = c; } }
                fprintf(stderr, "[se2gpu_ba] phase %-10s busy cycles: max %lld (CTA %d) mean %lld  (per optimize of %d iters)\n", names[g], mx, who, sum / h->pk_grid, done);
            }
        }
        if (stats && done > 0) SE2_CUDA(cudaMemcpyAsync(stats, h->stats_dev, sizeof(se2gpu_ba_iter_stats) * done, cudaMemcpyDeviceToHost, s));
        if (trace_poses && done > 0) SE2_CUDA(cudaMemcpyAsync(trace_poses, h->trace_p, sizeof(double) * (size_t)done * 3 * h->P, cudaMemcpyDeviceToHost, s));
        if (trace_points && done > 0) SE2_CUDA(cudaMemcpyAsync(trace_points, h->trace_l, sizeof(double) * (size_t)done * 3 * h->L, cudaMemcpyDeviceToHost, s));
        SE2_CUDA(cudaStreamSynchronize(s));
        return done;
    }
    int done = 0;
    bool ok = true;
    // Sharded runs: every rank must take the same abort decision, otherwise one leaves the loop while the others enter the
    // next collective. The flag each rank sees is therefore summed over the ranks: once at entry, then as a third word of
    // the per-trial [chi2, scale] all-reduce (LMState::stop_all).
    bool stop_all = stop_flag && *stop_flag;
    if (h->world > 1 && stop_flag) {
        const double mine = stop_all ? 1.0 : 0.0;
        double all = 0;
        SE2_CUDA(cudaMemcpyAsync(d.scal + 2, &mine, sizeof(double), cudaMemcpyHostToDevice, s));
        int rc0 = ar(h, d.scal + 2, 1, 0);
        if (rc0 != SE2GPU_OK) return rc0;
        SE2_CUDA(cudaMemcpyAsync(&all, d.scal + 2, sizeof(double), cudaMemcpyDeviceToHost, s));
        SE2_CUDA(cudaStreamSynchronize(s));
        stop_all = all > 0.0;
    }
    for (int it = 0; it < max_iters && !stop_all && ok; ++it) {
        const int itg = first_iteration + it;
        int rc = launch_linearize(h);
        if (rc != SE2GPU_OK) return rc;
        h->prof.begin(6, s);
        SE2_LAUNCH(ba_iter_begin, 1, 256, 0, s, d, it, 0, itg);
        h->prof.end(s);
        if (h->world > 1) {
            // chi2 is summed; lambda_init needs max|diag| over the SUMMED pose diagonal and all landmarks
            if ((rc = ar(h, d.scal, 1, 0)) != SE2GPU_OK) return rc;
            if (itg == 0) {
                if ((rc = ar(h, d.scal + 1, 1, 1)) != SE2GPU_OK) return rc;   // max over ranks of the landmark diagonal
                // pose diagonal: sum the 6 x nf block array across ranks on a scratch copy (S is free here), fold its
                // diagonal maximum into scal[1] on the device - no host round trip
                double* scratch = d.S;
                SE2_CUDA(cudaMemcpyAsync(scratch, d.Hpp, sizeof(double) * 6 * d.nf, cudaMemcpyDeviceToDevice, s));
                if ((rc = ar(h, scratch, 6 * (size_t)d.nf, 0)) != SE2GPU_OK) return rc;
                SE2_LAUNCH(ba_pose_diag_max, 1, 256, 0, s, scratch, d.nf, d.scal + 1);
                SE2_CUDA(cudaMemsetAsync(d.S, 0, sizeof(double) * 6 * d.nf, s));
            }
            SE2_LAUNCH(ba_iter_begin, 1, 256, 0, s, d, it, 1, itg);
        }
        bool retry = true;
        while (retry) {
            if ((rc = launch_solve(h)) != SE2GPU_OK) return rc;
            h->prof.begin(5, s);
            SE2_LAUNCH(ba_backsub_update, h->nb_scale, LM_THREADS, 0, s, d);
            h->prof.end(s);
            h->prof.begin(0, s);
            if (d.nb_lm + d.nb_odo > 0) SE2_LAUNCH(ba_linearize<false>, d.nb_lm + d.nb_odo, LM_THREADS, 0, s, d, h->cam, 1);
            h->prof.end(s);
            h->prof.begin(6, s);
            SE2_LAUNCH(ba_decide, 1, 256, 0, s, d, h->nb_scale, 0, h->stats_dev, (stop_flag && *stop_flag) ? 1 : 0);
            h->prof.end(s);
            if (h->world > 1) {
                if ((rc = ar(h, d.scal, 3, 0)) != SE2GPU_OK) return rc;
                SE2_LAUNCH(ba_decide, 1, 256, 0, s, d, h->nb_scale, 1, h->stats_dev, 0);
            }
            SE2_CUDA(cudaMemcpyAsync(h->st_host, d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
            SE2_CUDA(cudaStreamSynchronize(s));
            retry = h->st_host->retry != 0;          // already cleared on the device when any rank raised the abort flag
            stop_all = h->st_host->stop_all != 0;
        }
        const LMState& st = *h->st_host;
        const se2gpu_ba_iter_stats o = lm_iter_stats(st.chi_before, st.chi_cur, st.lambda, st.rho, st.trials, st.accepted);
        if (stats) stats[it] = o;
        if (trace_poses) SE2_CUDA(cudaMemcpyAsync(trace_poses + (size_t)it * 3 * h->P, d.xp[st.cur], sizeof(double) * 3 * h->P, cudaMemcpyDeviceToHost, s));
        if (trace_points) SE2_CUDA(cudaMemcpyAsync(trace_points + (size_t)it * 3 * h->L, d.xl[st.cur], sizeof(double) * 3 * h->L, cudaMemcpyDeviceToHost, s));
        ok = !o.terminate;
        ++done;
    }
    SE2_CUDA(cudaStreamSynchronize(s));
    return done;
}

}  // extern "C"

namespace {

// Cluster size of the batched launch: 8 CTAs for every window. Measured against 2 and 4 on windows of 9, 19 and 49 free poses
// at B = 1 to 64 (tools/ba_batch_bench.py, DESIGN.md section 3 "Batches of windows"), 8 was the fastest on every workload, so
// no rule depends on the window. It never depends on the batch, so a window's bytes do not depend on its batchmates.
// SE2GPU_BA_BATCH_CLUSTER sets another size per context, for measuring.
constexpr int kBatchCluster = 8;
int batch_cluster_size(const se2gpu_ba* h) { return h->sw.batch_cluster ? h->sw.batch_cluster : kBatchCluster; }

// At first use of a cluster size on a device: the launch attribute for the largest window and the scheduling check. A size
// the device cannot schedule is an error; another size would give other results.
int check_cluster_size(int device, int C) {
    static std::mutex mu;
    static bool ok[se2gpu::kMaxDevices][9] = {};
    if (device < 0 || device >= se2gpu::kMaxDevices) return fail(SE2GPU_ERR_INVALID, "device %d", device);
    std::lock_guard<std::mutex> lock(mu);
    if (ok[device][C]) return SE2GPU_OK;
    const int smem_max = (int)pk_dyn_smem_bytes(SMEM_CHOL_MAX_N);
    SE2_CUDA(cudaFuncSetAttribute(ba_persistent_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = C; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(C); cfg.blockDim = dim3(PK_THREADS); cfg.dynamicSmemBytes = smem_max; cfg.attrs = &attr; cfg.numAttrs = 1;
    int clusters = 0;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&clusters, (void*)ba_persistent_cluster, &cfg);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(SE2GPU_ERR_CUDA, "cudaOccupancyMaxActiveClusters for clusters of %d CTAs: %s", C, cudaGetErrorString(e)); }
    if (clusters < 1) return fail(SE2GPU_ERR_CUDA, "device %d cannot schedule a cluster of %d CTAs of %d threads and %d bytes of shared memory", device, C, PK_THREADS, smem_max);
    ok[device][C] = true;
    return SE2GPU_OK;
}

}  // namespace

extern "C" {

int se2gpu_ba_batch_cluster(se2gpu_ba* h) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    return batch_cluster_size(h);
}

int se2gpu_ba_optimize_batch(se2gpu_ba* const* hs, int B, int max_iters, const volatile unsigned char* const* stop_flags, int* iterations,
                             se2gpu_ba_iter_stats* stats, double* const* trace_poses, double* const* trace_points) {
    if (!hs || B < 1) return fail(SE2GPU_ERR_INVALID, "no contexts");
    if (max_iters < 0) return fail(SE2GPU_ERR_INVALID, "negative iteration count");
    SE2_NVTX("se2gpu.ba.optimize_batch");
    // every refusal comes before anything changes
    std::unordered_map<const se2gpu_ba*, int> seen;
    for (int k = 0; k < B; ++k) {
        se2gpu_ba* h = hs[k];
        if (!h) return fail(SE2GPU_ERR_INVALID, "window %d: null context", k);
        const auto at = seen.emplace(h, k);
        if (!at.second) return fail(SE2GPU_ERR_INVALID, "window %d: the context of window %d again", k, at.first->second);
        if (h->device != hs[0]->device) return fail(SE2GPU_ERR_INVALID, "window %d: device %d, window 0 is on device %d", k, h->device, hs[0]->device);
        if (h->world != 1) return fail(SE2GPU_ERR_INVALID, "window %d: sharded context (rank %d of %d)", k, h->rank, h->world);
        if (!h->loaded) return fail(SE2GPU_ERR_INVALID, "window %d: no problem loaded", k);
        if (h->pk_grid <= 0) return fail(SE2GPU_ERR_INVALID, "window %d: the persistent kernel is unavailable on this context", k);
        if (h->mode == 1) return fail(SE2GPU_ERR_INVALID, "window %d: context in multi-launch mode (se2gpu_ba_set_mode 1); the batch runs the persistent kernel", k);
        if (h->d.n > SMEM_CHOL_MAX_N) return fail(SE2GPU_ERR_CAPACITY, "window %d: %d unknowns > %d (se2gpu_ba_optimize runs it)", k, h->d.n, SMEM_CHOL_MAX_N);
        if (max_iters > h->max_stats) return fail(SE2GPU_ERR_CAPACITY, "window %d: max_iters > %d", k, h->max_stats);
    }
    const int device = hs[0]->device;
    SE2_CUDA(cudaSetDevice(device));
    // windows whose stop flag is already set do no iteration (as se2gpu_ba_optimize) and stay out of the launch
    std::vector<int> active;
    for (int k = 0; k < B; ++k) {
        if (iterations) iterations[k] = 0;
        if (max_iters > 0 && !(stop_flags && stop_flags[k] && *stop_flags[k])) active.push_back(k);
    }
    if (active.empty()) return SE2GPU_OK;
    for (int k : active) if (const int rc = check_cluster_size(device, batch_cluster_size(hs[k]))) return rc;
    // per window: trace capacity, the plan for its cluster, the abort word; then everything enqueued on its stream is waited
    // for, which orders the launch after it
    for (int k : active) {
        se2gpu_ba* h = hs[k];
        const bool tp = trace_poses && trace_poses[k], tl = trace_points && trace_points[k];
        if (tp && h->trace_cap_p < (size_t)max_iters * 3 * h->P) {
            h->trace_cap_p = 0;
            SE2_CUDA(h->bufs.regrow(&h->trace_p, (size_t)max_iters * 3 * h->P));
            h->trace_cap_p = (size_t)max_iters * 3 * h->P;
        }
        if (tl && h->trace_cap_l < (size_t)max_iters * 3 * h->L) {
            h->trace_cap_l = 0;
            SE2_CUDA(h->bufs.regrow(&h->trace_l, (size_t)max_iters * 3 * h->L));
            h->trace_cap_l = (size_t)max_iters * 3 * h->L;
        }
        if (const int rc = plan_for_grid(h, batch_cluster_size(h))) return rc;
        *h->abort_host = 0;
        SE2_CUDA(cudaStreamSynchronize(h->stream));
    }
    // descriptors grouped by cluster size, one launch per size present
    se2gpu_ba* h0 = hs[0];
    cudaStream_t s = h0->stream;
    std::vector<PKWindow> desc;
    desc.reserve(active.size());
    struct Group { int C, first, count; size_t smem; };
    std::vector<Group> groups;
    for (int C : {2, 4, 8}) {
        Group g{C, (int)desc.size(), 0, 0};
        for (int k : active) {
            se2gpu_ba* h = hs[k];
            if (batch_cluster_size(h) != C) continue;
            const size_t smem = pk_dyn_smem_bytes(h->d.n);     // the window's own arena: its Schur blocks are cached as on one context
            const bool tp = trace_poses && trace_poses[k], tl = trace_points && trace_points[k];
            PKArgs pa{max_iters, 0, h->stats_dev, tp ? h->trace_p : nullptr, tl ? h->trace_l : nullptr, h->abort_host_dev, h->abort_dev,
                      h->pk_part_chi, h->pk_part_scale, h->pk_part_max, nullptr, (int)smem, nullptr};
            desc.push_back(PKWindow{h->d, h->cam, pa});
            g.count++; g.smem = std::max(g.smem, smem);
        }
        if (g.count) groups.push_back(g);
    }
    const size_t words = desc.size() * sizeof(PKWindow) / 8;
    if (h0->bdesc_cap < words) {
        h0->bdesc_cap = 0;
        SE2_CUDA(h0->bufs.regrow(&h0->bdesc, words));
        h0->bdesc_cap = words;
    }
    h0->arena.reserve(words * 8 + 64);     // on failure the upload falls back to a pageable copy
    if (const int rc = h0->arena.up(h0->bdesc, reinterpret_cast<const unsigned long long*>(desc.data()), words, s)) return rc;
    const PKWindow* dev_desc = reinterpret_cast<const PKWindow*>(h0->bdesc);
    for (const Group& g : groups) {
        cudaLaunchAttribute attr{};
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = g.C; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(g.count * g.C); cfg.blockDim = dim3(PK_THREADS); cfg.dynamicSmemBytes = g.smem; cfg.stream = s;
        cfg.attrs = &attr; cfg.numAttrs = 1;
        const cudaError_t e = cudaLaunchKernelEx(&cfg, ba_persistent_cluster, dev_desc + g.first);
        if (e != cudaSuccess) {
            cudaStreamSynchronize(s);       // the launches already made finish before the error returns
            cudaGetLastError();
            return fail(SE2GPU_ERR_CUDA, "launch of the clusters of %d CTAs failed: %s", g.C, cudaGetErrorString(e));
        }
        se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    for (int k : active) SE2_CUDA(cudaMemcpyAsync(hs[k]->st_host, hs[k]->d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
    if (stop_flags) {   // the host forwards the stop flags while the windows run (setForceStopFlag)
        while (cudaStreamQuery(s) == cudaErrorNotReady)
            for (int k : active) if (stop_flags[k] && *stop_flags[k]) *(volatile int*)hs[k]->abort_host = 1;
    }
    SE2_CUDA(cudaStreamSynchronize(s));
    for (int k : active) {
        se2gpu_ba* h = hs[k];
        const int done = h->st_host->iter;
        if (iterations) iterations[k] = done;
        if (done <= 0) continue;
        if (stats) SE2_CUDA(cudaMemcpyAsync(stats + (size_t)k * max_iters, h->stats_dev, sizeof(se2gpu_ba_iter_stats) * done, cudaMemcpyDeviceToHost, s));
        if (trace_poses && trace_poses[k]) SE2_CUDA(cudaMemcpyAsync(trace_poses[k], h->trace_p, sizeof(double) * (size_t)done * 3 * h->P, cudaMemcpyDeviceToHost, s));
        if (trace_points && trace_points[k]) SE2_CUDA(cudaMemcpyAsync(trace_points[k], h->trace_l, sizeof(double) * (size_t)done * 3 * h->L, cudaMemcpyDeviceToHost, s));
    }
    SE2_CUDA(cudaStreamSynchronize(s));
    return SE2GPU_OK;
}

int se2gpu_ba_reset(se2gpu_ba* h) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    SE2_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (const int rc = reset_lm_state(h)) return rc;
    SE2_CUDA(cudaMemcpyAsync(h->d.xp[0], h->xp0, sizeof(double) * 3 * h->P, cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d.xl[0], h->xl0, sizeof(double) * 3 * h->L, cudaMemcpyDeviceToDevice, s));
    return SE2GPU_OK;
}

int se2gpu_ba_set_mode(se2gpu_ba* h, int mode) {
    if (!h || mode < 0 || mode > 2) return fail(SE2GPU_ERR_INVALID, "mode must be 0 (auto), 1 (multi-launch) or 2 (persistent)");
    h->mode = mode;
    return SE2GPU_OK;
}

int se2gpu_ba_profile(se2gpu_ba* h, int enable) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(h->device));
    h->prof.enable(enable != 0);
    h->pk_launches = 0;
    SE2_CUDA(cudaMemset(h->phase_cycles, 0, 8 * sizeof(long long)));
    return SE2GPU_OK;
}

int se2gpu_ba_profile_read(se2gpu_ba* h, double* ms, int* launches) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(h->device));
    h->prof.flush();
    for (int g = 0; g < SE2GPU_BA_PROFILE_GROUPS; ++g) { if (ms) ms[g] = h->prof.ms[g]; if (launches) launches[g] = h->prof.launches[g]; }
    if (h->pk_launches > 0) {
        // persistent mode: groups 0..6 are the in-kernel phase times of CTA 0 (SM cycles / nominal max clock), one "launch" per optimize()
        long long cyc[8];
        SE2_CUDA(cudaMemcpy(cyc, h->phase_cycles, sizeof cyc, cudaMemcpyDeviceToHost));
        for (int g = 0; g < 7; ++g) { if (ms) ms[g] = (double)cyc[g] / (double)(h->clock_khz > 0 ? h->clock_khz : FALLBACK_CLOCK_KHZ); if (launches) launches[g] = h->pk_launches; }
        if (ms) ms[8] = (double)cyc[7] / (double)(h->clock_khz > 0 ? h->clock_khz : FALLBACK_CLOCK_KHZ);
        if (launches) launches[8] = h->pk_launches;
    }
    return SE2GPU_OK;
}

int se2gpu_ba_get(se2gpu_ba* h, double* poses, double* points) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    SE2_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    SE2_CUDA(cudaMemcpyAsync(h->st_host, h->d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    const int cur = h->st_host->cur;
    if (poses) SE2_CUDA(cudaMemcpyAsync(poses, h->d.xp[cur], sizeof(double) * 3 * h->P, cudaMemcpyDeviceToHost, s));
    if (points) SE2_CUDA(cudaMemcpyAsync(points, h->d.xl[cur], sizeof(double) * 3 * h->L, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    return SE2GPU_OK;
}

int se2gpu_ba_get_f32(se2gpu_ba* h, float* poses, float* points) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    SE2_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    SE2_CUDA(cudaMemcpyAsync(h->st_host, h->d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    const int cur = h->st_host->cur;
    const int n = std::max(h->P, h->L);
    // narrow on the device into the context's float write-back buffer, then one copy per array
    float* fp = h->wb32;
    float* fl = fp + 3 * (size_t)h->P + 8;
    SE2_LAUNCH(ba_writeback_f32, (n + 255) / 256, 256, 0, s, h->d.xp[cur], h->P, h->d.xl[cur], h->L, poses ? fp : nullptr, points ? fl : nullptr);
    if (poses) SE2_CUDA(cudaMemcpyAsync(poses, fp, sizeof(float) * 3 * h->P, cudaMemcpyDeviceToHost, s));
    if (points) SE2_CUDA(cudaMemcpyAsync(points, fl, sizeof(float) * 3 * h->L, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    return SE2GPU_OK;
}

int se2gpu_ba_debug_system(se2gpu_ba* h, double lambda, double* chi2, double* Hpp, double* bp, double* Hll, double* bl,
                           double* Hpl, double* S, double* bs, double* dx_p, double* dx_l) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    if (h->world != 1) return fail(SE2GPU_ERR_INVALID, "debug_system is single-GPU only");
    SE2_CUDA(cudaSetDevice(h->device));
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    const int n = d.n, nf = d.nf, L = d.L, E = d.E;
    int rc = launch_linearize(h);
    if (rc != SE2GPU_OK) return rc;
    SE2_LAUNCH(ba_iter_begin, 1, 256, 0, s, d, 1, 0, 1);   // itg != 0: keeps lambda untouched, sets chi_cur
    SE2_CUDA(cudaMemcpyAsync(h->st_host, d.st, sizeof(LMState), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    LMState saved = *h->st_host;
    if (chi2) *chi2 = saved.chi_cur;
    h->st_host->lambda = lambda;
    SE2_CUDA(cudaMemcpyAsync(d.st, h->st_host, sizeof(LMState), cudaMemcpyHostToDevice, s));
    if ((rc = launch_schur(h)) != SE2GPU_OK) return rc;
    const size_t S_elems = stored_S_elems(h);
    const int u6[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};   // (row, column) of the 6 stored entries of a symmetric 3x3 block
    std::vector<double> tmp;
    auto get = [&](const double* dev, size_t cnt) { tmp.resize(cnt); return cudaMemcpyAsync(tmp.data(), dev, cnt * 8, cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess; };
    if (S) {
        if (!get(d.S, S_elems)) return fail(SE2GPU_ERR_CUDA, "copy S");
        if (!h->band.active) memcpy(S, tmp.data(), tmp.size() * 8);
        else {                         // band storage -> dense lower triangle
            const int bw = h->band.bw;
            memset(S, 0, sizeof(double) * (size_t)n * n);
            for (int r = 0; r < n; ++r) for (int c = std::max(0, r - bw); c <= r; ++c) S[(size_t)r * n + c] = tmp[(size_t)r * (bw + 1) + (c - r + bw)];
        }
    }
    if (bs) { if (!get(d.bs, n)) return fail(SE2GPU_ERR_CUDA, "copy bs"); memcpy(bs, tmp.data(), tmp.size() * 8); }
    if ((rc = launch_reduced_solve(h)) != SE2GPU_OK) return rc;
    SE2_LAUNCH(ba_backsub_update, h->nb_scale, LM_THREADS, 0, s, d);
    if (Hpp) {
        if (!get(d.Hpp, 6 * (size_t)nf)) return fail(SE2GPU_ERR_CUDA, "copy Hpp");
        // diagonal blocks only (off-diagonal odometry blocks are folded into S directly)
        memset(Hpp, 0, sizeof(double) * n * n);
        for (int a = 0; a < nf; ++a)
            for (int q = 0; q < 6; ++q) {
                Hpp[(size_t)(3 * a + u6[q][0]) * n + 3 * a + u6[q][1]] = tmp[q * (size_t)nf + a];
                Hpp[(size_t)(3 * a + u6[q][1]) * n + 3 * a + u6[q][0]] = tmp[q * (size_t)nf + a];
            }
    }
    if (bp) { if (!get(d.bp, n)) return fail(SE2GPU_ERR_CUDA, "copy bp"); memcpy(bp, tmp.data(), tmp.size() * 8); }
    if (Hll) {
        if (!get(d.Hll, 6 * (size_t)L)) return fail(SE2GPU_ERR_CUDA, "copy Hll");
        std::vector<int> lmp(L + 1);
        cudaMemcpy(lmp.data(), d.lm_ptr, sizeof(int) * (L + 1), cudaMemcpyDeviceToHost);
        for (int j = 0; j < L; ++j)
            for (int q = 0; q < 6; ++q) {
                double v = lmp[j + 1] > lmp[j] ? tmp[q * (size_t)L + j] : 0.0;
                Hll[9 * (size_t)j + u6[q][0] * 3 + u6[q][1]] = v; Hll[9 * (size_t)j + u6[q][1] * 3 + u6[q][0]] = v;
            }
    }
    if (bl) {
        if (!get(d.bl, 3 * (size_t)L)) return fail(SE2GPU_ERR_CUDA, "copy bl");
        std::vector<int> lmp(L + 1);
        cudaMemcpy(lmp.data(), d.lm_ptr, sizeof(int) * (L + 1), cudaMemcpyDeviceToHost);
        for (int j = 0; j < L; ++j) for (int q = 0; q < 3; ++q) bl[3 * (size_t)j + q] = lmp[j + 1] > lmp[j] ? tmp[q * (size_t)L + j] : 0.0;
    }
    if (Hpl) {
        if (!get(d.Hpl, EB * (size_t)E)) return fail(SE2GPU_ERR_CUDA, "copy Hpl");
        std::vector<int> eh(E);
        cudaMemcpy(eh.data(), d.e_hidx, sizeof(int) * E, cudaMemcpyDeviceToHost);
        std::vector<int> dperm;   // a device load keeps the landmark sort on the device only
        if (h->dl.valid) { dperm.resize(E); cudaMemcpy(dperm.data(), h->dl.perm, sizeof(int) * E, cudaMemcpyDeviceToHost); }
        const int* perm = h->dl.valid ? dperm.data() : h->perm.data();
        memset(Hpl, 0, sizeof(double) * 9 * (size_t)h->E);
        for (int k = 0; k < E; ++k) if (eh[k] >= 0) for (int q = 0; q < 9; ++q) Hpl[9 * (size_t)perm[k] + q] = tmp[(size_t)k * EB + q];
    }
    if (dx_p) { if (!get(d.dxp, n)) return fail(SE2GPU_ERR_CUDA, "copy dxp"); memcpy(dx_p, tmp.data(), tmp.size() * 8); }
    if (dx_l) { if (!get(d.dxl, 3 * (size_t)L)) return fail(SE2GPU_ERR_CUDA, "copy dxl"); memcpy(dx_l, tmp.data(), tmp.size() * 8); }
    // restore the LM scalars (estimates were never swapped: `cur` untouched)
    *h->st_host = saved;
    SE2_CUDA(cudaMemcpyAsync(d.st, h->st_host, sizeof(LMState), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    return n;
}

int se2gpu_ba_debug_plan(se2gpu_ba* h, int* out, int n_out) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    if (n_out < 0 || (n_out > 0 && !out)) return fail(SE2GPU_ERR_INVALID, "bad output buffer");
    for (int k = 0; k < std::min(n_out, SE2GPU_BA_PLAN_FIELDS); ++k) out[k] = h->plan[k];
    return SE2GPU_BA_PLAN_FIELDS;
}

}  // extern "C"
