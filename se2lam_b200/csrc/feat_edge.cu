// Feature-graph constraints: GlobalMapper::CreateFeatEdge (reference src/GlobalMapper.cpp:737-1032) and
// Sparsifier::DoMarginalizeSE3XYZ / InfoSE3 (src/sparsifier.cpp:59-274) for B keyframe pairs, one CTA each: the
// two-keyframe BA, the chi2 outlier cut, the marginalisation and the clamped information inside one kernel.
//
// What a pair is (DESIGN.md section 10): two g2o VertexSE3 (Isometry3D, camera-to-world, oplus = X * fromVectorMQT) with the
// EdgeSE3Prior of addVertexSE3PlaneMotion, one marginalised VertexPointXYZ per point with a Huber EdgeSE3PointXYZ to each
// keyframe, optimised by OptimizationAlgorithmLevenberg over BlockSolver's Schur complement. Everything is double precision.
//
// Per CTA: a thread owns the points tid, tid + 128, ...: a point's two edges, its Hll, its Hpl blocks, Hll^-1, its Schur
// contribution and its back-substitution never leave that thread. The reduced system (12 x 12 when both keyframes are free)
// is summed block by block, one 6 x 6 block per pass over the points, each pass recomputing the point's linearisation; a
// pass is a warp xor-shuffle tree and then the 4 warp sums in index order (no atomics: bit-reproducible, independent of the
// CTA's position in the batch). Thread 0 adds the priors, damps, factorises (LL^T), applies oplus, and runs InfoSE3.
// The marginalisation is the same thread-per-point Schur pass over the reference's forward-difference Jacobians: H22 is
// block diagonal, so H11 - H12 H22^-1 H21 is a sum over points and the (12 + 3N)^2 matrix is never formed. The matrix given
// to the reference's SVD is symmetric, so its singular-value clamp is applied to the eigenvalues of a cyclic Jacobi
// eigen-decomposition: f(l) = clamp(l, 1e-6, 1e4) for l >= 0 and 1e-6 for l < 0.
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstring>

#include "common.h"
#include "lm.h"
#include "se3iso.h"

using namespace se2gpu;

namespace {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kStageMax = 192;  // points whose measurements are staged in shared memory: 168 B each, 31.5 KB
constexpr int kRed = 36;        // widest reduction: the 6 x 6 off-diagonal block

struct Params {
    float Tbc[16];
    float xrot, yrot, zinfo;
    double delta, cut;
    int iterations, min_points, mode;
};

// the measurements of one CTA's points: z [P*3] float and Omega [P*9] double per keyframe
struct Meas {
    const float* z[2];
    const double* om[2];
};

__device__ inline void se3_map(const SE3& T, const double* p, double* out) {
    qrot(T.q, p, out);
    for (int i = 0; i < 3; ++i) out[i] += T.t[i];
}

// SE3Quat::fromMinimalVector of toMinimalVector() = (t, qx, qy, qz) with delta added to entry i
__device__ SE3 se3_perturbed(const SE3& T, int i, double delta) {
    double v[6] = {T.t[0], T.t[1], T.t[2], T.q.x, T.q.y, T.q.z};
    v[i] += delta;
    SE3 r;
    const double w = 1. - v[3] * v[3] - v[4] * v[4] - v[5] * v[5];
    if (w > 0) r.q = {v[3], v[4], v[5], sqrt(w)};
    else r.q = {-v[3], -v[4], -v[5], 0};
    r.t[0] = v[0]; r.t[1] = v[1]; r.t[2] = v[2];
    return r;
}

// Eigen's fixed-size 3 x 3 inverse: cofactors over the determinant
__device__ inline void inv3(const double* m, double* o) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02, id = 1. / det;
    o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = c01 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = c02 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// 2 skew(pc)^T M for a 3 x N matrix M: the rotational rows of Jp^T M, Jp = [-I | 2 skew(pc)]
template <int N>
__device__ inline void skew2t_mul(const double* pc, const double* M, double* out) {
#pragma unroll
    for (int c = 0; c < N; ++c) {
        out[c] = 2 * (pc[2] * M[N + c] - pc[1] * M[2 * N + c]);
        out[N + c] = 2 * (-pc[2] * M[c] + pc[0] * M[2 * N + c]);
        out[2 * N + c] = 2 * (pc[1] * M[c] - pc[0] * M[N + c]);
    }
}

// one EdgeSE3PointXYZ at (Xi = X^-1, p): e = Xi p - z, the robust chi2 into chi (the plain one returned), and with LIN the
// weighted pieces W = rho' Omega, W e, W Jl (Jl = Xi.R), and the point's Hll / bl contributions
template <bool LIN>
__device__ inline double edge_eval(const Iso& Xi, const double* p, const float* zf, const double* Om, double delta, double& chi,
                                   double* pc, double* W, double* We, double* WJl, double* Hll, double* bl) {
    double e[3], Oe[3];
    mulv3(Xi.R, p, pc);
#pragma unroll
    for (int i = 0; i < 3; ++i) { pc[i] += Xi.t[i]; e[i] = pc[i] - (double)zf[i]; }
    mulv3(Om, e, Oe);
    const double c2 = e[0] * Oe[0] + e[1] * Oe[1] + e[2] * Oe[2];
    const double dsqr = delta * delta;
    const bool inlier = c2 <= dsqr;
    const double sq = inlier ? 0.0 : sqrt(c2);
    chi += inlier ? c2 : 2 * sq * delta - dsqr;
    if (!LIN) return c2;
    const double rho1 = inlier ? 1.0 : delta / sq;
#pragma unroll
    for (int i = 0; i < 9; ++i) W[i] = rho1 * Om[i];
    mulv3(W, e, We);
    mul3(W, Xi.R, WJl);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) Hll[r * 3 + c] += Xi.R[r] * WJl[c] + Xi.R[3 + r] * WJl[3 + c] + Xi.R[6 + r] * WJl[6 + c];
        bl[r] -= Xi.R[r] * We[0] + Xi.R[3 + r] * We[1] + Xi.R[6 + r] * We[2];
    }
    return c2;
}

// the pose-side blocks of one edge: Hpl = Jp^T W Jl (6 x 3); with DIAG the upper triangle of Jp^T W Jp into Hpp [21] and
// -Jp^T W e into bp [6] (added)
template <bool DIAG>
__device__ inline void edge_pose_blocks(const double* pc, const double* W, const double* We, const double* WJl, double* Hpl,
                                        double* Hpp, double* bp) {
#pragma unroll
    for (int k = 0; k < 9; ++k) Hpl[k] = -WJl[k];
    skew2t_mul<3>(pc, WJl, Hpl + 9);
    if (!DIAG) return;
    // W Jp = [-W | W S], S = 2 skew(pc)
    double WS[9], RR[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        WS[r * 3] = 2 * (W[r * 3 + 1] * pc[2] - W[r * 3 + 2] * pc[1]);
        WS[r * 3 + 1] = 2 * (-W[r * 3] * pc[2] + W[r * 3 + 2] * pc[0]);
        WS[r * 3 + 2] = 2 * (W[r * 3] * pc[1] - W[r * 3 + 1] * pc[0]);
    }
    skew2t_mul<3>(pc, WS, RR);
    // upper triangle, row-major: rows 0-2 = -(W Jp) = [W | -W S], rows 3-5 (columns 3-5 only) = S^T W S
    int k = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = r; c < 3; ++c) Hpp[k++] += W[r * 3 + c];
#pragma unroll
        for (int c = 0; c < 3; ++c) Hpp[k++] += -WS[r * 3 + c];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c) Hpp[k++] += RR[r * 3 + c];
    double rb[3];
    skew2t_mul<1>(pc, We, rb);
#pragma unroll
    for (int r = 0; r < 3; ++r) { bp[r] -= -We[r]; bp[3 + r] -= rb[r]; }
}

enum Pass { kBlock00 = 0, kBlock11 = 1, kBlock01 = 2, kBackSub = 3, kDiag = 4 };

// One point's share of one pass over the BA system at damping lambda.
//  kBlock00 / kBlock11: acc[0..20] the upper triangle of the keyframe's reduced 6 x 6 block, acc[21..26] its reduced b,
//                       acc[28..33] its unreduced b (computeScale uses that one); kBlock11 also adds the robust chi2 of
//                       both edges into acc[27]
//  kBlock01:            acc[0..35] the reduced off-diagonal block (rows keyframe 0, columns keyframe 1)
//  kBackSub:            xl = Hll^-1 (bl - Hpl^T xp) into xl [3], x (lambda x + b) of the point into acc[0]
//  kDiag:               acc[0..5] / acc[6..11] the diagonals of Jp^T W Jp of keyframe 0 / 1, acc[12] = max |Hll(i, i)|
template <int PASS>
__device__ __noinline__ void point_pass(const Iso* Xi, const double* p, const Meas& m, int j, double delta, double lambda, bool free0,
                                  const double* xp, double* acc, double* xl) {
    double Hll[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bl[3] = {0, 0, 0};
    double Hpl0[18], Hpl1[18], Hpp[21], bp[6], chi = 0;
#pragma unroll
    for (int k = 0; k < 21; ++k) Hpp[k] = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) bp[k] = 0;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        double pc[3], W[9], We[3], WJl[9];
        edge_eval<true>(Xi[k], p, m.z[k] + 3 * (size_t)j, m.om[k] + 9 * (size_t)j, delta, chi, pc, W, We, WJl, Hll, bl);
        const bool want_diag = (PASS == kBlock00 && k == 0) || (PASS == kBlock11 && k == 1) || PASS == kDiag;
        double* Hpl = k ? Hpl1 : Hpl0;
        if (PASS == kDiag) {
            double H[21], b6[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int i = 0; i < 21; ++i) H[i] = 0;
            edge_pose_blocks<true>(pc, W, We, WJl, Hpl, H, b6);
            const int dg[6] = {0, 6, 11, 15, 18, 20};
#pragma unroll
            for (int i = 0; i < 6; ++i) acc[6 * k + i] += H[dg[i]];
        } else if (want_diag) {
            edge_pose_blocks<true>(pc, W, We, WJl, Hpl, Hpp, bp);
        } else {
            edge_pose_blocks<false>(pc, W, We, WJl, Hpl, nullptr, nullptr);
        }
    }
    if (PASS == kDiag) {
        acc[12] = fmax(acc[12], fmax(fabs(Hll[0]), fmax(fabs(Hll[4]), fabs(Hll[8]))));
        return;
    }
    double D[9], Di[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) D[i] = Hll[i] + (i % 4 == 0 ? lambda : 0.0);
    inv3(D, Di);
    if (PASS == kBlock00 || PASS == kBlock11) {
        const double* Hpl = PASS == kBlock00 ? Hpl0 : Hpl1;
        double yb[3];
        mulv3(Di, bl, yb);
        int k = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r) {
            double Y[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) Y[c] = Hpl[r * 3] * Di[c] + Hpl[r * 3 + 1] * Di[3 + c] + Hpl[r * 3 + 2] * Di[6 + c];
#pragma unroll
            for (int c = r; c < 6; ++c, ++k)
                acc[k] += Hpp[k] - (Y[0] * Hpl[c * 3] + Y[1] * Hpl[c * 3 + 1] + Y[2] * Hpl[c * 3 + 2]);
            acc[21 + r] += bp[r] - (Hpl[r * 3] * yb[0] + Hpl[r * 3 + 1] * yb[1] + Hpl[r * 3 + 2] * yb[2]);
            acc[28 + r] += bp[r];
        }
        if (PASS == kBlock11) acc[27] += chi;
    } else if (PASS == kBlock01) {
#pragma unroll
        for (int r = 0; r < 6; ++r) {
            double Y[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) Y[c] = Hpl0[r * 3] * Di[c] + Hpl0[r * 3 + 1] * Di[3 + c] + Hpl0[r * 3 + 2] * Di[6 + c];
#pragma unroll
            for (int c = 0; c < 6; ++c) acc[r * 6 + c] -= Y[0] * Hpl1[c * 3] + Y[1] * Hpl1[c * 3 + 1] + Y[2] * Hpl1[c * 3 + 2];
        }
    } else {  // kBackSub
        double rhs[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double a = bl[c];
            if (free0)
#pragma unroll
                for (int r = 0; r < 6; ++r) a -= Hpl0[r * 3 + c] * xp[r];
#pragma unroll
            for (int r = 0; r < 6; ++r) a -= Hpl1[r * 3 + c] * xp[6 + r];
            rhs[c] = a;
        }
        mulv3(Di, rhs, xl);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[0] += xl[c] * (lambda * xl[c] + bl[c]);
    }
}

// Sparsifier::JacobianSE3XYZ + HessianSE3XYZ of one point against keyframe k: J^T Omega J split into the pose block PP
// (upper triangle, 21), the pose-point block PL (6 x 3) and the point block LL (3 x 3, added). KFi = KF^-1, KFdi [6] the
// inverses of the six perturbed keyframes.
__device__ inline void marg_edge(const SE3& KFi, const SE3* KFdi, const double* MP, const double* Om, double* PP, double* PL,
                                 double* LL) {
    const double delta = 1e-6;
    double zref[3], J[27];
    se3_map(KFi, MP, zref);
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        double zd[3];
        if (i < 6) {
            se3_map(KFdi[i], MP, zd);
        } else {
            double mp[3] = {MP[0], MP[1], MP[2]};
            mp[i - 6] += delta;
            se3_map(KFi, mp, zd);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) J[r * 9 + i] = (zd[r] - zref[r]) / delta;
    }
    double OJ[27];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 9; ++c) OJ[r * 9 + c] = Om[r * 3] * J[c] + Om[r * 3 + 1] * J[9 + c] + Om[r * 3 + 2] * J[18 + c];
    int k = 0;
#pragma unroll
    for (int r = 0; r < 9; ++r)
#pragma unroll
        for (int c = 0; c < 9; ++c) {
            const double h = J[r] * OJ[c] + J[9 + r] * OJ[9 + c] + J[18 + r] * OJ[18 + c];
            if (r < 6 && c < 6) { if (c >= r && PP) PP[k++] = h; }
            else if (r >= 6 && c >= 6) LL[(r - 6) * 3 + c - 6] += h;
            else if (r < 6) PL[r * 3 + c - 6] = h;
        }
}

// one point's share of H11 - H12 H22^-1 H21: kBlock00 / kBlock11 the upper triangle of a diagonal block into acc[0..20],
// kBlock01 the off-diagonal block into acc[0..35]
template <int PASS>
__device__ __noinline__ void marg_pass(const SE3* KFi, const SE3 (*KFdi)[6], const double* MP, const Meas& m, int j, double* acc) {
    double LL[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, PL0[18], PL1[18], PP[21], Di[9];
    marg_edge(KFi[0], KFdi[0], MP, m.om[0] + 9 * (size_t)j, PASS == kBlock00 ? PP : nullptr, PL0, LL);
    marg_edge(KFi[1], KFdi[1], MP, m.om[1] + 9 * (size_t)j, PASS == kBlock11 ? PP : nullptr, PL1, LL);
    inv3(LL, Di);
    const double* A = PASS == kBlock11 ? PL1 : PL0;
    const double* Bm = PASS == kBlock00 ? PL0 : PL1;
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        double Y[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) Y[c] = A[r * 3] * Di[c] + A[r * 3 + 1] * Di[3 + c] + A[r * 3 + 2] * Di[6 + c];
        if (PASS == kBlock01) {
#pragma unroll
            for (int c = 0; c < 6; ++c) acc[r * 6 + c] -= Y[0] * Bm[c * 3] + Y[1] * Bm[c * 3 + 1] + Y[2] * Bm[c * 3 + 2];
        } else {
#pragma unroll
            for (int c = r; c < 6; ++c, ++k) acc[k] += PP[k] - (Y[0] * Bm[c * 3] + Y[1] * Bm[c * 3 + 1] + Y[2] * Bm[c * 3 + 2]);
        }
    }
}

// inverse by LU with partial pivoting (what Eigen's inverse() does above 4 x 4); M is destroyed
__device__ void lu_inverse(int n, double* M, double* inv) {
    for (int i = 0; i < n * n; ++i) inv[i] = 0;
    for (int i = 0; i < n; ++i) inv[i * n + i] = 1;
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int r = c + 1; r < n; ++r)
            if (fabs(M[r * n + c]) > fabs(M[piv * n + c])) piv = r;
        if (piv != c)
            for (int k = 0; k < n; ++k) {
                double t = M[c * n + k]; M[c * n + k] = M[piv * n + k]; M[piv * n + k] = t;
                t = inv[c * n + k]; inv[c * n + k] = inv[piv * n + k]; inv[piv * n + k] = t;
            }
        const double d = M[c * n + c];
        for (int r = c + 1; r < n; ++r) {
            const double f = M[r * n + c] / d;
            for (int k = c; k < n; ++k) M[r * n + k] -= f * M[c * n + k];
            for (int k = 0; k < n; ++k) inv[r * n + k] -= f * inv[c * n + k];
        }
    }
    for (int c = n - 1; c >= 0; --c) {
        const double d = M[c * n + c];
        for (int k = 0; k < n; ++k) inv[c * n + k] /= d;
        for (int r = 0; r < c; ++r) {
            const double f = M[r * n + c];
            for (int k = 0; k < n; ++k) inv[r * n + k] -= f * inv[c * n + k];
        }
    }
}

// cyclic Jacobi eigen-decomposition of the symmetric 6 x 6 A (destroyed: its diagonal becomes the eigenvalues), V the vectors
__device__ void jacobi_eig6(double* A, double* V) {
    for (int i = 0; i < 36; ++i) V[i] = (i % 7 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0, dg = 0;
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) (r == c ? dg : off) += A[r * 6 + c] * A[r * 6 + c];
        if (off <= 1e-32 * dg) break;
        for (int p = 0; p < 5; ++p)
            for (int q = p + 1; q < 6; ++q) {
                const double apq = A[p * 6 + q];
                if (apq == 0) continue;
                const double theta = (A[q * 6 + q] - A[p * 6 + p]) / (2 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(1 + theta * theta));
                const double c = 1 / sqrt(1 + t * t), s = c * t;
                for (int k = 0; k < 6; ++k) {
                    const double akp = A[k * 6 + p], akq = A[k * 6 + q];
                    A[k * 6 + p] = c * akp - s * akq; A[k * 6 + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 6; ++k) {
                    const double apk = A[p * 6 + k], aqk = A[q * 6 + k];
                    A[p * 6 + k] = c * apk - s * aqk; A[q * 6 + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 6; ++k) {
                    const double vkp = V[k * 6 + p], vkq = V[k * 6 + q];
                    V[k * 6 + p] = c * vkp - s * vkq; V[k * 6 + q] = s * vkp + c * vkq;
                }
            }
    }
}

// Sparsifier::InfoSE3 (:219-274) on one thread. Hm [144] = H_marginal (destroyed); w [432] doubles of scratch; I [36] out.
__device__ __noinline__ void info_se3(const SE3& K1, const SE3& K2, double* Hm, double* w, double* I) {
    double* J = w;            // 6 x 12
    double* Hinv = w + 72;    // 12 x 12
    double* JH = w + 216;     // 6 x 12
    double* C = w + 288;      // 6 x 6
    double* V = w + 324;      // 6 x 6
    double* S = w + 360;      // 6 x 6
    const double delta = 1e-6;
    const SE3 K1i = se3_inv(K1);
    const SE3 zr = se3_mul(K1i, K2);
    const double zref[6] = {zr.t[0], zr.t[1], zr.t[2], zr.q.x, zr.q.y, zr.q.z};
    for (int i = 0; i < 12; ++i) {  // JacobianSE3: forward differences on toMinimalVector / fromMinimalVector
        const SE3 Kd = se3_perturbed(i < 6 ? K1 : K2, i % 6, delta);
        const SE3 zd = i < 6 ? se3_mul(se3_inv(Kd), K2) : se3_mul(K1i, Kd);
        const double z6[6] = {zd.t[0], zd.t[1], zd.t[2], zd.q.x, zd.q.y, zd.q.z};
        for (int r = 0; r < 6; ++r) J[r * 12 + i] = (z6[r] - zref[r]) / delta;
    }
    lu_inverse(12, Hm, Hinv);
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 12; ++c) {
            double acc = 0;
            for (int k = 0; k < 12; ++k) acc += J[r * 12 + k] * Hinv[k * 12 + c];
            JH[r * 12 + c] = acc;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 12; ++k) acc += JH[r * 12 + k] * J[c * 12 + k];
            C[r * 6 + c] = acc;
        }
    lu_inverse(6, C, S);
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) C[r * 6 + c] = (S[r * 6 + c] + S[c * 6 + r]) / 2;
    jacobi_eig6(C, V);
    double f[6];
    for (int i = 0; i < 6; ++i) {
        const double l = C[i * 7];
        f[i] = l >= 0 ? fmin(fmax(l, 1e-6), 1e4) : 1e-6;
    }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double acc = 0;
            for (int k = 0; k < 6; ++k) acc += (V[r * 6 + k] * f[k]) * V[c * 6 + k];
            S[r * 6 + c] = acc;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) I[r * 6 + c] = (S[r * 6 + c] + S[c * 6 + r]) / 2;
}

__global__ void __launch_bounds__(kThreads) k_feat_edge(const float* __restrict__ Tcw0, const float* __restrict__ Tcw1,
                                                        const int* __restrict__ point_ptr, const float* __restrict__ xyz,
                                                        const float* __restrict__ z0, const float* __restrict__ z1,
                                                        const double* __restrict__ info0, const double* __restrict__ info1, Params p,
                                                        float* __restrict__ measure, float* __restrict__ info,
                                                        int* __restrict__ status, int* __restrict__ iters,
                                                        se2gpu_ba_iter_stats* __restrict__ stats, uint8_t* __restrict__ outlier,
                                                        double* __restrict__ poses, double* __restrict__ points,
                                                        double* __restrict__ work, double* __restrict__ trace) {
    extern __shared__ double s_stage[];  // [2][kStageMax*9] Omega, then [2][kStageMax*3] z as float
    __shared__ double s_red[kWarps][kRed];
    __shared__ double s_sum[3][kRed];    // the reduced blocks 00 (+ b0), 11 (+ b1 + chi2), 01
    __shared__ double s_H[144], s_b[12], s_xp[12], s_w[432];
    __shared__ double s_Hprior[2][36], s_bprior[2][6];
    __shared__ Prior s_prior[2];
    __shared__ Iso s_X[2], s_trial[2];
    __shared__ SE3 s_KFi[2], s_KFdi[2][6], s_KF[2];
    __shared__ double s_cur, s_lambda, s_ni, s_pchi;
    __shared__ int s_ok2, s_more, s_stop, s_accept, s_last_trial;

    const int pb = blockIdx.x, tid = threadIdx.x;
    const int j0 = point_ptr[pb], P = point_ptr[pb + 1] - j0;
    if (P < p.min_points) {
        if (tid == 0) {
            if (iters) iters[pb] = 0;
            if (status) status[pb] = SE2GPU_FEAT_EDGE_TOO_FEW;
        }
        return;
    }
    const bool free0 = p.mode != 0;
    Meas m = {{z0 + 3 * (size_t)j0, z1 + 3 * (size_t)j0}, {info0 + 9 * (size_t)j0, info1 + 9 * (size_t)j0}};
    double* pts = points + 3 * (size_t)j0;
    double* wrk = work + 3 * (size_t)j0;
    if (P <= kStageMax) {
        float* sz = reinterpret_cast<float*>(s_stage + 18 * kStageMax);
        for (int k = 0; k < 2; ++k) {
            for (int i = tid; i < 9 * P; i += kThreads) s_stage[k * 9 * kStageMax + i] = m.om[k][i];
            for (int i = tid; i < 3 * P; i += kThreads) sz[k * 3 * kStageMax + i] = m.z[k][i];
        }
        m.om[0] = s_stage; m.om[1] = s_stage + 9 * kStageMax;
        m.z[0] = sz; m.z[1] = sz + 3 * kStageMax;
    }
    for (int i = tid; i < 3 * P; i += kThreads) pts[i] = (double)xyz[3 * (size_t)j0 + i];
    if (tid == 0) {
        s_X[0] = iso_from_Tcw(Tcw0 + 16 * (size_t)pb);
        s_X[1] = iso_from_Tcw(Tcw1 + 16 * (size_t)pb);
        for (int k = free0 ? 0 : 1; k < 2; ++k) plane_motion_prior(s_X[k], p.Tbc, p.xrot, p.yrot, p.zinfo, &s_prior[k]);
        s_stop = 0;
        s_last_trial = 0;  // with iterations = 0 the outlier cut reads the start estimate
    }
    __syncthreads();

    int it = 0, last_failed = 0;
    for (; it < p.iterations; ++it) {
        Iso Xi[2] = {iso_inv(s_X[0]), iso_inv(s_X[1])};
        if (tid == 0) {  // the priors' share of H, b and chi2 at the current estimate
            s_pchi = 0;
            for (int k = free0 ? 0 : 1; k < 2; ++k) s_pchi += prior_terms(s_prior[k], s_X[k], s_Hprior[k], s_bprior[k]);
            s_last_trial = 0;
        }
        if (it == 0) {  // computeLambdaInit over every free vertex
            double acc[13];
#pragma unroll
            for (int k = 0; k < 13; ++k) acc[k] = 0;
            for (int j = tid; j < P; j += kThreads) point_pass<kDiag>(Xi, pts + 3 * j, m, j, p.delta, 0.0, free0, nullptr, acc, nullptr);
            const double hmax = acc[12];
            cta_sum<12>(acc, s_red, s_sum[0]);
            double mx = cta_max(hmax, s_red);
            if (tid == 0) {
                for (int k = free0 ? 0 : 1; k < 2; ++k)
                    for (int i = 0; i < 6; ++i) mx = fmax(mx, fabs(s_sum[0][6 * k + i] + s_Hprior[k][i * 7]));
                lm_lambda_init(mx, s_lambda, s_ni);
            }
            __syncthreads();
        }
        // the iteration's stats live in st from here on: with chi2_before in a scalar instead, nvcc 12.9 contracts the
        // quat_to_R of iso_from_Tcw(Tcw0) above differently (another FMA), and the start rotation changes by an ulp
        se2gpu_ba_iter_stats st{};
        int qmax = 0, failed = 0, accepted = 0;
        double rho = 0;
        for (;;) {
            __syncthreads();
            const double lambda = s_lambda;
            {   // the Schur complement at this damping, block by block
                double acc[kRed];
#pragma unroll
                for (int k = 0; k < 34; ++k) acc[k] = 0;
                for (int j = tid; j < P; j += kThreads) point_pass<kBlock11>(Xi, pts + 3 * j, m, j, p.delta, lambda, free0, nullptr, acc, nullptr);
                cta_sum<34>(acc, s_red, s_sum[1]);
                if (free0) {
#pragma unroll
                    for (int k = 0; k < 34; ++k) acc[k] = 0;
                    for (int j = tid; j < P; j += kThreads) point_pass<kBlock00>(Xi, pts + 3 * j, m, j, p.delta, lambda, free0, nullptr, acc, nullptr);
                    cta_sum<34>(acc, s_red, s_sum[0]);
#pragma unroll
                    for (int k = 0; k < 36; ++k) acc[k] = 0;
                    for (int j = tid; j < P; j += kThreads) point_pass<kBlock01>(Xi, pts + 3 * j, m, j, p.delta, lambda, free0, nullptr, acc, nullptr);
                    cta_sum<36>(acc, s_red, s_sum[2]);
                }
            }
            double scale = 0;
            if (tid == 0) {
                if (qmax == 0) { s_cur = s_sum[1][27] + s_pchi; st.chi2_before = s_cur; }
                const int n = free0 ? 12 : 6, o1 = free0 ? 6 : 0;
                for (int i = 0; i < 144; ++i) s_H[i] = 0;
                for (int kf = free0 ? 0 : 1; kf < 2; ++kf) {
                    const int o = kf ? o1 : 0;
                    int k = 0;
                    for (int r = 0; r < 6; ++r) {
                        for (int c = r; c < 6; ++c, ++k) {
                            const double h = s_sum[kf][k] + s_Hprior[kf][r * 6 + c] + (r == c ? lambda : 0.0);
                            s_H[(o + r) * 12 + o + c] = h;
                            s_H[(o + c) * 12 + o + r] = h;
                        }
                        s_b[o + r] = s_sum[kf][21 + r] + s_bprior[kf][r];
                    }
                }
                if (free0)
                    for (int r = 0; r < 6; ++r)
                        for (int c = 0; c < 6; ++c) { s_H[r * 12 + 6 + c] = s_sum[2][r * 6 + c]; s_H[(6 + c) * 12 + r] = s_sum[2][r * 6 + c]; }
                double x[12];
                const bool ok2 = chol_factor(n, 12, s_H);
                if (ok2) chol_solve(n, 12, s_H, s_b, x);
                s_ok2 = ok2;
                for (int i = 0; i < 12; ++i) s_xp[i] = 0;
                double sp = 0;
                if (ok2) {
                    for (int i = 0; i < n; ++i) s_xp[(free0 ? 0 : 6) + i] = x[i];
                    s_trial[0] = free0 ? oplus(s_X[0], s_xp) : s_X[0];
                    s_trial[1] = oplus(s_X[1], s_xp + 6);
                    for (int kf = free0 ? 0 : 1; kf < 2; ++kf)  // computeScale over the poses, with the unreduced b
                        for (int r = 0; r < 6; ++r) sp += s_xp[6 * kf + r] * (lambda * s_xp[6 * kf + r] + (s_sum[kf][28 + r] + s_bprior[kf][r]));
                }
                s_w[0] = sp;
            }
            __syncthreads();
            double temp = DBL_MAX;
            if (s_ok2) {
                // back-substitution, the trial points, the robust chi2 at the trial state and the points' share of computeScale
                const Iso Ti[2] = {iso_inv(s_trial[0]), iso_inv(s_trial[1])};
                double a[3] = {0, 0, 0};
                for (int j = tid; j < P; j += kThreads) {
                    double xl[3], pt[3], sc[1] = {0};
                    point_pass<kBackSub>(Xi, pts + 3 * j, m, j, p.delta, lambda, free0, s_xp, sc, xl);
                    a[1] += sc[0];
#pragma unroll
                    for (int c = 0; c < 3; ++c) { pt[c] = pts[3 * j + c] + xl[c]; wrk[3 * j + c] = pt[c]; }
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        double pc[3];
                        edge_eval<false>(Ti[k], pt, m.z[k] + 3 * (size_t)j, m.om[k] + 9 * (size_t)j, p.delta, a[0], pc, nullptr, nullptr,
                                         nullptr, nullptr, nullptr);
                    }
                }
                double tot[3];
                cta_sum<2>(a, s_red, tot);
                if (tid == 0) {
                    double pchi = 0;
                    for (int k = free0 ? 0 : 1; k < 2; ++k) pchi += prior_terms(s_prior[k], s_trial[k], nullptr, nullptr);
                    temp = tot[0] + pchi;
                    scale = tot[1] + s_w[0];
                    s_last_trial = 1;
                }
            }
            if (tid == 0) {
                if (!s_ok2) ++failed;
                s_accept = lm_gain_step(temp, scale, s_ok2, s_cur, s_lambda, s_ni, rho);
                if (s_accept) { s_X[0] = s_trial[0]; s_X[1] = s_trial[1]; accepted = 1; }
                ++qmax;
                s_more = lm_retry(rho, qmax);
            }
            __syncthreads();
            if (s_accept)
                for (int j = tid; j < P; j += kThreads)
#pragma unroll
                    for (int c = 0; c < 3; ++c) pts[3 * j + c] = wrk[3 * j + c];
            if (!s_more) break;
        }
        if (tid == 0) {
            st = lm_iter_stats(st.chi2_before, s_cur, s_lambda, rho, qmax, accepted);
            last_failed = lm_not_pd(st, failed);
            if (stats) stats[(size_t)pb * p.iterations + it] = st;
            if (trace)
                for (int k = 0; k < 2; ++k) {
                    double* t = trace + ((size_t)pb * p.iterations + it) * 24 + 12 * k;
                    for (int i = 0; i < 9; ++i) t[i] = s_X[k].R[i];
                    for (int i = 0; i < 3; ++i) t[9 + i] = s_X[k].t[i];
                }
            s_stop = st.terminate;
        }
        __syncthreads();
        if (s_stop) { ++it; break; }
    }

    // OptKFPairMatch's outlier cut: EdgeSE3PointXYZ::chi2() holds the error of the last evaluated trial, accepted or not
    __syncthreads();
    if (tid < 12) {
        const int k = tid / 6, i = tid % 6;
        const SE3 KF = se3_from_iso(s_X[k]);
        s_KFdi[k][i] = se3_inv(se3_perturbed(KF, i, 1e-6));
        if (i == 0) { s_KF[k] = KF; s_KFi[k] = se3_inv(KF); }
    }
    uint8_t* out = outlier ? outlier + j0 : nullptr;
    const Iso Li[2] = {iso_inv(s_last_trial ? s_trial[0] : s_X[0]), iso_inv(s_last_trial ? s_trial[1] : s_X[1])};
    const double* lastp = s_last_trial ? wrk : pts;
    __syncthreads();
    // the marginalisation over the surviving points, block by block
    for (int pass = 0; pass < 3; ++pass) {
        double acc[kRed];
#pragma unroll
        for (int k = 0; k < kRed; ++k) acc[k] = 0;
        for (int j = tid; j < P; j += kThreads) {
            bool is_out = false;
            if (p.mode == 1) {
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    double pc[3], chi = 0;
                    const double c2 = edge_eval<false>(Li[k], lastp + 3 * j, m.z[k] + 3 * (size_t)j, m.om[k] + 9 * (size_t)j, p.delta, chi, pc,
                                                       nullptr, nullptr, nullptr, nullptr, nullptr);
                    if (c2 > p.cut) is_out = true;
                }
            }
            if (pass == 0 && out) out[j] = is_out;
            if (is_out) continue;
            if (pass == 0) marg_pass<kBlock00>(s_KFi, s_KFdi, pts + 3 * j, m, j, acc);
            else if (pass == 1) marg_pass<kBlock11>(s_KFi, s_KFdi, pts + 3 * j, m, j, acc);
            else marg_pass<kBlock01>(s_KFi, s_KFdi, pts + 3 * j, m, j, acc);
        }
        if (pass < 2) cta_sum<21>(acc, s_red, s_sum[pass]);
        else cta_sum<36>(acc, s_red, s_sum[2]);
    }
    __syncthreads();
    if (tid == 0) {
        for (int kf = 0; kf < 2; ++kf) {
            int k = 0;
            for (int r = 0; r < 6; ++r)
                for (int c = r; c < 6; ++c, ++k) {
                    const double h = s_sum[kf][k] + (r == c ? 1e-6 : 0.0);
                    s_H[(6 * kf + r) * 12 + 6 * kf + c] = h;
                    s_H[(6 * kf + c) * 12 + 6 * kf + r] = h;
                }
        }
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) { s_H[r * 12 + 6 + c] = s_sum[2][r * 6 + c]; s_H[(6 + c) * 12 + r] = s_sum[2][r * 6 + c]; }
        double I[36];
        info_se3(s_KF[0], s_KF[1], s_H, s_w, I);
        se3_to_f32(se3_mul(s_KFi[0], s_KF[1]), measure + 16 * (size_t)pb);
        for (int i = 0; i < 36; ++i) info[36 * (size_t)pb + i] = (float)I[i];
        if (iters) iters[pb] = it;
        if (status) status[pb] = last_failed ? SE2GPU_FEAT_EDGE_NOT_PD : SE2GPU_FEAT_EDGE_OK;
        if (poses) { store_pose(s_KF[0], poses + 14 * (size_t)pb); store_pose(s_KF[1], poses + 14 * (size_t)pb + 7); }
    }
}


int check_params(const se2gpu_feat_edge_params* prm, int mode, Params* p) {
    if (!prm) return fail(SE2GPU_ERR_INVALID, "null parameters");
    if (mode != 0 && mode != 1) return fail(SE2GPU_ERR_INVALID, "mode = %d", mode);
    if (prm->iterations[mode] < 0) return fail(SE2GPU_ERR_INVALID, "iterations = %d", prm->iterations[mode]);
    if (prm->min_points[mode] < 1) return fail(SE2GPU_ERR_INVALID, "min_points = %d", prm->min_points[mode]);
    std::memcpy(p->Tbc, prm->Tbc, sizeof p->Tbc);
    p->xrot = prm->xrot_info; p->yrot = prm->yrot_info; p->zinfo = prm->z_info;
    p->delta = prm->huber_delta; p->cut = prm->chi2_cut;
    p->iterations = prm->iterations[mode]; p->min_points = prm->min_points[mode]; p->mode = mode;
    return SE2GPU_OK;
}

constexpr size_t kStageBytes = (sizeof(double) * 18 + sizeof(float) * 6) * kStageMax;

int launch(int B, const float* d_Tcw0, const float* d_Tcw1, const int* d_ptr, const float* d_xyz, const float* d_z0,
           const float* d_z1, const double* d_info0, const double* d_info1, const Params& p, float* d_measure, float* d_info,
           int* d_status, int* d_iters, se2gpu_ba_iter_stats* d_stats, uint8_t* d_outlier, double* d_poses, double* d_points,
           double* d_work, double* d_trace, cudaStream_t stream) {
    SE2_NVTX("se2gpu_feat_edge");
    SE2_LAUNCH(k_feat_edge, B, kThreads, kStageBytes, stream, d_Tcw0, d_Tcw1, d_ptr, d_xyz, d_z0, d_z1, d_info0, d_info1, p,
               d_measure, d_info, d_status, d_iters, d_stats, d_outlier, d_poses, d_points, d_work, d_trace);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int host_run(int B, int mode, const float* Tcw0, const float* Tcw1, const int* point_ptr, const float* xyz, const float* z0,
             const float* z1, const double* info0, const double* info1, const se2gpu_feat_edge_params* params, float* measure,
             float* info, int* status, int* iterations, se2gpu_ba_iter_stats* stats, uint8_t* outlier, double* poses,
             double* points, double* trace, int device) {
    Params p;
    { const int rc = check_params(params, mode, &p); if (rc) return rc; }
    if (B < 0 || (B && (!Tcw0 || !Tcw1 || !point_ptr || !measure || !info))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (B && point_ptr[0] != 0) return fail(SE2GPU_ERR_INVALID, "point_ptr[0] must be 0");
    for (int b = 0; b < B; ++b)
        if (point_ptr[b + 1] < point_ptr[b]) return fail(SE2GPU_ERR_INVALID, "point_ptr not ascending at %d", b);
    const size_t P = B ? (size_t)point_ptr[B] : 0;
    if (P && (!xyz || !z0 || !z1 || !info0 || !info1)) return fail(SE2GPU_ERR_INVALID, "null point arrays");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (B == 0) return SE2GPU_OK;
    const size_t it = (size_t)p.iterations;
    const float* dT0 = st.upload(Tcw0, 16 * (size_t)B);
    const float* dT1 = st.upload(Tcw1, 16 * (size_t)B);
    const int* dptr = st.upload(point_ptr, (size_t)B + 1);
    const float* dx = st.upload(xyz, 3 * P);
    const float* dz0 = st.upload(z0, 3 * P);
    const float* dz1 = st.upload(z1, 3 * P);
    const double* di0 = st.upload(info0, 9 * P);
    const double* di1 = st.upload(info1, 9 * P);
    float* dm = st.inout(measure, 16 * (size_t)B);   // a TOO_FEW pair's outputs come back as they went in
    float* dinf = st.inout(info, 36 * (size_t)B);
    int* dsts = status ? st.output(status, B) : nullptr;
    int* dit = iterations ? st.output(iterations, B) : nullptr;
    se2gpu_ba_iter_stats* dst = stats ? st.output(stats, B * it) : nullptr;
    uint8_t* dout = outlier ? st.output(outlier, P) : nullptr;
    double* dposes = poses ? st.inout(poses, 14 * (size_t)B) : nullptr;
    double* dpts = points ? st.inout(points, 3 * P) : st.scratch<double>(3 * P);
    double* dwork = st.scratch<double>(3 * P);
    double* dtr = trace ? st.output(trace, 24 * B * it) : nullptr;
    if (dst) st.check(cudaMemset(dst, 0, sizeof(se2gpu_ba_iter_stats) * B * it), "cudaMemset");
    if (dtr) st.check(cudaMemset(dtr, 0, sizeof(double) * 24 * B * it), "cudaMemset");
    if (dout) st.check(cudaMemset(dout, 0, P), "cudaMemset");
    if (const int rc = st.status()) return rc;
    { const int rc = launch(B, dT0, dT1, dptr, dx, dz0, dz1, di0, di1, p, dm, dinf, dsts, dit, dst, dout, dposes, dpts, dwork, dtr, nullptr); if (rc) return rc; }
    return st.finish();
}

}  // namespace

int se2gpu_feat_edge(int B, int mode, const float* Tcw0, const float* Tcw1, const int* point_ptr, const float* xyz,
                     const float* z0, const float* z1, const double* info0, const double* info1,
                     const se2gpu_feat_edge_params* params, float* measure, float* info, int* status, int* iterations,
                     se2gpu_ba_iter_stats* stats, uint8_t* outlier, double* poses, double* points, int device) {
    return host_run(B, mode, Tcw0, Tcw1, point_ptr, xyz, z0, z1, info0, info1, params, measure, info, status, iterations, stats,
                    outlier, poses, points, nullptr, device);
}

int se2gpu_feat_edge_debug_trace(int B, int mode, const float* Tcw0, const float* Tcw1, const int* point_ptr, const float* xyz,
                                 const float* z0, const float* z1, const double* info0, const double* info1,
                                 const se2gpu_feat_edge_params* params, float* measure, float* info, int* status, int* iterations,
                                 se2gpu_ba_iter_stats* stats, uint8_t* outlier, double* poses, double* points, double* trace,
                                 int device) {
    return host_run(B, mode, Tcw0, Tcw1, point_ptr, xyz, z0, z1, info0, info1, params, measure, info, status, iterations, stats,
                    outlier, poses, points, trace, device);
}

int se2gpu_feat_edge_device(int B, int mode, const float* d_Tcw0, const float* d_Tcw1, const int* d_point_ptr, const float* d_xyz,
                            const float* d_z0, const float* d_z1, const double* d_info0, const double* d_info1,
                            const se2gpu_feat_edge_params* params, float* d_measure, float* d_info, int* d_status,
                            int* d_iterations, se2gpu_ba_iter_stats* d_stats, uint8_t* d_outlier, double* d_poses,
                            double* d_points, double* d_work, void* stream) {
    Params p;
    { const int rc = check_params(params, mode, &p); if (rc) return rc; }
    if (B < 0 || (B && (!d_Tcw0 || !d_Tcw1 || !d_point_ptr || !d_xyz || !d_z0 || !d_z1 || !d_info0 || !d_info1 || !d_measure ||
                        !d_info || !d_points || !d_work)))
        return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    if (B == 0) return SE2GPU_OK;
    return launch(B, d_Tcw0, d_Tcw1, d_point_ptr, d_xyz, d_z0, d_z1, d_info0, d_info1, p, d_measure, d_info, d_status, d_iterations,
                  d_stats, d_outlier, d_poses, d_points, d_work, nullptr, (cudaStream_t)stream);
}
