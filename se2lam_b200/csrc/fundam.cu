// Track::removeOutliers (reference src/Track.cpp:308-344) on the GPU: cv::findFundamentalMat(pt1, pt2, mask) with
// OpenCV 4.13's defaults (FM_RANSAC, 3 px, confidence 0.99, 1000 iterations; LMedS below 15 pairs), the mask applied to
// matches12 and the "fewer than 10 inliers drops every match" rule. One CTA per frame pair:
//   - the matched pairs are gathered in ascending keypoint order into shared memory;
//   - thread 0 draws a wave of up to kWave subsets from the call-local cv::RNG stream (duplicate and collinear redraws
//     included), one thread per subset runs the 7-point kernel, and the CTA scores every model of the wave (inlier count,
//     or the LMedS median);
//   - thread 0 walks the wave's models in hypothesis order with OpenCV's acceptance rule and niters update, and the loop
//     stops once the iteration count reaches niters. Subsets drawn past that point are discarded: the RNG is local to
//     the call, so they change nothing.
// Every floating-point operation is an explicitly rounded intrinsic in the host's evaluation order and nothing is fused
// (OpenCV's fundam.cpp is not built with FMA); the FFMA / DFMA left in the SASS expand __ddiv_rn / __dsqrt_rn
// (tests/test_fundam_sass.py). RANSACUpdateNumIters' glibc log / pow are a threshold table built on the host.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <mutex>

#include "common.h"

using namespace se2gpu;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kWave = 32;           // hypotheses drawn and scored per round
constexpr int kModelPoints = 7;
constexpr int kMaxPairs = kFundamMaxPairs;   // keypoint capacity of frame 1 (shared memory: 20 bytes per pair)
constexpr int kNitersTable = 1000;  // RANSACUpdateNumIters never exceeds maxIters = 1000

// c_niters[k - 1] = the least ep in [0, 1] with RANSACUpdateNumIters(0.99, ep, 7, 1000) >= k (glibc log / pow)
__constant__ double c_niters[kNitersTable];

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

// cv::RNG (multiply-with-carry) and RNG::uniform(0, n)
__device__ __forceinline__ int rng_uniform(uint64_t& s, int n) {
    s = (uint64_t)(unsigned)s * 4164903690u + (unsigned)(s >> 32);
    return (int)((unsigned)s % (unsigned)n);
}

// haveCollinearPoints on the subset: the 7th point against every pair of earlier ones (float differences, double products)
__device__ bool collinear(const float2* p, const int* idx) {
    const float2 pi = p[idx[kModelPoints - 1]];
    for (int j = 0; j < kModelPoints - 1; j++) {
        const float2 pj = p[idx[j]];
        const double dx1 = __fsub_rn(pj.x, pi.x), dy1 = __fsub_rn(pj.y, pi.y);
        for (int k = 0; k < j; k++) {
            const float2 pk = p[idx[k]];
            const double dx2 = __fsub_rn(pk.x, pi.x), dy2 = __fsub_rn(pk.y, pi.y);
            const double lhs = fabs(dsub(dmul(dx2, dy1), dmul(dy2, dx1)));
            const double sum = dadd(dadd(dadd(fabs(dx1), fabs(dy1)), fabs(dx2)), fabs(dy2));
            if (lhs <= dmul((double)FLT_EPSILON, sum)) return true;
        }
    }
    return false;
}

// getSubset(m1, m2, ms1, ms2, rng, max_attempts)
__device__ bool get_subset(const float2* p1, const float2* p2, int n, uint64_t& s, int max_attempts, int* idx) {
    for (int it = 0; it < max_attempts; it++) {
        for (int i = 0; i < kModelPoints; i++) {
            int v = rng_uniform(s, n);
            for (;;) {
                bool dup = false;
                for (int k = 0; k < i; k++) dup = dup || idx[k] == v;
                if (!dup) break;
                v = rng_uniform(s, n);
            }
            idx[i] = v;
        }
        if (!collinear(p1, idx) && !collinear(p2, idx)) return true;
    }
    return false;
}

__device__ __forceinline__ double cubic_at(double a1, double a2, double a3, double x) {
    return dadd(dmul(dadd(dmul(dadd(x, a1), x), a2), x), a3);
}
__device__ __forceinline__ long long ord(double x) {
    const long long u = __double_as_longlong(x);
    return u >= 0 ? u : (long long)(0x8000000000000000ull - (unsigned long long)u);
}
__device__ __forceinline__ double unord(long long o) {
    return __longlong_as_double(o >= 0 ? o : (long long)(0x8000000000000000ull - (unsigned long long)o));
}

// root of x^3 + a1 x^2 + a2 x + a3 in [lo, hi]: bisection over the ordered doubles (the oracle's bisect)
__device__ double bisect(double a1, double a2, double a3, double lo, double hi) {
    const bool neg_lo = cubic_at(a1, a2, a3, lo) < 0;
    long long l = ord(lo), h = ord(hi);
    while ((unsigned long long)h - (unsigned long long)l > 1) {
        const long long m = (long long)((unsigned long long)l + ((unsigned long long)h - (unsigned long long)l) / 2);
        const double x = unord(m), v = cubic_at(a1, a2, a3, x);
        if (v == 0) return x;
        if ((v < 0) == neg_lo) l = m; else h = m;
    }
    const double xl = unord(l), xh = unord(h);
    return fabs(cubic_at(a1, a2, a3, xl)) <= fabs(cubic_at(a1, a2, a3, xh)) ? xl : xh;
}

__device__ int solve_cubic(const double* c, double* r) {
    double a0 = c[0], a1 = c[1], a2 = c[2], a3 = c[3];
    if (a0 == 0) {
        if (a1 == 0) {
            if (a2 == 0) return 0;
            r[0] = __ddiv_rn(-a3, a2);
            return 1;
        }
        double d = dsub(dmul(a2, a2), dmul(dmul(4., a1), a3));
        if (!(d >= 0)) return 0;
        d = __dsqrt_rn(d);
        const double q1 = dmul(dadd(-a2, d), 0.5), q2 = dmul(dadd(a2, d), -0.5);
        const double q = fabs(q1) > fabs(q2) ? q1 : q2;
        r[0] = __ddiv_rn(q, a1); r[1] = __ddiv_rn(a3, q);
        return d > 0 ? 2 : 1;
    }
    a0 = __ddiv_rn(1., a0);
    a1 = dmul(a1, a0); a2 = dmul(a2, a0); a3 = dmul(a3, a0);
    // (a1 a1 (a2 a2 - 4 a1 a3) + 2 a2 (9 a1 a3 - 2 a2 a2) - 27 a3 a3) / 108
    const double u = dmul(dmul(a1, a1), dsub(dmul(a2, a2), dmul(dmul(4., a1), a3)));
    const double v = dmul(dmul(2., a2), dsub(dmul(dmul(9., a1), a3), dmul(dmul(2., a2), a2)));
    const double d = dmul(dsub(dadd(u, v), dmul(dmul(27., a3), a3)), 1. / 108);
    double B = fabs(a1);
    if (B < fabs(a2)) B = fabs(a2);
    if (B < fabs(a3)) B = fabs(a3);
    B = dadd(B, 1.);
    if (B > DBL_MAX) B = DBL_MAX;
    if (d > 0) {
        const double Q = dmul(dsub(dmul(a1, a1), dmul(3., a2)), 1. / 9);
        const double sq = __dsqrt_rn(Q), c0 = dmul(a1, -1. / 3);
        const double cl = dsub(c0, sq), ch = dadd(c0, sq);
        r[0] = bisect(a1, a2, a3, -B, cl);
        r[1] = bisect(a1, a2, a3, cl, ch);
        r[2] = bisect(a1, a2, a3, ch, B);
        return 3;
    }
    r[0] = bisect(a1, a2, a3, -B, B);
    return 1;
}

// 7-point kernel (the oracle's run7point): up to 3 row-major F into fm, returns their number. a [63] is scratch.
__device__ int run7point(const float2* p1, const float2* p2, const int* idx, double* a, double* fm) {
    double m1cx = 0, m1cy = 0, m2cx = 0, m2cy = 0;
    for (int i = 0; i < 7; i++) {
        const float2 u = p1[idx[i]], w = p2[idx[i]];
        m1cx = dadd(m1cx, (double)u.x); m1cy = dadd(m1cy, (double)u.y);
        m2cx = dadd(m2cx, (double)w.x); m2cy = dadd(m2cy, (double)w.y);
    }
    const double t = 1. / 7;
    m1cx = dmul(m1cx, t); m1cy = dmul(m1cy, t); m2cx = dmul(m2cx, t); m2cy = dmul(m2cy, t);
    double scale1 = 0, scale2 = 0;
    for (int i = 0; i < 7; i++) {
        const float2 u = p1[idx[i]], w = p2[idx[i]];
        const double ax = dsub(u.x, m1cx), ay = dsub(u.y, m1cy), bx = dsub(w.x, m2cx), by = dsub(w.y, m2cy);
        scale1 = dadd(scale1, __dsqrt_rn(dadd(dmul(ax, ax), dmul(ay, ay))));
        scale2 = dadd(scale2, __dsqrt_rn(dadd(dmul(bx, bx), dmul(by, by))));
    }
    scale1 = dmul(scale1, t); scale2 = dmul(scale2, t);
    if (scale1 < FLT_EPSILON || scale2 < FLT_EPSILON) return 0;
    scale1 = __ddiv_rn(1.4142135623730951, scale1);     // sqrt(2.) / scale
    scale2 = __ddiv_rn(1.4142135623730951, scale2);
    for (int i = 0; i < 7; i++) {
        const float2 u = p1[idx[i]], w = p2[idx[i]];
        const double x0 = dmul(dsub(u.x, m1cx), scale1), y0 = dmul(dsub(u.y, m1cy), scale1);
        const double x1 = dmul(dsub(w.x, m2cx), scale2), y1 = dmul(dsub(w.y, m2cy), scale2);
        double* row = a + 9 * i;
        row[0] = dmul(x1, x0); row[1] = dmul(x1, y0); row[2] = x1;
        row[3] = dmul(y1, x0); row[4] = dmul(y1, y0); row[5] = y1;
        row[6] = x0; row[7] = y0; row[8] = 1;
    }
    for (int r = 0; r < 7; r++) {
        double pivot = a[9 * r + r];
        int prow = r;
        for (int k = r + 1; k < 7; k++)
            if (fabs(pivot) < fabs(a[9 * k + r])) { pivot = a[9 * k + r]; prow = k; }
        if (fabs(pivot) < DBL_EPSILON) return 0;
        for (int c = r; c < 9; c++) { const double s = a[9 * prow + c]; a[9 * prow + c] = a[9 * r + c]; a[9 * r + c] = s; }
        for (int j = r + 1; j < 7; j++) {
            const double fac = __ddiv_rn(a[9 * j + r], pivot);
            for (int c = r; c < 9; c++) a[9 * j + c] = dsub(a[9 * j + c], dmul(fac, a[9 * r + c]));
        }
    }
    double f1[9], f2[9];
    f1[7] = 0; f1[8] = 1; f2[7] = 1; f2[8] = 0;
#pragma unroll
    for (int i = 6; i >= 0; i--) {
        double acc1 = 0, acc2 = 0;
#pragma unroll
        for (int j = i + 1; j < 9; j++) { acc1 = dsub(acc1, dmul(a[9 * i + j], f1[j])); acc2 = dsub(acc2, dmul(a[9 * i + j], f2[j])); }
        f1[i] = __ddiv_rn(acc1, a[9 * i + i]);
        f2[i] = __ddiv_rn(acc2, a[9 * i + i]);
    }
#pragma unroll
    for (int i = 0; i < 9; i++) f1[i] = dsub(f1[i], f2[i]);
    // x y - z w, and run7Point's cubic coefficients in its order of evaluation
#define M2(x, y, z, w) dsub(dmul(x, y), dmul(z, w))
    double t0 = M2(f2[4], f2[8], f2[5], f2[7]);
    double t1 = M2(f2[3], f2[8], f2[5], f2[6]);
    double t2 = M2(f2[3], f2[7], f2[4], f2[6]);
    double c[4], roots[3];
    c[3] = dadd(dsub(dmul(f2[0], t0), dmul(f2[1], t1)), dmul(f2[2], t2));
    {
        double s = dadd(dsub(dmul(f1[0], t0), dmul(f1[1], t1)), dmul(f1[2], t2));
        s = dsub(s, dmul(f1[3], M2(f2[1], f2[8], f2[2], f2[7])));
        s = dadd(s, dmul(f1[4], M2(f2[0], f2[8], f2[2], f2[6])));
        s = dsub(s, dmul(f1[5], M2(f2[0], f2[7], f2[1], f2[6])));
        s = dadd(s, dmul(f1[6], M2(f2[1], f2[5], f2[2], f2[4])));
        s = dsub(s, dmul(f1[7], M2(f2[0], f2[5], f2[2], f2[3])));
        c[2] = dadd(s, dmul(f1[8], M2(f2[0], f2[4], f2[1], f2[3])));
    }
    t0 = M2(f1[4], f1[8], f1[5], f1[7]);
    t1 = M2(f1[3], f1[8], f1[5], f1[6]);
    t2 = M2(f1[3], f1[7], f1[4], f1[6]);
    {
        double s = dadd(dsub(dmul(f2[0], t0), dmul(f2[1], t1)), dmul(f2[2], t2));
        s = dsub(s, dmul(f2[3], M2(f1[1], f1[8], f1[2], f1[7])));
        s = dadd(s, dmul(f2[4], M2(f1[0], f1[8], f1[2], f1[6])));
        s = dsub(s, dmul(f2[5], M2(f1[0], f1[7], f1[1], f1[6])));
        s = dadd(s, dmul(f2[6], M2(f1[1], f1[5], f1[2], f1[4])));
        s = dsub(s, dmul(f2[7], M2(f1[0], f1[5], f1[2], f1[3])));
        c[1] = dadd(s, dmul(f2[8], M2(f1[0], f1[4], f1[1], f1[3])));
    }
    c[0] = dadd(dsub(dmul(f1[0], t0), dmul(f1[1], t1)), dmul(f1[2], t2));
#undef M2
    const int n = solve_cubic(c, roots);

    const double T1[9] = {scale1, 0, -dmul(scale1, m1cx), 0, scale1, -dmul(scale1, m1cy), 0, 0, 1};
    const double T2[9] = {scale2, 0, -dmul(scale2, m2cx), 0, scale2, -dmul(scale2, m2cy), 0, 0, 1};
    for (int k = 0; k < n; k++) {
        double* F = fm + 9 * k;
        double lambda = roots[k], mu = 1.;
        const double s = dadd(dmul(f1[8], roots[k]), f2[8]);
        double g[9], h[9];
        if (fabs(s) > DBL_EPSILON) { mu = __ddiv_rn(1., s); lambda = dmul(lambda, mu); g[8] = 1.; }
        else g[8] = 0.;
#pragma unroll
        for (int i = 0; i < 8; i++) g[i] = dadd(dmul(f1[i], lambda), dmul(f2[i], mu));
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                double acc = 0;
#pragma unroll
                for (int q = 0; q < 3; q++) acc = dadd(acc, dmul(T2[3 * q + i], g[3 * q + j]));
                h[3 * i + j] = acc;
            }
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                double acc = 0;
#pragma unroll
                for (int q = 0; q < 3; q++) acc = dadd(acc, dmul(h[3 * i + q], T1[3 * q + j]));
                F[3 * i + j] = acc;
            }
        if (fabs(F[8]) > FLT_EPSILON) {
            const double inv = __ddiv_rn(1., F[8]);
            for (int i = 0; i < 9; i++) F[i] = dmul(F[i], inv);
        }
    }
    return n;
}

// FMEstimatorCallback::computeError for pair i
__device__ float epi_error(const double* F, float2 p, float2 q) {
    const double x1 = p.x, y1 = p.y, x2 = q.x, y2 = q.y;
    double a = dadd(dadd(dmul(F[0], x1), dmul(F[1], y1)), F[2]);
    double b = dadd(dadd(dmul(F[3], x1), dmul(F[4], y1)), F[5]);
    double c = dadd(dadd(dmul(F[6], x1), dmul(F[7], y1)), F[8]);
    const double s2 = __ddiv_rn(1., dadd(dmul(a, a), dmul(b, b)));
    const double d2 = dadd(dadd(dmul(x2, a), dmul(y2, b)), c);
    a = dadd(dadd(dmul(F[0], x2), dmul(F[3], y2)), F[6]);
    b = dadd(dadd(dmul(F[1], x2), dmul(F[4], y2)), F[7]);
    c = dadd(dadd(dmul(F[2], x2), dmul(F[5], y2)), F[8]);
    const double s1 = __ddiv_rn(1., dadd(dmul(a, a), dmul(b, b)));
    const double d1 = dadd(dadd(dmul(x1, a), dmul(y1, b)), c);
    const double e1 = dmul(dmul(d1, d1), s1), e2 = dmul(dmul(d2, d2), s2);
    return __double2float_rn(e1 < e2 ? e2 : e1);
}

// RANSACUpdateNumIters(0.99, (n - good) / n, 7, max_iters) through the host-built threshold table
__device__ int update_num_iters(int n, int good, int max_iters) {
    const double ep = __ddiv_rn((double)(n - good), (double)n);
    int lo = 0, hi = kNitersTable;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (c_niters[mid] <= ep) lo = mid + 1; else hi = mid;
    }
    return lo < max_iters ? lo : max_iters;
}

__device__ __forceinline__ int block_sum(int v, int* s_red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
    for (int w = 0; w < kWarps; w++) t += s_red[w];
    return t;
}

struct Wave {
    double a[kWave][64];                // 7-point elimination scratch, one row block per hypothesis
    double F[kWave * 3][9];             // models of the wave, 3 slots per hypothesis
    int sub[kWave][kModelPoints];
    int nm[kWave];
    float score_f[kWave * 3];           // LMedS median of each model
    int score_i[kWave * 3];             // RANSAC inlier count of each model
};

// What a call does with few matches. TRACK: Track::removeOutliers clears every match when fewer than 10 inliers remain after
// the estimate. LOOP: GlobalMapper::RemoveMatchOutlierRansac (src/GlobalMapper.cpp:1207-1248) clears every match when
// fewer than 10 are given and does not estimate; after an estimate it keeps the mask whatever its count.
enum Gate { TRACK, LOOP };

// One CTA per frame pair. Dynamic shared memory: float2 p1[cap1], float2 p2[cap1], int idx[cap1]. Pair b's frame-2
// keypoints are slot2[b] of kp2_all / n2_all (slot2 NULL: b); a negative slot2[b] makes the pair's frame 2 empty.
// ninliers may be NULL. The two gates are two kernels, k_remove_outliers (TRACK) and k_remove_outliers_loop (LOOP).
template <Gate G>
__device__ __forceinline__ void remove_outliers(
        const se2gpu_keypoint* __restrict__ kp1_all, const int* __restrict__ n1_all, int cap1,
        const se2gpu_keypoint* __restrict__ kp2_all, const int* __restrict__ n2_all, int cap2, const int* __restrict__ slot2,
        int* __restrict__ m12_all, int* __restrict__ ninliers, double* __restrict__ F_out, int* __restrict__ iters_out,
        int lmeds_niters) {
    extern __shared__ __align__(16) unsigned char smem[];
    float2* p1 = reinterpret_cast<float2*>(smem);
    float2* p2 = p1 + cap1;
    int* idx = reinterpret_cast<int*>(p2 + cap1);
    __shared__ Wave w;
    __shared__ double s_best[9];
    __shared__ int s_red[kWarps], s_scan[kWarps];
    __shared__ int s_nsub, s_fail, s_stop, s_iter, s_niters, s_best_good, s_have, s_thresh_bits;
    __shared__ double s_min_median;
    __shared__ uint64_t s_rng;

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int s2 = slot2 ? slot2[b] : b;
    const int n1 = n1_all ? min(max(n1_all[b], 0), cap1) : cap1;
    const int n2 = s2 < 0 ? 0 : n2_all ? min(max(n2_all[s2], 0), cap2) : cap2;
    const se2gpu_keypoint* kp1 = kp1_all + (size_t)b * cap1;
    const se2gpu_keypoint* kp2 = kp2_all + (size_t)max(s2, 0) * cap2;
    int* m12 = m12_all + (size_t)b * cap1;

    // gather the matched pairs in ascending keypoint order (matches past n2 count as unmatched)
    int n = 0;
    for (int base = 0; base < n1; base += kThreads) {
        const int i = base + tid;
        const int j = i < n1 ? m12[i] : -1;
        const bool on = j >= 0 && j < n2;
        const unsigned bal = __ballot_sync(0xffffffffu, on);
        if (lane == 0) s_scan[warp] = __popc(bal);
        __syncthreads();
        int off = n, tot = 0;
        for (int q = 0; q < kWarps; q++) { if (q < warp) off += s_scan[q]; tot += s_scan[q]; }
        if (on) {
            const int k = off + __popc(bal & ((1u << lane) - 1));
            p1[k] = make_float2(kp1[i].x, kp1[i].y);
            p2[k] = make_float2(kp2[j].x, kp2[j].y);
            idx[k] = i;
        }
        n += tot;
        __syncthreads();
    }

    if (G == LOOP && n < 10) {
        for (int i = tid; i < n1; i += kThreads) m12[i] = -1;
        if (tid == 0) {
            if (ninliers) ninliers[b] = 0;
            if (iters_out) iters_out[b] = 0;
        }
        if (F_out && tid < 9) F_out[9 * (size_t)b + tid] = 0.;
        return;
    }

    const bool lmeds = n < 15;
    if (tid == 0) {
        s_rng = ~0ull; s_iter = 0; s_niters = lmeds ? lmeds_niters : 1000; s_best_good = 0; s_have = 0;
        s_min_median = DBL_MAX; s_stop = 0;
        for (int k = 0; k < 9; k++) s_best[k] = 0;
    }
    __syncthreads();

    if (n == kModelPoints) {
        // the kernel alone: mask all ones, F = the first root's matrix
        if (tid == 0) {
            int id7[kModelPoints] = {0, 1, 2, 3, 4, 5, 6};
            const int nm = run7point(p1, p2, id7, w.a[0], &w.F[0][0]);
            if (nm > 0) for (int k = 0; k < 9; k++) s_best[k] = w.F[0][k];
            s_iter = 1;
        }
    } else if (n > kModelPoints) {
        const int k_med = n / 2;
        for (;;) {
            if (tid == 0) {
                const int want = min(kWave, s_niters - s_iter);
                int j = 0;
                s_fail = 0;
                uint64_t s = s_rng;
                for (; j < want; j++)
                    if (!get_subset(p1, p2, n, s, lmeds ? 1000 : 10000, w.sub[j])) { s_fail = 1; break; }
                s_rng = s;
                s_nsub = j;
            }
            __syncthreads();
            const int nsub = s_nsub;
            if (tid < nsub) w.nm[tid] = run7point(p1, p2, w.sub[tid], w.a[tid], &w.F[3 * tid][0]);
            __syncthreads();
            for (int slot = warp; slot < 3 * nsub; slot += kWarps) {
                if (slot % 3 >= w.nm[slot / 3]) continue;
                const double* F = w.F[slot];
                if (!lmeds) {
                    int good = 0;
                    for (int i = lane; i < n; i += 32) good += epi_error(F, p1[i], p2[i]) <= 9.f;
                    for (int o = 16; o; o >>= 1) good += __shfl_xor_sync(0xffffffffu, good, o);
                    if (lane == 0) w.score_i[slot] = good;
                } else {
                    // the k-th smallest error in the order of its bits (nth_element over the floats as int)
                    const float e = lane < n ? epi_error(F, p1[lane], p2[lane]) : 0.f;
                    const int eb = __float_as_int(e);
                    int less = 0, eq = 0;
                    for (int q = 0; q < n; q++) {
                        const int qb = __shfl_sync(0xffffffffu, eb, q);
                        less += qb < eb; eq += qb == eb;
                    }
                    if (lane < n && less <= k_med && k_med < less + eq) w.score_f[slot] = e;
                }
            }
            __syncthreads();
            if (tid == 0) {
                int iter = s_iter, niters = s_niters;
                for (int j = 0; j < nsub && iter < niters; j++, iter++)
                    for (int k = 0; k < w.nm[j]; k++) {
                        const int slot = 3 * j + k;
                        if (!lmeds) {
                            const int good = w.score_i[slot];
                            if (good > max(s_best_good, kModelPoints - 1)) {
                                s_best_good = good;
                                for (int q = 0; q < 9; q++) s_best[q] = w.F[slot][q];
                                niters = update_num_iters(n, good, niters);
                            }
                        } else if ((double)w.score_f[slot] < s_min_median) {
                            s_min_median = w.score_f[slot];
                            for (int q = 0; q < 9; q++) s_best[q] = w.F[slot][q];
                        }
                    }
                // getSubset gave up: no estimate if it was the first draw, else the loop ends
                if (iter < niters && s_fail) { s_stop = 1; if (iter == 0) { s_best_good = 0; s_min_median = DBL_MAX; } }
                if (iter >= niters) s_stop = 1;
                s_iter = iter; s_niters = niters;
            }
            __syncthreads();
            if (s_stop) break;
        }
        if (tid == 0) {
            if (!lmeds) {
                s_have = s_best_good > 0;
                s_thresh_bits = __float_as_int(9.f);
            } else if (s_min_median < DBL_MAX) {
                s_have = 1;
                const double fac = dmul(2.5 * 1.4826, dadd(1., __ddiv_rn(5., (double)(n - kModelPoints))));
                double sigma = dmul(fac, __dsqrt_rn(s_min_median));
                sigma = sigma < 0.001 ? 0.001 : sigma;
                s_thresh_bits = __float_as_int(__double2float_rn(dmul(sigma, sigma)));
            }
        }
        __syncthreads();
    }

    // apply the mask (never written when no model was found: every pair is an outlier) and Track's < 10 rule
    const bool have = s_have != 0;
    const float thr = __int_as_float(s_thresh_bits);
    int nin = 0;
    if (n > kModelPoints)
        for (int i = tid; i < n; i += kThreads) {
            const bool in = have && epi_error(s_best, p1[i], p2[i]) <= thr;
            nin += in;
            if (!in) m12[idx[i]] = -1;
        }
    nin = block_sum(nin, s_red);
    // a false LMedS result (fewer than 7 inliers) returns an empty F; the mask stays written
    const bool f_out = n == kModelPoints || (have && !(lmeds && nin < kModelPoints));
    if (n == kModelPoints) nin = kModelPoints;
    if (G == TRACK && nin < 10) {
        nin = 0;
        for (int i = tid; i < n1; i += kThreads) m12[i] = -1;
    }
    if (tid == 0) {
        if (ninliers) ninliers[b] = nin;
        if (iters_out) iters_out[b] = s_iter;
    }
    if (F_out && tid < 9) F_out[9 * (size_t)b + tid] = f_out ? s_best[tid] : 0.;
}

#define SE2_REMOVE_OUTLIERS_PARAMS                                                                                            \
    const se2gpu_keypoint* __restrict__ kp1_all, const int* __restrict__ n1_all, int cap1,                                    \
    const se2gpu_keypoint* __restrict__ kp2_all, const int* __restrict__ n2_all, int cap2, const int* __restrict__ slot2,      \
    int* __restrict__ m12_all, int* __restrict__ ninliers, double* __restrict__ F_out, int* __restrict__ iters_out, int lmeds_niters
#define SE2_REMOVE_OUTLIERS_ARGS kp1_all, n1_all, cap1, kp2_all, n2_all, cap2, slot2, m12_all, ninliers, F_out, iters_out, lmeds_niters
__global__ void __launch_bounds__(kThreads) k_remove_outliers(SE2_REMOVE_OUTLIERS_PARAMS) {
    remove_outliers<TRACK>(SE2_REMOVE_OUTLIERS_ARGS);
}
__global__ void __launch_bounds__(kThreads) k_remove_outliers_loop(SE2_REMOVE_OUTLIERS_PARAMS) {
    remove_outliers<LOOP>(SE2_REMOVE_OUTLIERS_ARGS);
}
#undef SE2_REMOVE_OUTLIERS_PARAMS
#undef SE2_REMOVE_OUTLIERS_ARGS

__global__ void k_debug_niters(int count, const int* n, const int* good, const int* max_iters, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = update_num_iters(n[i], good[i], max_iters[i]);
}

// ------------------------------------------------------------------------------------------ host side
int update_num_iters_host(double p, double ep, int model_points, int max_iters) {
    p = p < 0. ? 0. : p; p = 1. < p ? 1. : p;
    ep = ep < 0. ? 0. : ep; ep = 1. < ep ? 1. : ep;
    double num = 1. - p < DBL_MIN ? DBL_MIN : 1. - p;
    double denom = 1. - std::pow(1. - ep, model_points);
    if (denom < DBL_MIN) return 0;
    num = std::log(num);
    denom = std::log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)std::lrint(num / denom);
}

double g_table[kNitersTable];

void build_table() {
    // RANSACUpdateNumIters(0.99, ep, 7, 1000) rises with ep; for each k, bisect over the doubles of [0, 1] (all positive,
    // so their bit patterns are ordered) for the least ep reaching k
    for (int k = 1; k <= kNitersTable; k++) {
        uint64_t lo = 0, hi;
        double one = 1.0;
        std::memcpy(&hi, &one, 8);
        while (hi - lo > 1) {
            const uint64_t mid = lo + (hi - lo) / 2;
            double x;
            std::memcpy(&x, &mid, 8);
            if (update_num_iters_host(0.99, x, kModelPoints, kNitersTable) >= k) hi = mid; else lo = mid;
        }
        std::memcpy(&g_table[k - 1], &hi, 8);
    }
}

std::once_flag g_table_once;
const double* niters_table() {
    std::call_once(g_table_once, build_table);
    return g_table;
}

// per device: the table uploaded and the kernel's shared-memory limit raised
int prepare_device() {
    static std::mutex mu;
    static bool ready[kMaxDevices] = {};
    int dev = 0;
    SE2_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    if (dev < kMaxDevices && ready[dev]) return SE2GPU_OK;
    SE2_CUDA(cudaMemcpyToSymbol(c_niters, niters_table(), sizeof(double) * kNitersTable));
    SE2_CUDA(cudaFuncSetAttribute(k_remove_outliers, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * kMaxPairs));
    SE2_CUDA(cudaFuncSetAttribute(k_remove_outliers_loop, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * kMaxPairs));
    if (dev < kMaxDevices) ready[dev] = true;
    return SE2GPU_OK;
}

// OpenCV's LMedS iteration count (RANSACUpdateNumIters(0.99, 0.45, 7, 1000), at least 3)
int lmeds_niters() {
    static const int v = [] { const int n = update_num_iters_host(0.99, 0.45, kModelPoints, 1000); return n < 3 ? 3 : n; }();
    return v;
}

}  // namespace

int se2gpu::fundam_prepare() { return prepare_device(); }

int se2gpu::remove_outliers_loop(int batch, const se2gpu_keypoint* d_kp1, int cap1, const se2gpu_keypoint* d_kp2, int cap2,
                                 const int* d_slot2, int* d_matches12, cudaStream_t s) {
    if (batch == 0) return SE2GPU_OK;
    { const int rc = prepare_device(); if (rc) return rc; }
    SE2_LAUNCH(k_remove_outliers_loop, batch, kThreads, (size_t)20 * cap1, s, d_kp1, nullptr, cap1, d_kp2, nullptr, cap2, d_slot2,
               d_matches12, nullptr, nullptr, nullptr, lmeds_niters());
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_remove_outliers_device(int batch, const se2gpu_keypoint* d_kp1, const int* d_n1, int cap1, const se2gpu_keypoint* d_kp2,
                                  const int* d_n2, int cap2, int* d_matches12, int* d_ninliers, double* d_F, int* d_iters,
                                  void* stream) {
    if (batch < 0 || cap1 < 0 || cap2 < 0) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (cap1 > kMaxPairs) return fail(SE2GPU_ERR_CAPACITY, "cap1 = %d exceeds %d keypoints", cap1, kMaxPairs);
    if (batch && (!d_ninliers || (cap1 && (!d_kp1 || !d_matches12)) || (cap2 && !d_kp2)))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    { const int rc = require_device(); if (rc) return rc; }
    if (batch == 0) return SE2GPU_OK;
    { const int rc = prepare_device(); if (rc) return rc; }
    SE2_NVTX("se2gpu_remove_outliers");
    SE2_LAUNCH(k_remove_outliers, batch, kThreads, (size_t)20 * cap1, (cudaStream_t)stream, d_kp1, d_n1, cap1, d_kp2, d_n2, cap2,
               nullptr, d_matches12, d_ninliers, d_F, d_iters, lmeds_niters());
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_remove_outliers(int batch, const se2gpu_keypoint* kp1, const int* n1, int cap1, const se2gpu_keypoint* kp2, const int* n2,
                           int cap2, int* matches12, int* ninliers, double* F, int* iters, int device) {
    if (batch < 0 || cap1 < 0 || cap2 < 0) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (cap1 > kMaxPairs) return fail(SE2GPU_ERR_CAPACITY, "cap1 = %d exceeds %d keypoints", cap1, kMaxPairs);
    if (batch && (!ninliers || (cap1 && (!kp1 || !matches12)) || (cap2 && !kp2))) return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int b = 0; b < batch; b++) {
        const int c1 = n1 ? n1[b] : cap1, c2 = n2 ? n2[b] : cap2;
        if (c1 < 0 || c1 > cap1 || c2 < 0 || c2 > cap2) return fail(SE2GPU_ERR_INVALID, "pair %d: keypoint count out of range", b);
        for (int i = 0; i < c1; i++)
            if (matches12[(size_t)b * cap1 + i] >= c2)
                return fail(SE2GPU_ERR_INVALID, "pair %d: matches12[%d] = %d is not a frame-2 keypoint", b, i, matches12[(size_t)b * cap1 + i]);
    }
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (batch == 0) return SE2GPU_OK;
    const se2gpu_keypoint* dk1 = st.upload(kp1, (size_t)batch * cap1);
    const se2gpu_keypoint* dk2 = st.upload(kp2, (size_t)batch * cap2);
    const int* dn1 = n1 ? st.upload(n1, batch) : nullptr;
    const int* dn2 = n2 ? st.upload(n2, batch) : nullptr;
    int* dm = st.inout(matches12, (size_t)batch * cap1);
    int* dnin = st.output(ninliers, batch);
    double* dF = F ? st.output(F, 9 * (size_t)batch) : nullptr;
    int* dit = iters ? st.output(iters, batch) : nullptr;
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_remove_outliers_device(batch, dk1, dn1, cap1, dk2, dn2, cap2, dm, dnin, dF, dit, nullptr); if (rc) return rc; }
    return st.finish();
}

void se2gpu_fundam_niters_table(double* thresholds) { std::memcpy(thresholds, niters_table(), sizeof(double) * kNitersTable); }

int se2gpu_fundam_debug_niters(int count, const int* n, const int* good, const int* max_iters, int* out, int device) {
    if (count < 0 || (count && (!n || !good || !max_iters || !out))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    for (int i = 0; i < count; i++)
        if (n[i] <= 0 || good[i] < 0 || good[i] > n[i] || max_iters[i] < 0 || max_iters[i] > kNitersTable)
            return fail(SE2GPU_ERR_INVALID, "entry %d out of range", i);
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (count == 0) return SE2GPU_OK;
    { const int rc = prepare_device(); if (rc) return rc; }
    const int* dn = st.upload(n, count);
    const int* dg = st.upload(good, count);
    const int* dm = st.upload(max_iters, count);
    int* dout = st.output(out, count);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_debug_niters, (count + 255) / 256, 256, 0, nullptr, count, dn, dg, dm, dout);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}
