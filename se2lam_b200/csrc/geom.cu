// Two-view geometry over matches: cvu::triangulate, Track::doTriangulate, Track::calcSE3toXYZInfo and the MatchByProjection
// branch of LocalMapper::findCorrespd (DESIGN.md section 8). One thread per match; counts are reduced with warp ballots and
// one atomic per warp. Then the map-point updates MapPoint::addObservation / eraseObservation / updateMeasureInKFs
// (DESIGN.md section 13): one warp per map point, no atomics.
//
// Every floating-point operation is written with an explicitly rounded intrinsic, in the order the reference and OpenCV
// evaluate it on the host, so that the compiler cannot contract a multiply and an add the host keeps apart. The only fused
// multiply-adds of the reference's arithmetic are the rows of A (cv::addWeighted's dispatched SIMD kernel on an AVX2 host).
#include <cfloat>
#include <cstdint>
#include <type_traits>

#include "common.h"
#include "fround.h"
#include "median_desc.h"

using namespace se2gpu;

namespace {

constexpr int kBlock = 128;

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ F3 sub3(F3 a, F3 b) { return {fs(a.x, b.x), fs(a.y, b.y), fs(a.z, b.z)}; }
__device__ __forceinline__ float dot3(F3 a, F3 b) { return fa(fa(fm(a.x, b.x), fm(a.y, b.y)), fm(a.z, b.z)); }
__device__ __forceinline__ F3 cross3(F3 a, F3 b) {
    return {fs(fm(a.y, b.z), fm(a.z, b.y)), fs(fm(a.z, b.x), fm(a.x, b.z)), fs(fm(a.x, b.y), fm(a.y, b.x))};
}
// cv::norm(Point3_): sqrt of the double sum of squares
__device__ __forceinline__ double norm3(F3 p) {
    const double x = p.x, y = p.y, z = p.z;
    return __dsqrt_rn(da(da(dm(x, x), dm(y, y)), dm(z, z)));
}

// The double hypot of OpenCV's JacobiSVDImpl_: lapack.cpp's inline template (not libm's hypot), the larger magnitude times
// sqrt(1 + ratio^2), evaluated unfused as on the host.
__device__ __forceinline__ double cv_hypot(double a, double b) {
    a = fabs(a);
    b = fabs(b);
    if (a > b) return dm(a, __dsqrt_rn(da(1.0, dm(dd(b, a), dd(b, a)))));
    if (b > 0) return dm(b, __dsqrt_rn(da(1.0, dm(dd(a, b), dd(a, b)))));
    return 0.0;
}

// std::asin(float) of the host: glibc's __ieee754_asinf (sysdeps/ieee754/flt-32/e_asinf.c, glibc 2.39; it is not correctly
// rounded, so the device restates it operation by operation). Arguments here are >= 0 or NaN.
__device__ __forceinline__ float asinf_host(float x) {
    const float p0 = 1.666675248e-1f, p1 = 7.495297643e-2f, p2 = 4.547037598e-2f, p3 = 2.417951451e-2f, p4 = 4.216630880e-2f;
    const float pio2_hi = 1.57079637050628662109375f, pio2_lo = -4.37113900018624283e-8f, pio4_hi = 0.785398185253143310546875f;
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
    if (ix == 0x3f800000) return fa(fm(x, pio2_hi), fm(x, pio2_lo));
    if (ix > 0x3f800000) return __fdiv_rn(fs(x, x), fs(x, x));
    if (ix < 0x3f000000) {
        if (ix < 0x32000000) return x;
        const float t = fm(x, x);
        const float w = fm(t, fa(p0, fm(t, fa(p1, fm(t, fa(p2, fm(t, fa(p3, fm(t, p4)))))))));
        return fa(x, fm(x, w));
    }
    const float t = fm(fs(1.f, fabsf(x)), 0.5f);
    float p = fm(t, fa(p0, fm(t, fa(p1, fm(t, fa(p2, fm(t, fa(p3, fm(t, p4)))))))));
    const float s = __fsqrt_rn(t);
    float r;
    if (ix >= 0x3F79999A) {
        r = fs(pio2_hi, fs(fm(2.f, fa(s, fm(s, p))), pio2_lo));
    } else {
        const float w = __int_as_float(__float_as_int(s) & 0xfffff000);
        const float c = fd(fs(t, fm(w, w)), fa(s, w));
        p = fs(fm(fm(2.f, s), p), fs(pio2_lo, fm(2.f, c)));
        const float q = fs(pio4_hi, fm(2.f, w));
        r = fs(pio4_hi, fs(p, q));
    }
    return hx > 0 ? r : -r;
}

// cv::gemm(A[3x3], B[3x ncols], alpha) through OpenCV's small-matrix path: float sums left to right, then (float)(t*alpha + 0)
__device__ __forceinline__ float gemm3_elem(const float* A, int lda, int i, const float* B, int ldb, int j, double alpha) {
    const float t = fa(fa(fm(A[i * lda], B[j]), fm(A[i * lda + 1], B[ldb + j])), fm(A[i * lda + 2], B[2 * ldb + j]));
    return __double2float_rn(da(dm((double)t, alpha), 0.0));
}

// Kcam * T.rowRange(0,3)
__device__ __forceinline__ void projection(const float* K, const float* T, float* P) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) P[i * 4 + j] = gemm3_elem(K, 3, i, T, 4, j, 1.0);
}

// cvu::inv: [R^T | -R^T t]
__device__ __forceinline__ void inv4(const float* T, float* Ti) {
    float RT[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) RT[i * 3 + j] = T[j * 4 + i];
    const float t[3] = {T[3], T[7], T[11]};
#pragma unroll
    for (int i = 0; i < 16; i++) Ti[i] = (i % 5 == 0) ? 1.f : 0.f;
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) Ti[i * 4 + j] = RT[i * 3 + j];
        Ti[i * 4 + 3] = gemm3_elem(RT, 3, i, t, 1, 0, -1.0);
    }
}

// cv::SVD::compute(A, w, u, vt, MODIFY_A|FULL_UV) on a 4x4 float matrix: OpenCV's one-sided Jacobi (JacobiSVDImpl_<float>)
// on A^T, in registers. w and vt only.
__device__ __forceinline__ void svd4(const float* A, float* w_out, float (&Vt)[4][4]) {
    float At[4][4];
    double W[4];
    const float eps = FLT_EPSILON * 2;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) At[i][k] = A[k * 4 + i];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        double sd = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) sd = da(sd, dm((double)At[i][k], (double)At[i][k]));
        W[i] = sd;
#pragma unroll
        for (int k = 0; k < 4; k++) Vt[i][k] = (i == k) ? 1.f : 0.f;
    }
    for (int iter = 0; iter < 30; iter++) {
        bool changed = false;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = i + 1; j < 4; j++) {
                double a = W[i], p = 0, b = W[j];
#pragma unroll
                for (int k = 0; k < 4; k++) p = da(p, dm((double)At[i][k], (double)At[j][k]));
                if (fabs(p) <= dm((double)eps, __dsqrt_rn(dm(a, b)))) continue;
                p = dm(p, 2.0);
                const double beta = ds(a, b), gamma = cv_hypot(p, beta);
                float c, s;
                if (beta < 0) {
                    const double delta = dm(ds(gamma, beta), 0.5);
                    s = __double2float_rn(__dsqrt_rn(dd(delta, gamma)));
                    c = __double2float_rn(dd(p, dm(dm(gamma, (double)s), 2.0)));
                } else {
                    c = __double2float_rn(__dsqrt_rn(dd(da(gamma, beta), dm(gamma, 2.0))));
                    s = __double2float_rn(dd(p, dm(dm(gamma, (double)c), 2.0)));
                }
                a = 0; b = 0;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float t0 = fa(fm(c, At[i][k]), fm(s, At[j][k]));
                    const float t1 = fa(fm(-s, At[i][k]), fm(c, At[j][k]));
                    At[i][k] = t0; At[j][k] = t1;
                    a = da(a, dm((double)t0, (double)t0));
                    b = da(b, dm((double)t1, (double)t1));
                }
                W[i] = a; W[j] = b;
                changed = true;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float t0 = fa(fm(Vt[i][k], c), fm(Vt[j][k], s));
                    const float t1 = fs(fm(Vt[j][k], c), fm(Vt[i][k], s));
                    Vt[i][k] = t0; Vt[j][k] = t1;
                }
            }
        if (!changed) break;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        double sd = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) sd = da(sd, dm((double)At[i][k], (double)At[i][k]));
        W[i] = __dsqrt_rn(sd);
    }
    // descending selection sort; swaps are register moves by predicate so the arrays stay in registers
#pragma unroll
    for (int i = 0; i < 3; i++) {
        int j = i;
        double wj = W[i];
#pragma unroll
        for (int k = i + 1; k < 4; k++)
            if (wj < W[k]) { j = k; wj = W[k]; }
#pragma unroll
        for (int k = i + 1; k < 4; k++)
            if (j == k) {
                const double tw = W[i]; W[i] = W[k]; W[k] = tw;
#pragma unroll
                for (int q = 0; q < 4; q++) { const float tv = Vt[i][q]; Vt[i][q] = Vt[k][q]; Vt[k][q] = tv; }
            }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) w_out[i] = __double2float_rn(W[i]);
}

// cvu::triangulate: A rows = fma(x, P.row(2), -P.row(0)) (cv::addWeighted), SVD, vt.row(3), then x3D / w as
// convertTo(scale = 1./w): x * (float)(1.0 / w) + 0.
__device__ __forceinline__ F3 triangulate(float x1, float y1, float x2, float y2, const float* P1, const float* P2) {
    float A[16], w[4], Vt[4][4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        A[k] = __fmaf_rn(x1, P1[8 + k], -P1[k]);
        A[4 + k] = __fmaf_rn(y1, P1[8 + k], -P1[4 + k]);
        A[8 + k] = __fmaf_rn(x2, P2[8 + k], -P2[k]);
        A[12 + k] = __fmaf_rn(y2, P2[8 + k], -P2[4 + k]);
    }
    svd4(A, w, Vt);
    const double inv = dd(1.0, (double)Vt[3][3]);
    float r[3];
    if (fabs(inv) == 1.0) {
#pragma unroll
        for (int k = 0; k < 3; k++) r[k] = fa(__double2float_rn(dm((double)Vt[3][k], inv)), 0.f);
    } else {
        const float a = __double2float_rn(inv);
#pragma unroll
        for (int k = 0; k < 3; k++) r[k] = fa(fm(Vt[3][k], a), 0.f);
    }
    return {r[0], r[1], r[2]};
}

// cv::Rodrigues of a float rotation vector: double arithmetic, rounded to float
__device__ __forceinline__ void rodrigues(const float* rv, float* R) {
    double rx = rv[0], ry = rv[1], rz = rv[2];
    const double theta = __dsqrt_rn(da(da(dm(rx, rx), dm(ry, ry)), dm(rz, rz)));
    if (theta < DBL_EPSILON) {
#pragma unroll
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.f : 0.f;
        return;
    }
    double s, c;
    sincos(theta, &s, &c);
    const double c1 = ds(1.0, c);
    const double itheta = theta != 0.0 ? dd(1.0, theta) : 0.0;
    rx = dm(rx, itheta); ry = dm(ry, itheta); rz = dm(rz, itheta);
    const double rrt[9] = {dm(rx, rx), dm(rx, ry), dm(rx, rz), dm(rx, ry), dm(ry, ry), dm(ry, rz), dm(rx, rz), dm(ry, rz), dm(rz, rz)};
    const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
#pragma unroll
    for (int i = 0; i < 9; i++) {
        const double e = (i % 4 == 0) ? 1.0 : 0.0;
        R[i] = __double2float_rn(da(da(dm(c, e), dm(c1, rrt[i])), dm(s, r_x[i])));
    }
}

// Track::calcSE3toXYZInfo (Track.cpp:259-306); a null info1 / info2 skips that half
__device__ __forceinline__ void xyz_info(F3 xyz1, const float* Tcw1, const float* Tcw2, float fx, double* info1, double* info2) {
    float T1i[16], T2i[16];
    inv4(Tcw1, T1i);
    inv4(Tcw2, T2i);
    const F3 O1 = {T1i[3], T1i[7], T1i[11]}, O2 = {T2i[3], T2i[7], T2i[11]};
    const F3 xyz = se3map(T1i, xyz1);
    const F3 vO1 = sub3(xyz, O1), vO2 = sub3(xyz, O2);
    const float sinParallax = __double2float_rn(dd(norm3(cross3(vO1, vO2)), dm(norm3(vO1), norm3(vO2))));
    const F3 xyz2 = se3map(Tcw2, xyz);
    const float length1 = __double2float_rn(norm3(xyz1)), length2 = __double2float_rn(norm3(xyz2));
    const float dxy1 = fd(fm(2.f, length1), fx), dxy2 = fd(fm(2.f, length2), fx);
    const float dz1 = fd(dxy2, sinParallax), dz2 = fd(dxy1, sinParallax);
    const float d1[3] = {fd(1.f, fm(dxy1, dxy1)), fd(1.f, fm(dxy1, dxy1)), fd(1.f, fm(dz1, dz1))};
    const float d2[3] = {fd(1.f, fm(dxy2, dxy2)), fd(1.f, fm(dxy2, dxy2)), fd(1.f, fm(dz2, dz2))};
    const F3 xx[2] = {xyz1, xyz2};
    const float len[2] = {length1, length2};
    const float* dg[2] = {d1, d2};
    double* out[2] = {info1, info2};
#pragma unroll
    for (int v = 0; v < 2; v++) {
        if (!out[v]) continue;
        const F3 z = {0.f, 0.f, len[v]};
        const F3 k = cross3(xx[v], z);
        const float normk = __double2float_rn(norm3(k));
        const float sinv = __double2float_rn(dd((double)normk, dm(norm3(z), norm3(xx[v]))));
        const float f = fd(asinf_host(sinv), normk);
        const float kv[3] = {fm(k.x, f), fm(k.y, f), fm(k.z, f)};
        float R[9];
        rodrigues(kv, R);
        // R.t() * info (generic gemm, double sums; info is diagonal with +0 off the diagonal), then (...) * R (small path)
        float I[9] = {dg[v][0], 0.f, 0.f, 0.f, dg[v][1], 0.f, 0.f, 0.f, dg[v][2]};
        float tmp[9];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                double s = 0;
#pragma unroll
                for (int q = 0; q < 3; q++) s = da(s, dm((double)R[q * 3 + i], (double)I[q * 3 + j]));
                tmp[i * 3 + j] = __double2float_rn(dm(s, 1.0));
            }
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) out[v][i * 3 + j] = (double)gemm3_elem(tmp, 3, i, R, 3, j, 1.0);
    }
}

// warp-aggregated counter: one atomic per warp
__device__ __forceinline__ void warp_count(int* counter, bool pred) {
    const unsigned b = __ballot_sync(0xffffffffu, pred);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(counter, __popc(b));
}

__global__ void __launch_bounds__(kBlock) k_triangulate(int n, const float* __restrict__ pt1, const float* __restrict__ pt2,
                                                        const float* __restrict__ P, const int* __restrict__ idx1,
                                                        const int* __restrict__ idx2, float* __restrict__ xyz) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float P1[12], P2[12];
    const float* p1 = P + 12 * idx1[i];
    const float* p2 = P + 12 * idx2[i];
#pragma unroll
    for (int k = 0; k < 12; k++) { P1[k] = p1[k]; P2[k] = p2[k]; }
    const F3 r = triangulate(pt1[2 * i], pt1[2 * i + 1], pt2[2 * i], pt2[2 * i + 1], P1, P2);
    xyz[3 * i] = r.x; xyz[3 * i + 1] = r.y; xyz[3 * i + 2] = r.z;
}

// Track::doTriangulate for B streams, stream b on blockIdx.y: its keyframe keypoints, matches, good-parallax flags and local
// map points at b * cap, its frame keypoints at b * cap_fr, its Tcr at 16 b and its counts at 2 b. A stream whose gate is 0
// (the nMinFrames early return) leaves every output untouched.
__global__ void __launch_bounds__(kBlock) k_track_triangulate(se2gpu::TrackTriArgs a) {
    const int b = blockIdx.y;
    if (a.gate && !a.gate[b]) return;
    const size_t base = (size_t)b * a.cap;
    const se2gpu_keypoint* __restrict__ kp_kf = a.kp_kf + base;
    const se2gpu_keypoint* __restrict__ kp_fr = a.kp_fr + (size_t)b * a.cap_fr;
    int* __restrict__ matches = a.matches + base;
    const uint8_t* __restrict__ observed = a.observed_tab ? a.observed_tab[b] : a.observed + base;
    const float* __restrict__ view_mp = a.view_mp_tab ? a.view_mp_tab[b] : a.view_mp + 3 * base;
    float* __restrict__ local_mps = a.local_mps + 3 * base;
    uint8_t* __restrict__ good_prl = a.good_prl + base;
    int* __restrict__ counts = a.counts + 2 * b;
    // P_KF = Config::PrjMtrxEye, P = Kcam * Tcr.rowRange(0,3) and Ocam = inv(Tcr).col(3) are the same for the whole stream:
    // one thread per block builds them in shared memory
    __shared__ float sP[24], sO[3];
    if (threadIdx.x == 0) {
        float Tcr[16], K[9], Ti[16];
#pragma unroll
        for (int k = 0; k < 16; k++) Tcr[k] = a.Tcr[16 * b + k];
#pragma unroll
        for (int k = 0; k < 9; k++) K[k] = a.K[k];
        const float eye34[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
        projection(K, eye34, sP);
        projection(K, Tcr, sP + 12);
        inv4(Tcr, Ti);
        sO[0] = Ti[3]; sO[1] = Ti[7]; sO[2] = Ti[11];
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = count_of(a.d_n ? a.d_n + b : nullptr, a.cap);
    bool tracked = false, good = false;
    if (i < n) {
        good_prl[i] = 0;
        const int m = matches[i];
        if (m >= 0) {
            if (observed[i]) {
                local_mps[3 * i] = view_mp[3 * i]; local_mps[3 * i + 1] = view_mp[3 * i + 1]; local_mps[3 * i + 2] = view_mp[3 * i + 2];
                tracked = true;
            } else {
                float P_KF[12], P[12];
#pragma unroll
                for (int k = 0; k < 12; k++) { P_KF[k] = sP[k]; P[k] = sP[12 + k]; }
                const se2gpu_keypoint p = kp_kf[i], q = kp_fr[m];
                const F3 pos = triangulate(p.x, p.y, q.x, q.y, P_KF, P);
                if (pos.z >= a.lower && pos.z <= a.upper) {
                    local_mps[3 * i] = pos.x; local_mps[3 * i + 1] = pos.y; local_mps[3 * i + 2] = pos.z;
                    // cvu::checkParallax(0, Ocam, pos, deg)
                    const F3 p1 = sub3(pos, {0.f, 0.f, 0.f}), p2 = sub3(pos, {sO[0], sO[1], sO[2]});
                    const float cosp = __double2float_rn(dd(fabs((double)dot3(p1, p2)), dm(norm3(p1), norm3(p2))));
                    if (cosp < a.min_cos) { good = true; good_prl[i] = 1; }
                } else {
                    matches[i] = -1;
                }
            }
        }
    }
    warp_count(counts, tracked);
    warp_count(counts + 1, good);
}

__global__ void __launch_bounds__(kBlock) k_xyz_info(int n, const float* __restrict__ xyz1, const int* __restrict__ pose1,
                                                     const int* __restrict__ pose2, const float* __restrict__ Tcw, float fx,
                                                     double* __restrict__ info1, double* __restrict__ info2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float T1[16], T2[16];
    const float* a = Tcw + 16 * pose1[i];
    const float* b = Tcw + 16 * pose2[i];
#pragma unroll
    for (int k = 0; k < 16; k++) { T1[k] = a[k]; T2[k] = b[k]; }
    double o1[9], o2[9];
    xyz_info({xyz1[3 * i], xyz1[3 * i + 1], xyz1[3 * i + 2]}, T1, T2, fx, o1, o2);
#pragma unroll
    for (int k = 0; k < 9; k++) { info1[9 * i + k] = o1[k]; info2[9 * i + k] = o2[k]; }
}

struct MpTable {
    const float* main_measure; const int* main_pose; const int* main_octave; const float* normal;
    const float* min_dist; const float* max_dist;
};

__global__ void __launch_bounds__(kBlock) k_projection_observations(
    const se2gpu_keypoint* __restrict__ kf_kp, int cap, const int* __restrict__ d_n, const int* __restrict__ match_mp,
    const float* __restrict__ Tnew_g, MpTable mp, const float* __restrict__ Tcw_table, const float* __restrict__ K_g,
    float lower, float upper, float fx, uint8_t* __restrict__ accept, float* __restrict__ pos_out, double* __restrict__ info_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count_of(d_n, cap)) return;
    accept[i] = 0;
    const int m = match_mp[i];
    if (m < 0) return;
    float Tn[16], Tm[16], K[9], P1[12], P2[12];
    const float* tm = Tcw_table + 16 * mp.main_pose[m];
#pragma unroll
    for (int k = 0; k < 16; k++) { Tn[k] = Tnew_g[k]; Tm[k] = tm[k]; }
#pragma unroll
    for (int k = 0; k < 9; k++) K[k] = K_g[k];
    projection(K, Tm, P1);
    projection(K, Tn, P2);
    const se2gpu_keypoint kp = kf_kp[i];
    const F3 x3d = triangulate(mp.main_measure[2 * m], mp.main_measure[2 * m + 1], kp.x, kp.y, P1, P2);
    const F3 pos = se3map(Tn, x3d);
    // MapPoint::acceptNewObserve
    const F3 nv = {mp.normal[3 * m], mp.normal[3 * m + 1], mp.normal[3 * m + 2]};
    const float dist = __double2float_rn(norm3(pos));
    const float cosAngle = __double2float_rn(dd(fabs((double)dot3(pos, nv)), dm((double)dist, norm3(nv))));
    const bool c1 = abs(mp.main_octave[m] - kp.octave) <= 2;
    const bool c2 = cosAngle >= 0.866f;
    const bool c3 = dist >= mp.min_dist[m] && dist <= mp.max_dist[m];
    if (!(c1 && c2 && c3)) return;
    if (pos.z > upper || pos.z < lower) return;
    double info[9];
    xyz_info(pos, Tn, Tm, fx, info, nullptr);
    pos_out[3 * i] = pos.x; pos_out[3 * i + 1] = pos.y; pos_out[3 * i + 2] = pos.z;
#pragma unroll
    for (int k = 0; k < 9; k++) info_out[9 * i + k] = info[k];
    accept[i] = 1;
}

__global__ void k_debug_svd4(int n, const float* __restrict__ A, float* __restrict__ w, float* __restrict__ vt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float a[16], ww[4], V[4][4];
#pragma unroll
    for (int k = 0; k < 16; k++) a[k] = A[16 * i + k];
    svd4(a, ww, V);
#pragma unroll
    for (int k = 0; k < 4; k++) w[4 * i + k] = ww[k];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int k = 0; k < 4; k++) vt[16 * i + 4 * r + k] = V[r][k];
}

inline int blocks(int n) { return (n + kBlock - 1) / kBlock; }

const float kMinCos[4] = {0.9998f, 0.9994f, 0.9986f, 0.9976f};   // cvu::checkParallax

// ------------------------------------------------------------------------------------------ map-point updates (DESIGN.md section 13)
// One warp per map point. A list of up to kMpCap entries keeps its descriptor distance matrix in the warp's shared memory;
// a longer one recomputes distances row by row instead (the same median, found by bisection over the 257 distance values).
constexpr int kMpWarps = 4;
constexpr int kMpCap = 32;
constexpr int kMpMaxList = (1 << 22) - 1;        // list positions share a 32-bit key with a median of at most 256
constexpr unsigned kFull = 0xffffffffu;

// Point m's list and updates are well-formed: every observation inside the keyframe and slot tables (with an octave below
// nlevels when nlevels > 0), main_kf in [-1, K), and each update position inside the list and not repeated.
__host__ __device__ inline bool mp_point_ok(const se2gpu_mp_keyframes& kf, const se2gpu_mp_points& mp, const int* upd_ptr,
                                            const int* upd_pos, int nlevels, int m) {
    const int p0 = mp.obs_ptr[m], p1 = mp.obs_ptr[m + 1];
    if (p0 < 0 || p1 < p0 || p1 - p0 > kMpMaxList) return false;
    for (int j = p0; j < p1; ++j) {
        const int k = mp.obs_kf[j], idx = mp.obs_idx[j];
        if (k < 0 || k >= kf.n_kf || idx < 0) return false;
        const long long slot = (long long)kf.kp_base[k] + idx;
        if (kf.kp_base[k] < 0 || slot >= kf.n_slots) return false;
        if (nlevels > 0 && (kf.kp[slot].octave < 0 || kf.kp[slot].octave >= nlevels)) return false;
    }
    if (!upd_ptr) return true;
    if (mp.main_kf[m] < -1 || mp.main_kf[m] >= kf.n_kf) return false;
    const int u0 = upd_ptr[m], u1 = upd_ptr[m + 1];
    if (u0 < 0 || u1 < u0) return false;
    for (int u = u0; u < u1; ++u) {
        if (upd_pos[u] < 0 || upd_pos[u] >= p1 - p0) return false;
        for (int v = u0; v < u; ++v)
            if (upd_pos[v] == upd_pos[u]) return false;
    }
    return true;
}

__global__ void __launch_bounds__(kBlock) k_mp_check(se2gpu_mp_keyframes kf, se2gpu_mp_points mp, const int* __restrict__ upd_ptr,
                                                     const int* __restrict__ upd_pos, int nlevels, int n,
                                                     const int* __restrict__ points, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && (mp.obs_ptr[0] != 0 || (upd_ptr && upd_ptr[0] != 0))) *status = SE2GPU_ERR_INVALID;
    if (i >= n) return;
    const int m = points ? points[i] : i;
    if (m < 0 || m >= mp.n_mp || !mp_point_ok(kf, mp, upd_ptr, upd_pos, nlevels, m)) *status = SE2GPU_ERR_INVALID;
}

// Which list positions of a point are present while its update u runs. add: the list given is the list after every
// insertion, so the positions of later updates are absent, and after an abandonment (setNull at update `clear`) only the
// insertions since then are present. erase: the list given is the list before the call, so every position erased so far
// (this update's included) is absent.
struct MpList {
    const int* pos;
    int u0, u1, u, clear;
    bool add;
    __device__ __forceinline__ bool has(int j) const {
        if (!add) {
            for (int v = u0; v <= u; ++v)
                if (pos[v] == j) return false;
            return true;
        }
        for (int v = u + 1; v < u1; ++v)
            if (pos[v] == j) return false;
        if (clear < 0) return true;
        for (int v = clear + 1; v <= u; ++v)
            if (pos[v] == j) return true;
        return false;
    }
};

__device__ __forceinline__ int mp_slot(const se2gpu_mp_keyframes& kf, const se2gpu_mp_points& mp, int j) {
    return kf.kp_base[mp.obs_kf[j]] + mp.obs_idx[j];
}

// number of present entries of a list of L (warp-uniform)
__device__ int mp_count(const MpList& ls, int L, int lane) {
    int n = 0;
    for (int j0 = 0; j0 < L; j0 += 32) n += __popc(__ballot_sync(kFull, j0 + lane < L && ls.has(j0 + lane)));
    return n;
}

// p = o * (1.f / cv::norm(o)): the float / double quotient is a double, and Point3f * double rounds each product once
__device__ __forceinline__ F3 mp_unit(F3 o) {
    const double s = dd(1.0, norm3(o));
    return {__double2float_rn(dm((double)o.x, s)), __double2float_rn(dm((double)o.y, s)), __double2float_rn(dm((double)o.z, s))};
}

// Rcw^T * M * Rcw as the float MatExpr evaluates it: cv::gemm(R, M, GEMM_1_T) (double sums), then (...) * R (small path).
// T is the 4x4 pose, M a row-major 3x3.
__device__ __forceinline__ void rt_m_r(const float* T, const float* M, float* out) {
    float tmp[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            double s = 0;
#pragma unroll
            for (int q = 0; q < 3; q++) s = da(s, dm((double)T[q * 4 + i], (double)M[q * 3 + j]));
            tmp[i * 3 + j] = __double2float_rn(dm(s, 1.0));
        }
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) out[i * 3 + j] = gemm3_elem(tmp, 3, i, T, 4, j, 1.0);
}

// Rcw * M * Rcw^T: R * M (small path), then cv::gemm(..., R, GEMM_2_T) (double sums)
__device__ __forceinline__ void r_m_rt(const float* T, const float* M, float* out) {
    float tmp[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) tmp[i * 3 + j] = gemm3_elem(T, 4, i, M, 3, j, 1.0);
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            double s = 0;
#pragma unroll
            for (int q = 0; q < 3; q++) s = da(s, dm((double)tmp[i * 3 + q], (double)T[j * 4 + q]));
            out[i * 3 + j] = __double2float_rn(dm(s, 1.0));
        }
}

// Per-warp shared memory of the short-list median: the distance matrix and the compacted slots / list positions
struct MpShared {
    unsigned short dist[kMpCap * kMpCap];
    int slot[kMpCap], pos[kMpCap];
};

// MapPoint::updateMainKFandDescriptor (MapPoint.cpp:228-292) over the present entries of point m's list
__device__ void mp_update_main(const se2gpu_mp_keyframes& kf, const se2gpu_mp_points& mp, const se2gpu_mp_params& prm, int m,
                               int p0, int L, const MpList& ls, MpShared& sh, int lane) {
    if (mp.null[m]) return;
    const uint32_t* desc = reinterpret_cast<const uint32_t*>(kf.desc);
    auto valid = [&](int j) { return ls.has(j) && !kf.kf_null[mp.obs_kf[p0 + j]]; };
    int key = INT_MAX;
    if (L <= kMpCap) {
        const bool v = lane < L && valid(lane);
        const unsigned b = __ballot_sync(kFull, v);
        const int N = __popc(b);
        if (N == 0) return;
        if (v) {
            const int c = __popc(b & ((1u << lane) - 1));
            sh.slot[c] = mp_slot(kf, mp, p0 + lane);
            sh.pos[c] = lane;
        }
        __syncwarp();
        hamming_matrix(desc, [&sh](int i) { return sh.slot[i]; }, N, sh.dist, lane, 32);
        __syncwarp();
        const int kth = (int)(0.5 * (N - 1));
        if (lane < N) key = (rank_select(sh.dist + lane * N, N, kth) << 22) | sh.pos[lane];
        __syncwarp();
    } else {
        int N = 0;
        for (int j0 = 0; j0 < L; j0 += 32) N += __popc(__ballot_sync(kFull, j0 + lane < L && valid(j0 + lane)));
        if (N == 0) return;
        const int kth = (int)(0.5 * (N - 1));
        for (int j = 0; j < L; ++j) {
            if (!valid(j)) continue;
            const uint32_t* dj = desc + 8 * (size_t)mp_slot(kf, mp, p0 + j);
            int lo = 0, hi = 256;                  // the least v with more than kth distances <= v
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                int c = 0;
                for (int t = lane; t < L; t += 32)
                    if (valid(t)) c += (t == j ? 0 : hamming256(dj, desc + 8 * (size_t)mp_slot(kf, mp, p0 + t))) <= mid;
                c = __reduce_add_sync(kFull, c);
                if (c > kth) hi = mid; else lo = mid + 1;
            }
            key = min(key, (lo << 22) | j);
        }
    }
    // lexicographic (median, position): the first entry of the least median (:264-267)
    const int jb = __reduce_min_sync(kFull, key) & kMpMaxList;
    const int k = mp.obs_kf[p0 + jb], slot = mp_slot(kf, mp, p0 + jb);
    if (lane < 8) reinterpret_cast<uint32_t*>(mp.main_desc)[8 * (size_t)m + lane] = desc[8 * (size_t)slot + lane];
    if (lane == 0) {
        const se2gpu_keypoint p = kf.kp[slot];
        mp.main_measure[2 * m] = p.x; mp.main_measure[2 * m + 1] = p.y;
        const int cur = mp.main_kf[m];
        if (!(cur >= 0 && kf.kf_id[cur] == kf.kf_id[k])) {
            mp.main_kf[m] = k;
            mp.main_octave[m] = p.octave;
            const float scale = prm.scale_factors[p.octave];
            mp.level_scale[m] = scale;
            const float dist = __double2float_rn(norm3({kf.view_mp[3 * slot], kf.view_mp[3 * slot + 1], kf.view_mp[3 * slot + 2]}));
            const float mx = fm(dist, scale);
            mp.max_dist[m] = mx;
            mp.min_dist[m] = fd(mx, prm.scale_factors[prm.nlevels - 1]);
        }
    }
    __syncwarp();
}

// MapPoint::updateParallax(pKF) (MapPoint.cpp:124-185) for the entry at list position q; `size` is the present count.
// Returns true when it abandons the point.
__device__ bool mp_update_parallax(const se2gpu_mp_keyframes& kf, const se2gpu_mp_points& mp, const se2gpu_mp_params& prm, int m,
                                   int p0, int L, const MpList& ls, int q, int size, int lane) {
    if (mp.good_prl[m] || size <= 2) return false;
    // pKF0: the least mIdKF among the observers at most 6 ids older than pKF (null keyframes included), first entry on ties
    const int idn = kf.kf_id[mp.obs_kf[p0 + q]];
    int best_id = INT_MAX, best_j = INT_MAX;
    for (int j = lane; j < L; j += 32) {
        const int id = kf.kf_id[mp.obs_kf[p0 + j]];
        if (ls.has(j) && idn - id <= 6 && id < best_id) { best_id = id; best_j = j; }
    }
    const int id0 = __reduce_min_sync(kFull, best_id);
    const int j0 = (int)__reduce_min_sync(kFull, (unsigned)(best_id == id0 ? best_j : INT_MAX));
    const int k0 = mp.obs_kf[p0 + j0], k1 = mp.obs_kf[p0 + q];
    const int s0 = mp_slot(kf, mp, p0 + j0), s1 = mp_slot(kf, mp, p0 + q);
    bool ok = false;
    F3 posW = {0.f, 0.f, 0.f};
    float W[9];
    if (lane == 0) {
        float T0[16], T1[16], K[9], P0[12], P1[12];
#pragma unroll
        for (int i = 0; i < 16; i++) { T0[i] = kf.Tcw[16 * k0 + i]; T1[i] = kf.Tcw[16 * k1 + i]; }
#pragma unroll
        for (int i = 0; i < 9; i++) K[i] = prm.K[i];
        projection(K, T0, P0);
        projection(K, T1, P1);
        const se2gpu_keypoint a = kf.kp[s0], b = kf.kp[s1];
        posW = triangulate(a.x, a.y, b.x, b.y, P0, P1);
        const F3 pos0 = se3map(T0, posW), pos1 = se3map(T1, posW);
        if (pos0.z >= prm.lower_depth && pos0.z <= prm.upper_depth && pos1.z >= prm.lower_depth && pos1.z <= prm.upper_depth) {
            float Ti0[16], Ti1[16];
            inv4(T0, Ti0);
            inv4(T1, Ti1);
            const F3 v0 = sub3(posW, {Ti0[3], Ti0[7], Ti0[11]}), v1 = sub3(posW, {Ti1[3], Ti1[7], Ti1[11]});
            const float cosp = __double2float_rn(dd(fabs((double)dot3(v0, v1)), dm(norm3(v0), norm3(v1))));
            ok = cosp < 0.9994f;                 // checkParallax(..., 2)
            if (ok) {
                mp.pos[3 * m] = posW.x; mp.pos[3 * m + 1] = posW.y; mp.pos[3 * m + 2] = posW.z;
                mp.good_prl[m] = 1;
                double info0[9], info1[9];
                xyz_info(pos0, T0, T1, prm.fx, info0, info1);
                const F3 pv[2] = {pos0, pos1};
                const double* iv[2] = {info0, info1};
                const int sv[2] = {s0, s1};
                for (int v = 0; v < 2; v++) {      // setViewMP of pKF0, then of pKF (the same slot when pKF0 == pKF)
                    kf.view_mp[3 * sv[v]] = pv[v].x; kf.view_mp[3 * sv[v] + 1] = pv[v].y; kf.view_mp[3 * sv[v] + 2] = pv[v].z;
#pragma unroll
                    for (int e = 0; e < 9; e++) kf.view_info[9 * sv[v] + e] = iv[v][e];
                }
                float M0[9];
#pragma unroll
                for (int e = 0; e < 9; e++) M0[e] = (float)info0[e];    // toCvMat(Matrix3d): the float values, exactly
                rt_m_r(T0, M0, W);
            }
        }
    }
    ok = __shfl_sync(kFull, ok, 0);
    if (ok) {
        posW = {__shfl_sync(kFull, posW.x, 0), __shfl_sync(kFull, posW.y, 0), __shfl_sync(kFull, posW.z, 0)};
#pragma unroll
        for (int e = 0; e < 9; e++) W[e] = __shfl_sync(kFull, W[e], 0);
        const int id1 = kf.kf_id[k1];
        for (int j = lane; j < L; j += 32) {       // the other observers
            const int k = mp.obs_kf[p0 + j], id = kf.kf_id[k];
            if (!ls.has(j) || id == id1 || id == id0) continue;
            float Tk[16], Wk[9];
#pragma unroll
            for (int i = 0; i < 16; i++) Tk[i] = kf.Tcw[16 * k + i];
            const F3 pk = se3map(Tk, posW);
            r_m_rt(Tk, W, Wk);
            const int s = mp_slot(kf, mp, p0 + j);
            kf.view_mp[3 * s] = pk.x; kf.view_mp[3 * s + 1] = pk.y; kf.view_mp[3 * s + 2] = pk.z;
#pragma unroll
            for (int e = 0; e < 9; e++) kf.view_info[9 * s + e] = (double)Wk[e];
        }
    }
    __syncwarp();
    if (idn - id0 >= 6 && !ok) {                   // setNull (the point's own side)
        if (lane == 0) { mp.null[m] = 1; mp.good_prl[m] = 0; }
        __syncwarp();
        return true;
    }
    return false;
}

__global__ void __launch_bounds__(kMpWarps * 32) k_mp_add(se2gpu_mp_keyframes kf, se2gpu_mp_points mp, const int* __restrict__ upd_ptr,
                                                          const int* __restrict__ upd_pos, se2gpu_mp_params prm,
                                                          uint8_t* __restrict__ abandoned, const int* __restrict__ status) {
    __shared__ MpShared sh[kMpWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, m = blockIdx.x * kMpWarps + w;
    if (m >= mp.n_mp || *status) return;
    const int p0 = mp.obs_ptr[m], L = mp.obs_ptr[m + 1] - p0;
    MpList ls{upd_pos, upd_ptr[m], upd_ptr[m + 1], 0, -1, true};
    bool gone = false;
    for (int u = ls.u0; u < ls.u1; ++u) {
        ls.u = u;
        const int q = upd_pos[u];
        const int size = mp_count(ls, L, lane);
        mp_update_main(kf, mp, prm, m, p0, L, ls, sh[w], lane);
        if (mp_update_parallax(kf, mp, prm, m, p0, L, ls, q, size, lane)) { gone = true; ls.clear = u; }
        if (lane == 0) {                           // MapPoint.cpp:115-121, with the list size before the insert
            const int s = mp_slot(kf, mp, p0 + q);
            const F3 nn = mp_unit({kf.view_mp[3 * s], kf.view_mp[3 * s + 1], kf.view_mp[3 * s + 2]});
            const float old = (float)(size - 1), f = fd(1.f, (float)size);
            float* n = mp.normal + 3 * m;
            n[0] = fm(fa(fm(n[0], old), nn.x), f);
            n[1] = fm(fa(fm(n[1], old), nn.y), f);
            n[2] = fm(fa(fm(n[2], old), nn.z), f);
            mp.null[m] = 0;
        }
        __syncwarp();
    }
    if (lane == 0) abandoned[m] = gone;
}

__global__ void __launch_bounds__(kMpWarps * 32) k_mp_erase(se2gpu_mp_keyframes kf, se2gpu_mp_points mp, const int* __restrict__ upd_ptr,
                                                            const int* __restrict__ upd_pos, se2gpu_mp_params prm,
                                                            uint8_t* __restrict__ abandoned, const int* __restrict__ status) {
    __shared__ MpShared sh[kMpWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, m = blockIdx.x * kMpWarps + w;
    if (m >= mp.n_mp || *status) return;
    const int p0 = mp.obs_ptr[m], L = mp.obs_ptr[m + 1] - p0;
    MpList ls{upd_pos, upd_ptr[m], upd_ptr[m + 1], 0, -1, false};
    bool gone = false;
    for (int u = ls.u0; u < ls.u1; ++u) {
        ls.u = u;
        const int s = mp_slot(kf, mp, p0 + upd_pos[u]);
        const F3 np = mp_unit({kf.view_mp[3 * s], kf.view_mp[3 * s + 1], kf.view_mp[3 * s + 2]});   // before the erase
        const int size = mp_count(ls, L, lane);
        if (!mp.null[m] && size == 0) {            // setNull
            if (lane == 0) { mp.null[m] = 1; mp.good_prl[m] = 0; }
            gone = true;
        } else {
            mp_update_main(kf, mp, prm, m, p0, L, ls, sh[w], lane);
            if (lane == 0) {
                const float up = (float)(size + 1), f = fd(1.f, (float)size);
                float* n = mp.normal + 3 * m;
                n[0] = fm(fs(fm(n[0], up), np.x), f);
                n[1] = fm(fs(fm(n[1], up), np.y), f);
                n[2] = fm(fs(fm(n[2], up), np.z), f);
            }
        }
        __syncwarp();
    }
    if (lane == 0) abandoned[m] = gone;
}

__global__ void __launch_bounds__(kMpWarps * 32) k_mp_update_measure(se2gpu_mp_keyframes kf, se2gpu_mp_points mp, int n,
                                                                     const int* __restrict__ points, const int* __restrict__ status) {
    const int i = blockIdx.x * kMpWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n || *status) return;
    const int m = points[i];
    const F3 pos = {mp.pos[3 * m], mp.pos[3 * m + 1], mp.pos[3 * m + 2]};
    for (int j = mp.obs_ptr[m] + lane; j < mp.obs_ptr[m + 1]; j += 32) {
        const int k = mp.obs_kf[j];
        if (kf.kf_null[k]) continue;
        float T[16];
#pragma unroll
        for (int e = 0; e < 16; e++) T[e] = kf.Tcw[16 * k + e];
        const F3 p = se3map(T, pos);
        const int s = mp_slot(kf, mp, j);
        kf.view_mp[3 * s] = p.x; kf.view_mp[3 * s + 1] = p.y; kf.view_mp[3 * s + 2] = p.z;
    }
}

bool mp_tables_set(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, bool updates) {
    if (!kf || !mp || kf->n_kf < 0 || kf->n_slots < 0 || mp->n_mp < 0 || !mp->obs_ptr) return false;
    if (kf->n_kf && (!kf->kf_id || !kf->kf_null || !kf->Tcw || !kf->kp_base)) return false;
    if (kf->n_slots && (!kf->view_mp || (updates && (!kf->kp || !kf->desc || !kf->view_info)))) return false;
    if (mp->n_mp && (!mp->pos || (updates && (!mp->good_prl || !mp->null || !mp->main_kf || !mp->main_desc || !mp->main_octave ||
                                              !mp->main_measure || !mp->level_scale || !mp->normal || !mp->min_dist || !mp->max_dist))))
        return false;
    return true;
}

int mp_updates_device(bool add, const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* d_upd_ptr,
                      const int* d_upd_pos, const se2gpu_mp_params* prm, uint8_t* d_abandoned, int* d_status, void* stream) {
    if (!mp_tables_set(kf, mp, true) || !prm || !d_status || !d_upd_ptr || (mp->n_mp && (!d_upd_pos || !d_abandoned)))
        return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (prm->nlevels < 1 || prm->nlevels > SE2GPU_MP_MAX_LEVELS) return fail(SE2GPU_ERR_INVALID, "nlevels out of range");
    { const int rc = require_device(); if (rc) return rc; }
    cudaStream_t s = (cudaStream_t)stream;
    SE2_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int), s));
    SE2_LAUNCH(k_mp_check, blocks(std::max(mp->n_mp, 1)), kBlock, 0, s, *kf, *mp, d_upd_ptr, d_upd_pos, prm->nlevels, mp->n_mp,
               nullptr, d_status);
    if (mp->n_mp) {
        const int grid = (mp->n_mp + kMpWarps - 1) / kMpWarps;
        if (add) SE2_LAUNCH(k_mp_add, grid, kMpWarps * 32, 0, s, *kf, *mp, d_upd_ptr, d_upd_pos, *prm, d_abandoned, d_status);
        else SE2_LAUNCH(k_mp_erase, grid, kMpWarps * 32, 0, s, *kf, *mp, d_upd_ptr, d_upd_pos, *prm, d_abandoned, d_status);
    }
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

// Host form of both updates: the same checks on the host, then every table through the stage
int mp_updates_host(bool add, const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* upd_ptr, const int* upd_pos,
                    const se2gpu_mp_params* prm, uint8_t* abandoned, int device) {
    if (!mp_tables_set(kf, mp, true) || !prm || !upd_ptr || (mp->n_mp && !abandoned)) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (prm->nlevels < 1 || prm->nlevels > SE2GPU_MP_MAX_LEVELS) return fail(SE2GPU_ERR_INVALID, "nlevels out of range");
    const int M = mp->n_mp;
    if (mp->obs_ptr[0] != 0 || upd_ptr[0] != 0) return fail(SE2GPU_ERR_INVALID, "obs_ptr[0] and upd_ptr[0] must be 0");
    if (M && upd_ptr[M] > 0 && !upd_pos) return fail(SE2GPU_ERR_INVALID, "null upd_pos");
    for (int m = 0; m < M; ++m)
        if (!mp_point_ok(*kf, *mp, upd_ptr, upd_pos, prm->nlevels, m)) return fail(SE2GPU_ERR_INVALID, "map point %d: index out of range or repeated update", m);
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (M == 0) return SE2GPU_OK;
    const size_t K = kf->n_kf, S = kf->n_slots, nobs = mp->obs_ptr[M], nupd = upd_ptr[M];
    auto up = [&](auto* p, size_t n) { using T = std::remove_cv_t<std::remove_pointer_t<decltype(p)>>; return n ? st.upload(p, n) : st.scratch<T>(1); };
    auto io = [&](auto* p, size_t n) { using T = std::remove_pointer_t<decltype(p)>; return n ? st.inout(p, n) : st.scratch<T>(1); };
    se2gpu_mp_keyframes dk{kf->n_kf, up(kf->kf_id, K), up(kf->kf_null, K), up(kf->Tcw, 16 * K), up(kf->kp_base, K), kf->n_slots,
                           up(kf->kp, S), up(kf->desc, 32 * S), io(kf->view_mp, 3 * S), io(kf->view_info, 9 * S)};
    se2gpu_mp_points dm{M, io(mp->pos, 3 * (size_t)M), io(mp->good_prl, M), io(mp->null, M), io(mp->main_kf, M),
                        io(mp->main_desc, 32 * (size_t)M), io(mp->main_octave, M), io(mp->main_measure, 2 * (size_t)M),
                        io(mp->level_scale, M), io(mp->normal, 3 * (size_t)M), io(mp->min_dist, M), io(mp->max_dist, M),
                        up(mp->obs_ptr, (size_t)M + 1), up(mp->obs_kf, nobs), up(mp->obs_idx, nobs)};
    const int* d_ptr = up(upd_ptr, (size_t)M + 1);
    const int* d_pos = up(upd_pos, nupd);
    uint8_t* d_ab = st.output(abandoned, M);
    int* d_status = st.scratch<int>(1);
    if (const int rc = st.status()) return rc;
    { const int rc = mp_updates_device(add, &dk, &dm, d_ptr, d_pos, prm, d_ab, d_status, nullptr); if (rc) return rc; }
    return st.finish();
}

}  // namespace

// ------------------------------------------------------------------------------------------ device-buffer entries
int se2gpu_triangulate_device(int n, const float* d_pt1, const float* d_pt2, const float* d_P, const int* d_idx1,
                              const int* d_idx2, float* d_xyz, void* stream) {
    if (n < 0 || (n && (!d_pt1 || !d_pt2 || !d_P || !d_idx1 || !d_idx2 || !d_xyz))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    if (n == 0) return SE2GPU_OK;
    SE2_LAUNCH(k_triangulate, blocks(n), kBlock, 0, (cudaStream_t)stream, n, d_pt1, d_pt2, d_P, d_idx1, d_idx2, d_xyz);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

namespace se2gpu {
int track_triangulate_launch(const TrackTriArgs& a, int B, cudaStream_t s) {
    SE2_CUDA(cudaMemsetAsync(a.counts, 0, 2 * sizeof(int) * B, s));
    if (B == 0 || a.cap == 0) return SE2GPU_OK;
    SE2_LAUNCH(k_track_triangulate, dim3(blocks(a.cap), B), kBlock, 0, s, a);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}
float track_min_cos(int min_parallax_deg) { return kMinCos[min_parallax_deg - 1]; }
}  // namespace se2gpu

int se2gpu_track_triangulate_device(const se2gpu_keypoint* d_kp_kf, int n_kf, const int* d_n_kf, const se2gpu_keypoint* d_kp_frame,
                                    int* d_matches12, const uint8_t* d_kf_observed, const float* d_kf_view_mp, const float* d_Tcr,
                                    const float* d_K, float lower_depth, float upper_depth, int min_parallax_deg,
                                    float* d_local_mps, uint8_t* d_good_prl, int* d_counts, void* stream) {
    return se2gpu_track_triangulate_batch_device(1, d_kp_kf, n_kf, d_n_kf, d_kp_frame, 0, d_matches12, d_kf_observed, d_kf_view_mp,
                                                 d_Tcr, nullptr, d_K, lower_depth, upper_depth, min_parallax_deg, d_local_mps,
                                                 d_good_prl, d_counts, stream);
}

int se2gpu_track_triangulate_batch_device(int B, const se2gpu_keypoint* d_kp_kf, int cap, const int* d_n, const se2gpu_keypoint* d_kp_frame,
                                          int cap_frame, int* d_matches12, const uint8_t* d_kf_observed, const float* d_kf_view_mp,
                                          const float* d_Tcr, const int* d_gate, const float* d_K, float lower_depth,
                                          float upper_depth, int min_parallax_deg, float* d_local_mps, uint8_t* d_good_prl,
                                          int* d_counts, void* stream) {
    if (B < 0 || cap < 0 || cap_frame < 0 || !d_counts || min_parallax_deg < 1 || min_parallax_deg > 4 || !d_Tcr || !d_K)
        return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (B && cap && (!d_kp_kf || !d_kp_frame || !d_matches12 || !d_kf_observed || !d_kf_view_mp || !d_local_mps || !d_good_prl))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    if (B > 65535) return fail(SE2GPU_ERR_CAPACITY, "%d streams per call: at most 65535 (the grid's y dimension)", B);
    { const int rc = require_device(); if (rc) return rc; }
    if (B == 0) return SE2GPU_OK;
    TrackTriArgs a{};
    a.kp_kf = d_kp_kf; a.cap = cap; a.d_n = d_n; a.kp_fr = d_kp_frame; a.cap_fr = cap_frame; a.matches = d_matches12;
    a.observed = d_kf_observed; a.view_mp = d_kf_view_mp; a.Tcr = d_Tcr; a.gate = d_gate; a.K = d_K;
    a.lower = lower_depth; a.upper = upper_depth; a.min_cos = kMinCos[min_parallax_deg - 1];
    a.local_mps = d_local_mps; a.good_prl = d_good_prl; a.counts = d_counts;
    return track_triangulate_launch(a, B, (cudaStream_t)stream);
}

int se2gpu_xyz_info_device(int n, const float* d_xyz1, const int* d_pose1, const int* d_pose2, const float* d_Tcw, float fx,
                           double* d_info1, double* d_info2, void* stream) {
    if (n < 0 || (n && (!d_xyz1 || !d_pose1 || !d_pose2 || !d_Tcw || !d_info1 || !d_info2))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    if (n == 0) return SE2GPU_OK;
    SE2_LAUNCH(k_xyz_info, blocks(n), kBlock, 0, (cudaStream_t)stream, n, d_xyz1, d_pose1, d_pose2, d_Tcw, fx, d_info1, d_info2);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_projection_observations_device(const se2gpu_keypoint* d_kf_kp, int n_kf, const int* d_n_kf, const int* d_matches_idx_mp,
                                          const float* d_Tcw_new, const float* d_mp_main_measure, const int* d_mp_main_pose,
                                          const int* d_mp_main_octave, const float* d_mp_normal, const float* d_mp_min_dist,
                                          const float* d_mp_max_dist, const float* d_Tcw_table, const float* d_K, float lower_depth,
                                          float upper_depth, float fx, uint8_t* d_accept, float* d_pos_new_kf, double* d_info_new,
                                          void* stream) {
    if (n_kf < 0) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n_kf && (!d_kf_kp || !d_matches_idx_mp || !d_Tcw_new || !d_mp_main_measure || !d_mp_main_pose || !d_mp_main_octave ||
                 !d_mp_normal || !d_mp_min_dist || !d_mp_max_dist || !d_Tcw_table || !d_K || !d_accept || !d_pos_new_kf || !d_info_new))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    { const int rc = require_device(); if (rc) return rc; }
    if (n_kf == 0) return SE2GPU_OK;
    const MpTable mp{d_mp_main_measure, d_mp_main_pose, d_mp_main_octave, d_mp_normal, d_mp_min_dist, d_mp_max_dist};
    SE2_LAUNCH(k_projection_observations, blocks(n_kf), kBlock, 0, (cudaStream_t)stream, d_kf_kp, n_kf, d_n_kf, d_matches_idx_mp,
               d_Tcw_new, mp, d_Tcw_table, d_K, lower_depth, upper_depth, fx, d_accept, d_pos_new_kf, d_info_new);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

// ------------------------------------------------------------------------------------------ host-buffer entries
namespace {
bool indices_ok(const int* idx, int n, int hi) {
    for (int i = 0; i < n; i++)
        if (idx[i] < 0 || idx[i] >= hi) return false;
    return true;
}
}  // namespace

int se2gpu_triangulate(int n, const float* pt1, const float* pt2, const float* P, int n_proj, const int* idx1, const int* idx2,
                       float* xyz, int device) {
    if (n < 0 || n_proj < 0 || (n && (!pt1 || !pt2 || !P || !idx1 || !idx2 || !xyz))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (!indices_ok(idx1, n, n_proj) || !indices_ok(idx2, n, n_proj)) return fail(SE2GPU_ERR_INVALID, "projection index out of range");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n == 0) return SE2GPU_OK;
    const float* d1 = st.upload(pt1, 2 * (size_t)n);
    const float* d2 = st.upload(pt2, 2 * (size_t)n);
    const float* dP = st.upload(P, 12 * (size_t)n_proj);
    const int* i1 = st.upload(idx1, n);
    const int* i2 = st.upload(idx2, n);
    float* dx = st.output(xyz, 3 * (size_t)n);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_triangulate_device(n, d1, d2, dP, i1, i2, dx, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_track_triangulate(const se2gpu_keypoint* kp_kf, int n_kf, const se2gpu_keypoint* kp_frame, int n_frame, int* matches12,
                             const uint8_t* kf_observed, const float* kf_view_mp, const float* Tcr, const float* K,
                             float lower_depth, float upper_depth, int min_parallax_deg, float* local_mps, uint8_t* good_prl,
                             int* counts, int device) {
    if (n_kf < 0 || n_frame < 0 || !counts || !Tcr || !K || min_parallax_deg < 1 || min_parallax_deg > 4)
        return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n_kf && (!kp_kf || !matches12 || !kf_observed || !kf_view_mp || !local_mps || !good_prl)) return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int i = 0; i < n_kf; i++)
        if (matches12[i] >= n_frame) return fail(SE2GPU_ERR_INVALID, "matches12[%d] = %d is not a frame keypoint", i, matches12[i]);
    if (n_frame && !kp_frame) return fail(SE2GPU_ERR_INVALID, "null argument");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    counts[0] = counts[1] = 0;
    if (n_kf == 0) return SE2GPU_OK;
    const se2gpu_keypoint* dk = st.upload(kp_kf, n_kf);
    const se2gpu_keypoint* df = st.upload(kp_frame, n_frame);
    int* dm12 = st.inout(matches12, n_kf);
    const uint8_t* dobs = st.upload(kf_observed, n_kf);
    const float* dvm = st.upload(kf_view_mp, 3 * (size_t)n_kf);
    const float* dT = st.upload(Tcr, 16);
    const float* dK = st.upload(K, 9);
    float* dl = st.inout(local_mps, 3 * (size_t)n_kf);
    uint8_t* dg = st.output(good_prl, n_kf);
    int* dc = st.output(counts, 2);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_track_triangulate_device(dk, n_kf, nullptr, df, dm12, dobs, dvm, dT, dK, lower_depth, upper_depth,
                                                     min_parallax_deg, dl, dg, dc, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_xyz_info(int n, const float* xyz1, const int* pose1, const int* pose2, const float* Tcw, int n_pose, float fx,
                    double* info1, double* info2, int device) {
    if (n < 0 || n_pose < 0 || (n && (!xyz1 || !pose1 || !pose2 || !Tcw || !info1 || !info2))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (!indices_ok(pose1, n, n_pose) || !indices_ok(pose2, n, n_pose)) return fail(SE2GPU_ERR_INVALID, "pose index out of range");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n == 0) return SE2GPU_OK;
    const float* dx = st.upload(xyz1, 3 * (size_t)n);
    const int* p1 = st.upload(pose1, n);
    const int* p2 = st.upload(pose2, n);
    const float* dT = st.upload(Tcw, 16 * (size_t)n_pose);
    double* i1 = st.output(info1, 9 * (size_t)n);
    double* i2 = st.output(info2, 9 * (size_t)n);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_xyz_info_device(n, dx, p1, p2, dT, fx, i1, i2, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_projection_observations(const se2gpu_keypoint* kf_kp, int n_kf, const int* matches_idx_mp, const float* Tcw_new,
                                   const float* mp_main_measure, const int* mp_main_pose, const int* mp_main_octave,
                                   const float* mp_normal, const float* mp_min_dist, const float* mp_max_dist, int n_mp,
                                   const float* Tcw_table, int n_pose, const float* K, float lower_depth, float upper_depth,
                                   float fx, uint8_t* accept, float* pos_new_kf, double* info_new, int device) {
    if (n_kf < 0 || n_mp < 0 || n_pose < 0) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n_kf && (!kf_kp || !matches_idx_mp || !Tcw_new || !K || !accept || !pos_new_kf || !info_new)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (n_mp && (!mp_main_measure || !mp_main_pose || !mp_main_octave || !mp_normal || !mp_min_dist || !mp_max_dist || !Tcw_table))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int i = 0; i < n_kf; i++)
        if (matches_idx_mp[i] >= n_mp) return fail(SE2GPU_ERR_INVALID, "matches_idx_mp[%d] = %d is not a map point", i, matches_idx_mp[i]);
    if (!indices_ok(mp_main_pose, n_mp, n_pose)) return fail(SE2GPU_ERR_INVALID, "main keyframe index out of range");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n_kf == 0) return SE2GPU_OK;
    const size_t m = n_mp ? n_mp : 1;
    const float zero16[16] = {0};
    const se2gpu_keypoint* dk = st.upload(kf_kp, n_kf);
    const int* dmi = st.upload(matches_idx_mp, n_kf);
    const float* dTn = st.upload(Tcw_new, 16);
    const float* dmm = n_mp ? st.upload(mp_main_measure, 2 * m) : st.upload(zero16, 2);
    const int* dmp = n_mp ? st.upload(mp_main_pose, m) : st.scratch<int>(1);
    const int* dmo = n_mp ? st.upload(mp_main_octave, m) : st.scratch<int>(1);
    const float* dnv = n_mp ? st.upload(mp_normal, 3 * m) : st.upload(zero16, 3);
    const float* dmin = n_mp ? st.upload(mp_min_dist, m) : st.upload(zero16, 1);
    const float* dmax = n_mp ? st.upload(mp_max_dist, m) : st.upload(zero16, 1);
    const float* dtab = n_pose ? st.upload(Tcw_table, 16 * (size_t)n_pose) : st.upload(zero16, 16);
    const float* dK = st.upload(K, 9);
    uint8_t* dacc = st.output(accept, n_kf);
    float* dpos = st.inout(pos_new_kf, 3 * (size_t)n_kf);
    double* dinfo = st.inout(info_new, 9 * (size_t)n_kf);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_projection_observations_device(dk, n_kf, nullptr, dmi, dTn, dmm, dmp, dmo, dnv, dmin, dmax, dtab, dK,
                                                           lower_depth, upper_depth, fx, dacc, dpos, dinfo, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_debug_svd4(int n, const float* A, float* w, float* vt, int device) {
    if (n < 0 || (n && (!A || !w || !vt))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n == 0) return SE2GPU_OK;
    const float* dA = st.upload(A, 16 * (size_t)n);
    float* dw = st.output(w, 4 * (size_t)n);
    float* dv = st.output(vt, 16 * (size_t)n);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_debug_svd4, blocks(n), kBlock, 0, (cudaStream_t)0, n, dA, dw, dv);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

// ------------------------------------------------------------------------------------------ map-point updates
int se2gpu_mp_add_observations(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* upd_ptr, const int* upd_pos,
                               const se2gpu_mp_params* params, uint8_t* abandoned, int device) {
    return mp_updates_host(true, kf, mp, upd_ptr, upd_pos, params, abandoned, device);
}

int se2gpu_mp_erase_observations(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* upd_ptr, const int* upd_pos,
                                 const se2gpu_mp_params* params, uint8_t* abandoned, int device) {
    return mp_updates_host(false, kf, mp, upd_ptr, upd_pos, params, abandoned, device);
}

int se2gpu_mp_add_observations_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* d_upd_ptr,
                                      const int* d_upd_pos, const se2gpu_mp_params* params, uint8_t* d_abandoned, int* d_status,
                                      void* stream) {
    return mp_updates_device(true, kf, mp, d_upd_ptr, d_upd_pos, params, d_abandoned, d_status, stream);
}

int se2gpu_mp_erase_observations_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* d_upd_ptr,
                                        const int* d_upd_pos, const se2gpu_mp_params* params, uint8_t* d_abandoned,
                                        int* d_status, void* stream) {
    return mp_updates_device(false, kf, mp, d_upd_ptr, d_upd_pos, params, d_abandoned, d_status, stream);
}

int se2gpu_mp_update_measure_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, int n, const int* d_points,
                                    int* d_status, void* stream) {
    if (!mp_tables_set(kf, mp, false) || n < 0 || !d_status || (n && !d_points)) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    cudaStream_t s = (cudaStream_t)stream;
    SE2_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int), s));
    SE2_LAUNCH(k_mp_check, blocks(std::max(n, 1)), kBlock, 0, s, *kf, *mp, nullptr, nullptr, 0, n, d_points, d_status);
    if (n) SE2_LAUNCH(k_mp_update_measure, (n + kMpWarps - 1) / kMpWarps, kMpWarps * 32, 0, s, *kf, *mp, n, d_points, d_status);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_mp_update_measure(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, int n, const int* points, int device) {
    if (!mp_tables_set(kf, mp, false) || n < 0 || (n && !points)) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    const int M = mp->n_mp;
    if (mp->obs_ptr[0] != 0) return fail(SE2GPU_ERR_INVALID, "obs_ptr[0] must be 0");
    for (int i = 0; i < n; ++i)
        if (points[i] < 0 || points[i] >= M || !mp_point_ok(*kf, *mp, nullptr, nullptr, 0, points[i]))
            return fail(SE2GPU_ERR_INVALID, "points[%d]: index out of range", i);
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n == 0) return SE2GPU_OK;
    const size_t K = kf->n_kf, S = kf->n_slots, nobs = mp->obs_ptr[M];
    auto up = [&](auto* p, size_t c) { using T = std::remove_cv_t<std::remove_pointer_t<decltype(p)>>; return c ? st.upload(p, c) : st.scratch<T>(1); };
    se2gpu_mp_keyframes dk{kf->n_kf, up(kf->kf_id, K), up(kf->kf_null, K), up(kf->Tcw, 16 * K), up(kf->kp_base, K), kf->n_slots,
                           nullptr, nullptr, S ? st.inout(kf->view_mp, 3 * S) : st.scratch<float>(1), nullptr};
    se2gpu_mp_points dm{};
    dm.n_mp = M;
    dm.pos = st.upload(mp->pos, 3 * (size_t)M);
    dm.obs_ptr = up(mp->obs_ptr, (size_t)M + 1);
    dm.obs_kf = up(mp->obs_kf, nobs);
    dm.obs_idx = up(mp->obs_idx, nobs);
    const int* d_points = up(points, n);
    int* d_status = st.scratch<int>(1);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_mp_update_measure_device(&dk, &dm, n, d_points, d_status, nullptr); if (rc) return rc; }
    return st.finish();
}
