// Outlier-rejection oracle (TEST INFRASTRUCTURE ONLY): a restatement of the reference's Track::removeOutliers
// (src/Track.cpp:308-344) and of the path cv::findFundamentalMat(pt1, pt2, mask) takes in OpenCV 4.13 with its defaults
// (FM_RANSAC, 3 px, confidence 0.99, 1000 iterations), written from OpenCV's published algorithm:
//   n < 7        no estimate, the mask is never created
//   n == 7       the 7-point kernel alone, mask all ones
//   8 <= n < 15  the LMedS registrator (FM_RANSAC falls back to LMedS below 15 points)
//   n >= 15      the RANSAC registrator
// The RNG, getSubset, haveCollinearPoints, the epipolar error, findInliers, the acceptance rule and RANSACUpdateNumIters
// (glibc log / pow) follow OpenCV operation by operation. The 7-point kernel's null space (Gaussian elimination with
// partial pivoting) and cubic roots (bisection over the doubles) are this project's own: OpenCV's SVD and trigonometric
// cubic are not restated bit for bit (DESIGN.md section 8). Built with -ffp-contract=off: nothing is fused.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

namespace {

constexpr int kModelPoints = 7;

// cv::RNG: multiply-with-carry, state seeded with (uint64)-1
struct Rng {
    uint64_t s = ~0ull;
    unsigned next() { s = (uint64_t)(unsigned)s * 4164903690u + (unsigned)(s >> 32); return (unsigned)s; }
    int uniform(int a, int b) { return a == b ? a : (int)(next() % (unsigned)(b - a) + a); }
};

// haveCollinearPoints(m, count): the last point against every pair of earlier ones
bool collinear(const float* p, const int* idx, int count) {
    const int i = count - 1;
    for (int j = 0; j < i; j++) {
        double dx1 = p[2 * idx[j]] - p[2 * idx[i]];
        double dy1 = p[2 * idx[j] + 1] - p[2 * idx[i] + 1];
        for (int k = 0; k < j; k++) {
            double dx2 = p[2 * idx[k]] - p[2 * idx[i]];
            double dy2 = p[2 * idx[k] + 1] - p[2 * idx[i] + 1];
            if (std::fabs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (std::fabs(dx1) + std::fabs(dy1) + std::fabs(dx2) + std::fabs(dy2)))
                return true;
        }
    }
    return false;
}

// RANSACPointSetRegistrator::getSubset with checkPartialSubsets = false
bool get_subset(const float* p1, const float* p2, int count, Rng& rng, int max_attempts, int* idx) {
    for (int it = 0; it < max_attempts; it++) {
        for (int i = 0; i < kModelPoints; i++) {
            int v = rng.uniform(0, count);
            for (;;) {
                bool dup = false;
                for (int k = 0; k < i; k++) dup = dup || idx[k] == v;
                if (!dup) break;
                v = rng.uniform(0, count);
            }
            idx[i] = v;
        }
        if (!collinear(p1, idx, kModelPoints) && !collinear(p2, idx, kModelPoints)) return true;
    }
    return false;
}

// p(x) = ((x + a1) x + a2) x + a3
inline double cubic_at(const double* a, double x) { return ((x + a[1]) * x + a[2]) * x + a[3]; }

inline int64_t ord(double x) { int64_t u; std::memcpy(&u, &x, 8); return u >= 0 ? u : INT64_MIN - u; }
inline double unord(int64_t o) { const int64_t u = o >= 0 ? o : INT64_MIN - o; double x; std::memcpy(&x, &u, 8); return x; }

// the root of the monic cubic in [lo, hi] by bisection over the ordered doubles: at most 64 halvings, ending on the
// endpoint with the smaller |p|
double bisect(const double* a, double lo, double hi) {
    const bool neg_lo = cubic_at(a, lo) < 0;
    int64_t l = ord(lo), h = ord(hi);
    while ((uint64_t)h - (uint64_t)l > 1) {
        const int64_t m = (int64_t)((uint64_t)l + ((uint64_t)h - (uint64_t)l) / 2);
        const double x = unord(m), v = cubic_at(a, x);
        if (v == 0) return x;
        if ((v < 0) == neg_lo) l = m; else h = m;
    }
    const double xl = unord(l), xh = unord(h);
    return std::fabs(cubic_at(a, xl)) <= std::fabs(cubic_at(a, xh)) ? xl : xh;
}

// real roots of c0 x^3 + c1 x^2 + c2 x + c3: cv::solveCubic's case split and discriminant, roots by bisection
int solve_cubic(const double* c, double* r) {
    double a0 = c[0], a1 = c[1], a2 = c[2], a3 = c[3];
    if (a0 == 0) {
        if (a1 == 0) {
            if (a2 == 0) return 0;
            r[0] = -a3 / a2;
            return 1;
        }
        double d = a2 * a2 - 4 * a1 * a3;
        if (!(d >= 0)) return 0;
        d = std::sqrt(d);
        const double q1 = (-a2 + d) * 0.5, q2 = (a2 + d) * -0.5;
        if (std::fabs(q1) > std::fabs(q2)) { r[0] = q1 / a1; r[1] = a3 / q1; }
        else { r[0] = q2 / a1; r[1] = a3 / q2; }
        return d > 0 ? 2 : 1;
    }
    a0 = 1. / a0;
    a1 *= a0; a2 *= a0; a3 *= a0;
    const double m[4] = {1., a1, a2, a3};
    const double d = (a1 * a1 * (a2 * a2 - 4 * a1 * a3) + 2 * a2 * (9 * a1 * a3 - 2 * a2 * a2) - 27 * a3 * a3) * (1. / 108);
    double B = std::fabs(a1);
    if (B < std::fabs(a2)) B = std::fabs(a2);
    if (B < std::fabs(a3)) B = std::fabs(a3);
    B = B + 1;
    if (B > DBL_MAX) B = DBL_MAX;
    if (d > 0) {
        const double Q = (a1 * a1 - 3 * a2) * (1. / 9), sq = std::sqrt(Q), c0 = a1 * (-1. / 3);
        const double cl = c0 - sq, ch = c0 + sq;
        r[0] = bisect(m, -B, cl);
        r[1] = bisect(m, cl, ch);
        r[2] = bisect(m, ch, B);
        return 3;
    }
    r[0] = bisect(m, -B, B);
    return 1;
}

// FMEstimatorCallback::runKernel for 7 points: up to 3 row-major F, returns their number
int run7point(const float* p1, const float* p2, const int* idx, double* fm) {
    double m1cx = 0, m1cy = 0, m2cx = 0, m2cy = 0;
    for (int i = 0; i < 7; i++) {
        m1cx += (double)p1[2 * idx[i]]; m1cy += (double)p1[2 * idx[i] + 1];
        m2cx += (double)p2[2 * idx[i]]; m2cy += (double)p2[2 * idx[i] + 1];
    }
    const double t = 1. / 7;
    m1cx *= t; m1cy *= t; m2cx *= t; m2cy *= t;
    double scale1 = 0, scale2 = 0;
    for (int i = 0; i < 7; i++) {
        const double ax = p1[2 * idx[i]] - m1cx, ay = p1[2 * idx[i] + 1] - m1cy;
        const double bx = p2[2 * idx[i]] - m2cx, by = p2[2 * idx[i] + 1] - m2cy;
        scale1 += std::sqrt(ax * ax + ay * ay);
        scale2 += std::sqrt(bx * bx + by * by);
    }
    scale1 *= t; scale2 *= t;
    if (scale1 < FLT_EPSILON || scale2 < FLT_EPSILON) return 0;
    scale1 = std::sqrt(2.) / scale1;
    scale2 = std::sqrt(2.) / scale2;

    double a[7 * 9];
    for (int i = 0; i < 7; i++) {
        const double x0 = (p1[2 * idx[i]] - m1cx) * scale1, y0 = (p1[2 * idx[i] + 1] - m1cy) * scale1;
        const double x1 = (p2[2 * idx[i]] - m2cx) * scale2, y1 = (p2[2 * idx[i] + 1] - m2cy) * scale2;
        double* row = a + 9 * i;
        row[0] = x1 * x0; row[1] = x1 * y0; row[2] = x1;
        row[3] = y1 * x0; row[4] = y1 * y0; row[5] = y1;
        row[6] = x0; row[7] = y0; row[8] = 1;
    }
    // null space of A: forward elimination with partial pivoting, then back substitution for the two free columns
    for (int r = 0; r < 7; r++) {
        double pivot = a[9 * r + r];
        int prow = r;
        for (int k = r + 1; k < 7; k++)
            if (std::fabs(pivot) < std::fabs(a[9 * k + r])) { pivot = a[9 * k + r]; prow = k; }
        if (std::fabs(pivot) < DBL_EPSILON) return 0;
        for (int c = r; c < 9; c++) { const double s = a[9 * prow + c]; a[9 * prow + c] = a[9 * r + c]; a[9 * r + c] = s; }
        for (int j = r + 1; j < 7; j++) {
            const double fac = a[9 * j + r] / pivot;
            for (int c = r; c < 9; c++) a[9 * j + c] -= fac * a[9 * r + c];
        }
    }
    double f1[9], f2[9];
    f1[7] = 0; f1[8] = 1; f2[7] = 1; f2[8] = 0;
    for (int i = 6; i >= 0; i--) {
        double acc1 = 0, acc2 = 0;
        for (int j = i + 1; j < 9; j++) { acc1 -= a[9 * i + j] * f1[j]; acc2 -= a[9 * i + j] * f2[j]; }
        f1[i] = acc1 / a[9 * i + i];
        f2[i] = acc2 / a[9 * i + i];
    }
    // det(lambda f1 + (1 - lambda) f2) = 0: run7Point's cubic
    for (int i = 0; i < 9; i++) f1[i] -= f2[i];
    double t0 = f2[4] * f2[8] - f2[5] * f2[7];
    double t1 = f2[3] * f2[8] - f2[5] * f2[6];
    double t2 = f2[3] * f2[7] - f2[4] * f2[6];
    double c[4], roots[3];
    c[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
    c[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 -
           f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) +
           f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
           f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) +
           f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) -
           f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) +
           f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
    t0 = f1[4] * f1[8] - f1[5] * f1[7];
    t1 = f1[3] * f1[8] - f1[5] * f1[6];
    t2 = f1[3] * f1[7] - f1[4] * f1[6];
    c[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 -
           f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) +
           f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
           f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) +
           f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) -
           f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) +
           f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
    c[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
    const int n = solve_cubic(c, roots);

    const double T1[9] = {scale1, 0, -scale1 * m1cx, 0, scale1, -scale1 * m1cy, 0, 0, 1};
    const double T2[9] = {scale2, 0, -scale2 * m2cx, 0, scale2, -scale2 * m2cy, 0, 0, 1};
    for (int k = 0; k < n; k++) {
        double* F = fm + 9 * k;
        double lambda = roots[k], mu = 1.;
        const double s = f1[8] * roots[k] + f2[8];
        double g[9];
        if (std::fabs(s) > DBL_EPSILON) { mu = 1. / s; lambda *= mu; g[8] = 1.; }
        else g[8] = 0.;
        for (int i = 0; i < 8; i++) g[i] = f1[i] * lambda + f2[i] * mu;
        // F = T2^T g T1, each entry a left-to-right sum of three products
        double h[9];
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                double acc = 0;
                for (int q = 0; q < 3; q++) acc += T2[3 * q + i] * g[3 * q + j];
                h[3 * i + j] = acc;
            }
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                double acc = 0;
                for (int q = 0; q < 3; q++) acc += h[3 * i + q] * T1[3 * q + j];
                F[3 * i + j] = acc;
            }
        if (std::fabs(F[8]) > FLT_EPSILON) {
            const double inv = 1. / F[8];
            for (int i = 0; i < 9; i++) F[i] *= inv;
        }
    }
    return n;
}

// FMEstimatorCallback::computeError: the larger squared distance to the two epipolar lines, rounded to float
float epi_error(const double* F, const float* p1, const float* p2, int i) {
    const double x1 = p1[2 * i], y1 = p1[2 * i + 1], x2 = p2[2 * i], y2 = p2[2 * i + 1];
    double a = F[0] * x1 + F[1] * y1 + F[2];
    double b = F[3] * x1 + F[4] * y1 + F[5];
    double c = F[6] * x1 + F[7] * y1 + F[8];
    const double s2 = 1. / (a * a + b * b);
    const double d2 = x2 * a + y2 * b + c;
    a = F[0] * x2 + F[3] * y2 + F[6];
    b = F[1] * x2 + F[4] * y2 + F[7];
    c = F[2] * x2 + F[5] * y2 + F[8];
    const double s1 = 1. / (a * a + b * b);
    const double d1 = x1 * a + y1 * b + c;
    const double e1 = d1 * d1 * s1, e2 = d2 * d2 * s2;
    return (float)(e1 < e2 ? e2 : e1);   // std::max
}

int find_inliers(const double* F, const float* p1, const float* p2, int n, double thresh, uint8_t* mask) {
    const float t = (float)(thresh * thresh);
    int nz = 0;
    for (int i = 0; i < n; i++) {
        const int f = epi_error(F, p1, p2, i) <= t;
        if (mask) mask[i] = (uint8_t)f;
        nz += f;
    }
    return nz;
}

// cv::RANSACUpdateNumIters
int update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = p < 0. ? 0. : p; p = 1. < p ? 1. : p;
    ep = ep < 0. ? 0. : ep; ep = 1. < ep ? 1. : ep;
    double num = 1. - p < DBL_MIN ? DBL_MIN : 1. - p;
    double denom = 1. - std::pow(1. - ep, model_points);
    if (denom < DBL_MIN) return 0;
    num = std::log(num);
    denom = std::log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)std::lrint(num / denom);
}

// the k-th smallest error in the order of its bits (std::nth_element over errf.ptr<int>())
float kth_by_bits(const float* e, int n, int k) {
    for (int i = 0; i < n; i++) {
        int32_t bi; std::memcpy(&bi, &e[i], 4);
        int less = 0, eq = 0;
        for (int j = 0; j < n; j++) {
            int32_t bj; std::memcpy(&bj, &e[j], 4);
            less += bj < bi; eq += bj == bi;
        }
        if (less <= k && k < less + eq) return e[i];
    }
    return e[k];
}

// RANSACPointSetRegistrator::run for n >= 15: returns whether a model was accepted
bool ransac(const float* p1, const float* p2, int n, uint8_t* mask, double* best, int* iters) {
    Rng rng;
    int niters = 1000, max_good = 0, iter = 0, idx[7];
    double fm[27];
    for (; iter < niters; iter++) {
        if (!get_subset(p1, p2, n, rng, 10000, idx)) {
            if (iter == 0) { *iters = 0; return false; }
            break;
        }
        const int nm = run7point(p1, p2, idx, fm);
        for (int i = 0; i < nm; i++) {
            const int good = find_inliers(fm + 9 * i, p1, p2, n, 3., nullptr);
            if (good > (max_good > kModelPoints - 1 ? max_good : kModelPoints - 1)) {
                std::memcpy(best, fm + 9 * i, sizeof(double) * 9);
                max_good = good;
                niters = update_num_iters(0.99, (double)(n - good) / n, kModelPoints, niters);
            }
        }
    }
    *iters = iter;
    if (max_good > 0) find_inliers(best, p1, p2, n, 3., mask);
    return max_good > 0;
}

// LMeDSPointSetRegistrator::run for 7 < n: returns the registrator's result; *have_model when the mask was written
bool lmeds(const float* p1, const float* p2, int n, uint8_t* mask, double* best, int* iters, bool* have_model) {
    Rng rng;
    double min_median = DBL_MAX, fm[27];
    float err[16];
    int idx[7], iter = 0;
    int niters = update_num_iters(0.99, 0.45, kModelPoints, 1000);
    niters = niters < 3 ? 3 : niters;
    *have_model = false;
    for (; iter < niters; iter++) {
        if (!get_subset(p1, p2, n, rng, 1000, idx)) {
            if (iter == 0) { *iters = 0; return false; }
            break;
        }
        const int nm = run7point(p1, p2, idx, fm);
        for (int i = 0; i < nm; i++) {
            for (int k = 0; k < n; k++) err[k] = epi_error(fm + 9 * i, p1, p2, k);
            const double median = kth_by_bits(err, n, n / 2);
            if (median < min_median) { min_median = median; std::memcpy(best, fm + 9 * i, sizeof(double) * 9); }
        }
    }
    *iters = iter;
    if (!(min_median < DBL_MAX)) return false;
    double sigma = 2.5 * 1.4826 * (1 + 5. / (n - kModelPoints)) * std::sqrt(min_median);
    sigma = sigma < 0.001 ? 0.001 : sigma;
    *have_model = true;
    return find_inliers(best, p1, p2, n, sigma, mask) >= kModelPoints;
}

}  // namespace

extern "C" {

// cv::findFundamentalMat(p1, p2, mask) with the defaults on n float pairs (p1 / p2 [2n]).
// mask [n] is the mask as the caller's std::vector<uchar> holds it: zeros where OpenCV leaves it unwritten.
// F [27] receives the returned matrix (n == 7: one 3x3 per root), zeros past it. Returns the number of 3x3 blocks in the
// returned matrix (0 = empty Mat); *mask_created is 0 when the mask is never created (n < 7); *iters = hypotheses run.
__attribute__((visibility("default")))
int fundam_oracle_find(const float* p1, const float* p2, int n, uint8_t* mask, double* F, int* mask_created, int* iters) {
    std::memset(F, 0, sizeof(double) * 27);
    if (n > 0) std::memset(mask, 0, n);
    *iters = 0;
    *mask_created = n >= kModelPoints;
    if (n < kModelPoints) return 0;
    int idx[7] = {0, 1, 2, 3, 4, 5, 6};
    if (n == kModelPoints) {
        std::memset(mask, 1, n);
        *iters = 1;
        const int nm = run7point(p1, p2, idx, F);
        return nm > 0 ? nm : 0;
    }
    if (n >= 15) return ransac(p1, p2, n, mask, F, iters) ? 1 : 0;
    bool have = false;
    const bool ok = lmeds(p1, p2, n, mask, F, iters, &have);
    if (!ok) std::memset(F, 0, sizeof(double) * 9);
    return ok ? 1 : 0;
}

// Track::removeOutliers(kp1, kp2, matches) on keypoint records of `kp_stride` floats whose first two are pt.x, pt.y.
// matches [n1] is updated in place; returns nInlier. F [9] = the returned model's first 3x3 (zeros for an empty Mat),
// *iters = hypotheses run.
__attribute__((visibility("default")))
int fundam_oracle_remove_outliers(const float* kp1, int n1, const float* kp2, int kp_stride, int* matches, double* F, int* iters) {
    float* p1 = new float[2 * (size_t)(n1 > 0 ? n1 : 1)];
    float* p2 = new float[2 * (size_t)(n1 > 0 ? n1 : 1)];
    int* idx = new int[n1 > 0 ? n1 : 1];
    uint8_t* mask = new uint8_t[n1 > 0 ? n1 : 1];
    int n = 0;
    for (int i = 0; i < n1; i++) {
        if (matches[i] < 0) continue;
        idx[n] = i;
        p1[2 * n] = kp1[(size_t)kp_stride * i]; p1[2 * n + 1] = kp1[(size_t)kp_stride * i + 1];
        p2[2 * n] = kp2[(size_t)kp_stride * matches[i]]; p2[2 * n + 1] = kp2[(size_t)kp_stride * matches[i] + 1];
        n++;
    }
    double Fall[27];
    int created = 0, ninlier = 0;
    std::memset(Fall, 0, sizeof Fall);
    *iters = 0;
    if (n != 0) fundam_oracle_find(p1, p2, n, mask, Fall, &created, iters);
    std::memcpy(F, Fall, sizeof(double) * 9);
    for (int i = 0; created && i < n; i++) {
        if (!mask[i]) matches[idx[i]] = -1;
        else ninlier++;
    }
    if (ninlier < 10) {
        ninlier = 0;
        for (int i = 0; i < n1; i++) matches[i] = -1;
    }
    delete[] p1; delete[] p2; delete[] idx; delete[] mask;
    return ninlier;
}

// RANSACUpdateNumIters(0.99, (n - good) / n, 7, max_iters) for n in [n_lo, n_hi] and good in [0, n], row after row
__attribute__((visibility("default")))
void fundam_oracle_niters_range(int n_lo, int n_hi, int max_iters, int* out) {
    for (int n = n_lo; n <= n_hi; n++)
        for (int good = 0; good <= n; good++) *out++ = update_num_iters(0.99, (double)(n - good) / n, kModelPoints, max_iters);
}

__attribute__((visibility("default")))
int fundam_oracle_niters(double ep, int max_iters) { return update_num_iters(0.99, ep, kModelPoints, max_iters); }

}  // extern "C"
