// CPU oracle (TEST INFRASTRUCTURE ONLY) of the host part of Track::mTrack (reference src/Track.cpp:162-188, :346-376):
// updateFramePose with the preSE2 pre-integration, and needNewKF, in the reference's types - Se2 in float with glibc's
// cosf / sinf (std::cos / std::sin on float), cv::Mat 4x4 float products through OpenCV's small-matrix gemm (float sums
// left to right, then (float)(t * alpha + 0)), cv::norm of a float 3x1 as a double sum of squares, and the Eigen double
// algebra of the pre-integration with Eigen's unrolled coefficient sums x0 + (x1 + x2) for 3x3 products.
#include <cmath>
#include <cstring>

#define TR_EXPORT extern "C" __attribute__((visibility("default")))

namespace {

struct Se2 {
    float x = 0, y = 0, theta = 0;
    Se2() = default;
    Se2(float x_, float y_, float th) : x(x_), y(y_), theta((float)norm_angle(th)) {}
    static double norm_angle(double t) {
        if (t >= -M_PI && t < M_PI) return t;
        double m = std::floor(t / (2 * M_PI));
        t = t - m * 2 * M_PI;
        if (t >= M_PI) t -= 2 * M_PI;
        if (t < -M_PI) t += 2 * M_PI;
        return t;
    }
    Se2 operator-(const Se2& that) const {
        float dx = x - that.x, dy = y - that.y;
        float dth = (float)norm_angle(theta - that.theta);
        float c = std::cos(that.theta), s = std::sin(that.theta);
        return Se2(c * dx + s * dy, -s * dx + c * dy, dth);
    }
    void toCvSE3(float* M) const {
        float c = std::cos(theta), s = std::sin(theta);
        float v[16] = {c, -s, 0, x, s, c, 0, y, 0, 0, 1, 0, 0, 0, 0, 1};
        std::memcpy(M, v, sizeof v);
    }
};

void matmul4(const float* A, const float* B, float* D) {
    float out[16];
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) {
            float t = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c] + A[r * 4 + 3] * B[3 * 4 + c];
            out[r * 4 + c] = (float)((double)t * 1.0 + 0.0);
        }
    std::memcpy(D, out, sizeof out);
}

void cam(const float* cTb, const float* bTc, const Se2& d, float* T) {
    float M[16], tmp[16];
    d.toCvSE3(M);
    matmul4(cTb, M, tmp);
    matmul4(tmp, bTc, T);
}

struct M3 {   // Eigen::Matrix3d, column-major
    double v[9] = {0};
    double& operator()(int r, int c) { return v[r + 3 * c]; }
    double operator()(int r, int c) const { return v[r + 3 * c]; }
    static M3 eye() { M3 m; m(0, 0) = m(1, 1) = m(2, 2) = 1; return m; }
    M3 t() const { M3 m; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) m(r, c) = (*this)(c, r); return m; }
    M3 operator*(const M3& o) const {
        M3 m;
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) m(r, c) = (*this)(r, 0) * o(0, c) + ((*this)(r, 1) * o(1, c) + (*this)(r, 2) * o(2, c));
        return m;
    }
    M3 operator+(const M3& o) const { M3 m; for (int k = 0; k < 9; k++) m.v[k] = v[k] + o.v[k]; return m; }
};

}  // namespace

// updateFramePose: Tcr [16]; meas [3] / cov [9] (column-major) updated in place
TR_EXPORT void track_oracle_pose(const float* cTb, const float* bTc, const float* odo_noise, const float* odom, const float* kf_odom,
                                 const float* last_odom, float* Tcr, double* meas, double* cov) {
    const Se2 fr(odom[0], odom[1], odom[2]), kf(kf_odom[0], kf_odom[1], kf_odom[2]), last(last_odom[0], last_odom[1], last_odom[2]);
    const Se2 dOdo = kf - fr;
    cam(cTb, bTc, dOdo, Tcr);
    const Se2 odok = fr - last;
    const double ox = odok.x, oy = odok.y;
    const double ca = std::cos(meas[2]), sa = std::sin(meas[2]);
    const double P00 = ca, P01 = -sa, P10 = sa, P11 = ca;
    meas[0] += P00 * ox + P01 * oy;
    meas[1] += P10 * ox + P11 * oy;
    meas[2] += odok.theta;
    M3 Ak = M3::eye(), Bk = M3::eye(), Sv = M3::eye(), Sk;
    Ak(0, 2) = P00 * -oy + P01 * ox;
    Ak(1, 2) = P10 * -oy + P11 * ox;
    Bk(0, 0) = P00; Bk(0, 1) = P01; Bk(1, 0) = P10; Bk(1, 1) = P11;
    for (int k = 0; k < 3; k++) Sv(k, k) = odo_noise[k] * odo_noise[k];
    std::memcpy(Sk.v, cov, sizeof Sk.v);
    const M3 out = (Ak * Sk) * Ak.t() + (Bk * Sv) * Bk.t();
    std::memcpy(cov, out.v, sizeof out.v);
}

// needNewKF: returns bNeedNewKF after acceptNewKF, *abort = setAbortBA was called
TR_EXPORT int track_oracle_decide(const float* cTb, const float* bTc, float upper_depth, int max_ftr, int min_frames, int max_frames,
                                  int dframes, int n_tracked_old, int n_old_kp, int n_good_prl, int n_matched, const float* odom,
                                  const float* kf_odom, int accept, int* abort) {
    bool c0 = dframes > min_frames;
    bool c1 = (float)n_tracked_old <= (float)n_old_kp * 0.5f;
    bool c2 = n_good_prl > 40;
    bool c3 = dframes > max_frames;
    bool c4 = n_matched < 0.1f * max_ftr || n_matched < 20;
    bool need = c0 && ((c1 && c2) || c3 || c4);
    const Se2 fr(odom[0], odom[1], odom[2]), kf(kf_odom[0], kf_odom[1], kf_odom[2]);
    Se2 d = fr - kf;
    bool c5 = std::fabs(d.theta) >= 0.0349f;
    float cTc[16];
    cam(cTb, bTc, Se2(d.x, d.y, d.theta), cTc);
    double s = 0;
    for (int r = 0; r < 3; r++) s += (double)cTc[r * 4 + 3] * cTc[r * 4 + 3];
    bool c6 = std::sqrt(s) >= (0.0523f * upper_depth * 0.1f);
    bool by_odo = c5 || c6;
    need = need && by_odo;
    *abort = 0;
    if (accept) return need;
    if (c0 && (c4 || c3) && by_odo) *abort = 1;
    return 0;
}

// the pieces the numpy restatement cannot call: glibc's float cos / sin
TR_EXPORT float track_oracle_cosf(float x) { return std::cos(x); }
TR_EXPORT float track_oracle_sinf(float x) { return std::sin(x); }
