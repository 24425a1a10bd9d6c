// The reference's Se2 odometry arithmetic on the host, shared by the tracker (track.cu) and the localization handle
// (loc.cu): normalize_angle, Se2::operator-, Se2::toCvSE3 and the cv::Mat 4x4 float products, with glibc's cosf / sinf so
// the poses are the reference's bit for bit.
#pragma once

#include <cmath>
#include <cstring>

namespace se2gpu {

struct Se2 { float x, y, theta; };

// normalize_angle (reference include/se2lam/Config.h), in double
inline double normalize_angle(double theta) {
    if (theta >= -M_PI && theta < M_PI) return theta;
    const double multiplier = std::floor(theta / (2 * M_PI));
    theta = theta - multiplier * 2 * M_PI;
    if (theta >= M_PI) theta -= 2 * M_PI;
    if (theta < -M_PI) theta += 2 * M_PI;
    return theta;
}

inline Se2 se2(float x, float y, float theta) { return {x, y, (float)normalize_angle(theta)}; }

// Se2::operator- (src/Config.cpp:215-223): that.inv() + *this
inline Se2 se2_minus(const Se2& a, const Se2& that) {
    const float dx = a.x - that.x, dy = a.y - that.y;
    const float dth = (float)normalize_angle(a.theta - that.theta);
    const float c = cosf(that.theta), s = sinf(that.theta);
    return se2(c * dx + s * dy, -s * dx + c * dy, dth);
}

// Se2::toCvSE3
inline void se2_mat(const Se2& a, float* T) {
    const float c = cosf(a.theta), s = sinf(a.theta);
    const float v[16] = {c, -s, 0, a.x, s, c, 0, a.y, 0, 0, 1, 0, 0, 0, 0, 1};
    std::memcpy(T, v, sizeof v);
}

// cv::Mat * cv::Mat on 4x4 float: OpenCV's small-matrix gemm, float sums left to right, then (float)(t*1 + 0)
inline void gemm4(const float* A, const float* B, float* D) {
    float R[16];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            float t = A[4 * i] * B[j];
            for (int k = 1; k < 4; k++) t = t + A[4 * i + k] * B[4 * k + j];
            R[4 * i + j] = (float)((double)t * 1.0 + 0.0);
        }
    std::memcpy(D, R, sizeof R);
}

// Config::cTb * dOdo.toCvSE3() * Config::bTc
inline void cam_motion(const float* cTb, const float* bTc, const Se2& d, float* T) {
    float M[16];
    se2_mat(d, M);
    gemm4(cTb, M, T);
    gemm4(T, bTc, T);
}

}  // namespace se2gpu
