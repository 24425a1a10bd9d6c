// Two-view geometry oracle (TEST INFRASTRUCTURE ONLY): a restatement of the reference's cvu::triangulate / inv / se3map /
// checkParallax, Config::acceptDepth, Track::doTriangulate, Track::calcSE3toXYZInfo, MapPoint::acceptNewObserve and the
// MatchByProjection branch of LocalMapper::findCorrespd, in the reference's float types, with every OpenCV primitive they
// reach restated operation by operation (oracle/pin_geom_against_cv2.py checks each one cv2 exposes, DESIGN.md section 8).
// Built with -ffp-contract=off: the only fused multiply-add is the explicit fmaf of the A rows.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

namespace {

struct P3 { float x, y, z; };

inline P3 sub(P3 a, P3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline float dot(P3 a, P3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }          // Point3_::dot (float)
inline P3 cross(P3 a, P3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline double norm3(P3 p) { return std::sqrt((double)p.x * p.x + (double)p.y * p.y + (double)p.z * p.z); }  // cv::norm(Point3_)

// cv::gemm(A[3x3], B[3xncols], alpha) with flags 0: OpenCV's small-matrix path (float sums, left to right, not fused;
// the result is (float)(t*alpha + 0*beta)).
void gemm3_fast(const float* A, int lda, const float* B, int ldb, int ncols, double alpha, float* D, int ldd) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < ncols; j++) {
            float t = A[i * lda] * B[j] + A[i * lda + 1] * B[ldb + j] + A[i * lda + 2] * B[2 * ldb + j];
            D[i * ldd + j] = (float)(t * alpha + 0.0 * 0.0);
        }
}

// cv::gemm(A, B, 1, noArray(), 0, D, GEMM_1_T) on 3x3 float: the generic GEMMSingleMul<float, double> loop.
void gemm3_at_b(const float* A, const float* B, float* D) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += (double)A[k * 3 + i] * (double)B[k * 3 + j];
            D[i * 3 + j] = (float)(s * 1.0);
        }
}

// cvu::inv (cvutil.cpp:15-23): [R^T | -R^T t]
void inv4(const float* T, float* Ti) {
    float RT[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) RT[i * 3 + j] = T[j * 4 + i];
    float t[3] = {T[3], T[7], T[11]}, nt[3];
    gemm3_fast(RT, 3, t, 1, 1, -1.0, nt, 1);
    for (int i = 0; i < 16; i++) Ti[i] = (i % 5 == 0) ? 1.f : 0.f;
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) Ti[i * 4 + j] = RT[i * 3 + j];
        Ti[i * 4 + 3] = nt[i];
    }
}

// cvu::se3map (cvutil.cpp:131-136): Matx33f * Point3f (float sums from 0) + t
P3 se3map(const float* T, P3 p) {
    float r[3];
    for (int i = 0; i < 3; i++) {
        float s = 0;
        s += T[i * 4] * p.x; s += T[i * 4 + 1] * p.y; s += T[i * 4 + 2] * p.z;
        r[i] = s;
    }
    return {r[0] + T[3], r[1] + T[7], r[2] + T[11]};
}

// The double hypot of OpenCV's JacobiSVDImpl_ is lapack.cpp's own inline template, not libm's hypot (cv2 imports no
// double hypot): the larger magnitude times sqrt(1 + ratio^2).
double cv_hypot(double a, double b) {
    a = std::abs(a);
    b = std::abs(b);
    if (a > b) {
        b /= a;
        return a * std::sqrt(1 + b * b);
    }
    if (b > 0) {
        a /= b;
        return b * std::sqrt(1 + a * a);
    }
    return 0;
}

// Config::Kcam * Tcw.rowRange(0,3)
void projection(const float* K, const float* T, float* P) { gemm3_fast(K, 3, T, 4, 4, 1.0, P, 4); }

double libm_hypot(double a, double b) { return std::hypot(a, b); }

// cv::SVD::compute(A, w, u, vt, MODIFY_A | FULL_UV) on a 4x4 CV_32F: JacobiSVDImpl_<float> on A^T (FLT_EPSILON*2,
// at most max(4, 30) sweeps, double accumulators, lapack.cpp's hypot, descending sort). Only w and vt are produced (u needs
// OpenCV's RNG for zero singular values and the reference never reads it). `hyp` is cv_hypot except in the pin's check
// that its sample tells cv_hypot and libm's hypot apart.
void svd4_impl(const float* A, float* w_out, float* vt_out, double (*hyp)(double, double)) {
    float At[4][4], Vt[4][4];
    double W[4];
    const float eps = FLT_EPSILON * 2;
    for (int i = 0; i < 4; i++)
        for (int k = 0; k < 4; k++) At[i][k] = A[k * 4 + i];
    for (int i = 0; i < 4; i++) {
        double sd = 0;
        for (int k = 0; k < 4; k++) { float t = At[i][k]; sd += (double)t * t; }
        W[i] = sd;
        for (int k = 0; k < 4; k++) Vt[i][k] = 0;
        Vt[i][i] = 1;
    }
    for (int iter = 0; iter < 30; iter++) {
        bool changed = false;
        for (int i = 0; i < 3; i++)
            for (int j = i + 1; j < 4; j++) {
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < 4; k++) p += (double)At[i][k] * At[j][k];
                if (std::abs(p) <= eps * std::sqrt((double)a * b)) continue;
                p *= 2;
                double beta = a - b, gamma = hyp(p, beta);
                float c, s;
                if (beta < 0) {
                    double delta = (gamma - beta) * 0.5;
                    s = (float)std::sqrt(delta / gamma);
                    c = (float)(p / (gamma * s * 2));
                } else {
                    c = (float)std::sqrt((gamma + beta) / (gamma * 2));
                    s = (float)(p / (gamma * c * 2));
                }
                a = b = 0;
                for (int k = 0; k < 4; k++) {
                    float t0 = c * At[i][k] + s * At[j][k];
                    float t1 = -s * At[i][k] + c * At[j][k];
                    At[i][k] = t0; At[j][k] = t1;
                    a += (double)t0 * t0; b += (double)t1 * t1;
                }
                W[i] = a; W[j] = b;
                changed = true;
                for (int k = 0; k < 4; k++) {
                    float t0 = Vt[i][k] * c + Vt[j][k] * s;
                    float t1 = Vt[j][k] * c - Vt[i][k] * s;
                    Vt[i][k] = t0; Vt[j][k] = t1;
                }
            }
        if (!changed) break;
    }
    for (int i = 0; i < 4; i++) {
        double sd = 0;
        for (int k = 0; k < 4; k++) { float t = At[i][k]; sd += (double)t * t; }
        W[i] = std::sqrt(sd);
    }
    for (int i = 0; i < 3; i++) {
        int j = i;
        for (int k = i + 1; k < 4; k++)
            if (W[j] < W[k]) j = k;
        if (i != j) {
            std::swap(W[i], W[j]);
            for (int k = 0; k < 4; k++) std::swap(At[i][k], At[j][k]);
            for (int k = 0; k < 4; k++) std::swap(Vt[i][k], Vt[j][k]);
        }
    }
    for (int i = 0; i < 4; i++) w_out[i] = (float)W[i];
    if (vt_out) std::memcpy(vt_out, Vt, sizeof(Vt));
}

}  // namespace

extern "C" {

void geom_oracle_svd4(const float* A, float* w_out, float* vt_out) { svd4_impl(A, w_out, vt_out, cv_hypot); }
void geom_oracle_svd4_libm_hypot(const float* A, float* w_out, float* vt_out) { svd4_impl(A, w_out, vt_out, libm_hypot); }

// A of cvu::triangulate: A.row(r) = x * P.row(2) - P.row(0) is cv::addWeighted(P.row(2), x, P.row(0), -1, 0), whose
// dispatched SIMD kernel evaluates fma(x, P2k, -P0k) on an AVX2 host.
void geom_oracle_build_a(const float* pt1, const float* pt2, const float* P1, const float* P2, float* A) {
    for (int k = 0; k < 4; k++) {
        A[k] = std::fmaf(pt1[0], P1[8 + k], -P1[k]);
        A[4 + k] = std::fmaf(pt1[1], P1[8 + k], -P1[4 + k]);
        A[8 + k] = std::fmaf(pt2[0], P2[8 + k], -P2[k]);
        A[12 + k] = std::fmaf(pt2[1], P2[8 + k], -P2[4 + k]);
    }
}

// cvu::triangulate (cvutil.cpp:46-59). x3D.rowRange(0,3) / w is convertTo(scale = 1./w): x * (float)(1.0 / w) + 0.
void geom_oracle_triangulate1(const float* pt1, const float* pt2, const float* P1, const float* P2, float* xyz) {
    float A[16], w[4], vt[16];
    geom_oracle_build_a(pt1, pt2, P1, P2, A);
    geom_oracle_svd4(A, w, vt);
    double inv = 1. / (double)vt[15];
    if (std::fabs(inv) == 1.0) {
        for (int k = 0; k < 3; k++) xyz[k] = (float)((double)vt[12 + k] * inv) + 0.f;
    } else {
        float a = (float)inv;
        for (int k = 0; k < 3; k++) xyz[k] = vt[12 + k] * a + 0.f;
    }
}

void geom_oracle_triangulate(int n, const float* pt1, const float* pt2, const float* P, const int* idx1, const int* idx2,
                             float* xyz) {
    for (int i = 0; i < n; i++)
        geom_oracle_triangulate1(pt1 + 2 * i, pt2 + 2 * i, P + 12 * idx1[i], P + 12 * idx2[i], xyz + 3 * i);
}

void geom_oracle_inv(const float* T, float* Ti) { inv4(T, Ti); }
void geom_oracle_gemm3_fast(const float* A, const float* B, int ncols, double alpha, float* D) { gemm3_fast(A, 3, B, ncols, ncols, alpha, D, ncols); }
void geom_oracle_gemm3_at_b(const float* A, const float* B, float* D) { gemm3_at_b(A, B, D); }

// cvu::checkParallax (cvutil.cpp:121-128)
int geom_oracle_check_parallax(const float* o1, const float* o2, const float* pt3, int min_degree) {
    static const float minCos[4] = {0.9998f, 0.9994f, 0.9986f, 0.9976f};
    P3 p = {pt3[0], pt3[1], pt3[2]};
    P3 p1 = sub(p, {o1[0], o1[1], o1[2]}), p2 = sub(p, {o2[0], o2[1], o2[2]});
    float cosParallax = (float)(std::fabs((double)dot(p1, p2)) / (norm3(p1) * norm3(p2)));
    return cosParallax < minCos[min_degree - 1];
}

// cv::Rodrigues of a float rotation vector (double internally, rounded to float)
void geom_oracle_rodrigues(const float* rv, float* R) {
    double rx = rv[0], ry = rv[1], rz = rv[2];
    double theta = std::sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < DBL_EPSILON) {
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.f : 0.f;
        return;
    }
    double c = std::cos(theta), s = std::sin(theta), c1 = 1. - c;
    double itheta = theta ? 1. / theta : 0.;
    rx *= itheta; ry *= itheta; rz *= itheta;
    const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int i = 0; i < 9; i++) {
        double e = (i % 4 == 0) ? 1. : 0.;
        R[i] = (float)((c * e + c1 * rrt[i]) + s * r_x[i]);
    }
}

// Track::calcSE3toXYZInfo (Track.cpp:259-306); info1/info2 are the float results widened as toMatrix3d does
void geom_oracle_xyz_info1(const float* xyz1p, const float* Tcw1, const float* Tcw2, float fx, double* info1, double* info2) {
    float T1i[16], T2i[16];
    inv4(Tcw1, T1i);
    inv4(Tcw2, T2i);
    P3 xyz1 = {xyz1p[0], xyz1p[1], xyz1p[2]};
    P3 O1 = {T1i[3], T1i[7], T1i[11]}, O2 = {T2i[3], T2i[7], T2i[11]};
    P3 xyz = se3map(T1i, xyz1);
    P3 vO1 = sub(xyz, O1), vO2 = sub(xyz, O2);
    float sinParallax = (float)(norm3(cross(vO1, vO2)) / (norm3(vO1) * norm3(vO2)));
    P3 xyz2 = se3map(Tcw2, xyz);
    float length1 = (float)norm3(xyz1), length2 = (float)norm3(xyz2);
    float dxy1 = 2.f * length1 / fx, dxy2 = 2.f * length2 / fx;
    float dz1 = dxy2 / sinParallax, dz2 = dxy1 / sinParallax;
    float I1[9] = {1.f / (dxy1 * dxy1), 0, 0, 0, 1.f / (dxy1 * dxy1), 0, 0, 0, 1.f / (dz1 * dz1)};
    float I2[9] = {1.f / (dxy2 * dxy2), 0, 0, 0, 1.f / (dxy2 * dxy2), 0, 0, 0, 1.f / (dz2 * dz2)};
    const P3 z1 = {0, 0, length1}, z2 = {0, 0, length2};
    P3 k[2] = {cross(xyz1, z1), cross(xyz2, z2)};
    const P3 zz[2] = {z1, z2}, xx[2] = {xyz1, xyz2};
    const float* info_xyz[2] = {I1, I2};
    double* out[2] = {info1, info2};
    for (int v = 0; v < 2; v++) {
        float normk = (float)norm3(k[v]);
        float sinv = (float)(normk / (norm3(zz[v]) * norm3(xx[v])));
        float f = std::asin(sinv) / normk;
        float kv[3] = {k[v].x * f, k[v].y * f, k[v].z * f};
        float R[9], tmp[9], res[9];
        geom_oracle_rodrigues(kv, R);
        gemm3_at_b(R, info_xyz[v], tmp);            // R.t() * info_xyz
        gemm3_fast(tmp, 3, R, 3, 3, 1.0, res, 3);   // (...) * R
        for (int e = 0; e < 9; e++) out[v][e] = (double)res[e];
    }
}

void geom_oracle_xyz_info(int n, const float* xyz1, const int* pose1, const int* pose2, const float* Tcw, float fx,
                          double* info1, double* info2) {
    for (int i = 0; i < n; i++)
        geom_oracle_xyz_info1(xyz1 + 3 * i, Tcw + 16 * pose1[i], Tcw + 16 * pose2[i], fx, info1 + 9 * i, info2 + 9 * i);
}

// keypoint layout of cv::KeyPoint / se2gpu_keypoint (28 bytes: x, y, size, angle, response, octave, class_id)
struct KP { float x, y, size, angle, response; int octave, class_id; };

// Track::doTriangulate (Track.cpp:378-419) after the nMinFrames early return. Returns nTrackedOld; counts = {nTrackedOld, nGoodPrl}.
int geom_oracle_track_triangulate(const KP* kp_kf, int n_kf, const KP* kp_frame, int* matches12, const uint8_t* kf_observed,
                                  const float* kf_view_mp, const float* Tcr, const float* K, float lower, float upper,
                                  int min_prl_deg, float* local_mps, uint8_t* good_prl, int* counts) {
    float Ti[16], P_KF[12], P[12];
    inv4(Tcr, Ti);
    const float eye34[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    projection(K, eye34, P_KF);                       // Config::PrjMtrxEye = Kcam * eye(3,4)
    projection(K, Tcr, P);
    const float O0[3] = {0, 0, 0}, Ocam[3] = {Ti[3], Ti[7], Ti[11]};
    int nTrackedOld = 0, nGoodPrl = 0;
    for (int i = 0; i < n_kf; i++) {
        good_prl[i] = 0;
        if (matches12[i] < 0) continue;
        if (kf_observed[i]) {
            std::memcpy(local_mps + 3 * i, kf_view_mp + 3 * i, 12);
            nTrackedOld++;
            continue;
        }
        const float pk[2] = {kp_kf[i].x, kp_kf[i].y}, pf[2] = {kp_frame[matches12[i]].x, kp_frame[matches12[i]].y};
        float pos[3];
        geom_oracle_triangulate1(pk, pf, P_KF, P, pos);
        if (pos[2] >= lower && pos[2] <= upper) {     // Config::acceptDepth
            std::memcpy(local_mps + 3 * i, pos, 12);
            if (geom_oracle_check_parallax(O0, Ocam, pos, min_prl_deg)) {
                nGoodPrl++;
                good_prl[i] = 1;
            }
        } else {
            matches12[i] = -1;
        }
    }
    counts[0] = nTrackedOld;
    counts[1] = nGoodPrl;
    return nTrackedOld;
}

// MapPoint::acceptNewObserve (MapPoint.cpp:202-209)
int geom_oracle_accept_new_observe(const float* pos, const float* normal, int main_octave, int octave, float min_dist,
                                   float max_dist) {
    P3 p = {pos[0], pos[1], pos[2]}, nv = {normal[0], normal[1], normal[2]};
    float dist = (float)norm3(p);
    float cosAngle = (float)(std::fabs((double)dot(p, nv)) / (dist * norm3(nv)));
    bool c1 = std::abs(main_octave - octave) <= 2;
    bool c2 = cosAngle >= 0.866f;
    bool c3 = dist >= min_dist && dist <= max_dist;
    return c1 && c2 && c3;
}

// LocalMapper::findCorrespd, body of the MatchByProjection loop (LocalMapper.cpp:119-141) without the object-graph
// updates. Writes accept[i] for every i; pos_new_kf / info_new only where accept[i] == 1.
void geom_oracle_projection_observations(int n_kf, const KP* kf_kp, const int* matches_idx_mp, const float* Tcw_new,
                                         const float* mp_main_measure, const int* mp_main_pose, const int* mp_main_octave,
                                         const float* mp_normal, const float* mp_min_dist, const float* mp_max_dist,
                                         const float* Tcw_table, const float* K, float lower, float upper, float fx,
                                         uint8_t* accept, float* pos_new_kf, double* info_new) {
    float P2[12];
    projection(K, Tcw_new, P2);
    for (int i = 0; i < n_kf; i++) {
        accept[i] = 0;
        int m = matches_idx_mp[i];
        if (m < 0) continue;
        const float* Tmain = Tcw_table + 16 * mp_main_pose[m];
        float P1[12];
        projection(K, Tmain, P1);
        const float pt[2] = {kf_kp[i].x, kf_kp[i].y};
        float x3d[3];
        geom_oracle_triangulate1(mp_main_measure + 2 * m, pt, P1, P2, x3d);
        P3 pn = se3map(Tcw_new, {x3d[0], x3d[1], x3d[2]});
        const float pos[3] = {pn.x, pn.y, pn.z};
        if (!geom_oracle_accept_new_observe(pos, mp_normal + 3 * m, mp_main_octave[m], kf_kp[i].octave, mp_min_dist[m], mp_max_dist[m]))
            continue;
        if (pn.z > upper || pn.z < lower) continue;
        double info_old[9];
        geom_oracle_xyz_info1(pos, Tcw_new, Tmain, fx, info_new + 9 * i, info_old);
        std::memcpy(pos_new_kf + 3 * i, pos, 12);
        accept[i] = 1;
    }
}

}  // extern "C"
