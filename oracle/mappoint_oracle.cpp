// Map-point update oracle (TEST INFRASTRUCTURE ONLY): a restatement of the reference's MapPoint::addObservation (with
// updateMainKFandDescriptor and updateParallax), MapPoint::eraseObservation and MapPoint::updateMeasureInKFs in the
// reference's float types, over the flattened tables of include/se2gpu.h's se2gpu_mp_* entries (DESIGN.md section 13).
// Each point's list is held as the reference holds mObservations: a sequence that insertions and erasures change one
// entry at a time. The OpenCV pieces it adds to geom_oracle.cpp's (the chained float gemms of Rcw^T M Rcw and
// Rcw M Rcw^T, cv::norm(Point3f) and Point3f * double) are pinned by oracle/pin_mappoint_against_cv2.py.
#include "geom_oracle.cpp"

#include <algorithm>
#include <climits>
#include <vector>

#define MP_EXPORT extern "C" __attribute__((visibility("default")))

namespace {

// the layouts of se2gpu_mp_keyframes / se2gpu_mp_points / se2gpu_mp_params
struct MpKeyframes {
    int n_kf;
    const int* kf_id;
    const uint8_t* kf_null;
    const float* Tcw;
    const int* kp_base;
    int n_slots;
    const KP* kp;
    const uint8_t* desc;
    float* view_mp;
    double* view_info;
};
struct MpPoints {
    int n_mp;
    float* pos;
    uint8_t* good_prl;
    uint8_t* null;
    int* main_kf;
    uint8_t* main_desc;
    int* main_octave;
    float* main_measure;
    float* level_scale;
    float* normal;
    float* min_dist;
    float* max_dist;
    const int* obs_ptr;
    const int* obs_kf;
    const int* obs_idx;
};
struct MpParams {
    float K[9];
    float lower_depth, upper_depth, fx;
    int nlevels;
    float scale_factors[32];
};

// cv::gemm(A, B, 1, noArray(), 0, D, GEMM_2_T) on 3x3 float: the generic loop with double sums
void gemm3_a_bt(const float* A, const float* B, float* D) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += (double)A[i * 3 + k] * (double)B[j * 3 + k];
            D[i * 3 + j] = (float)(s * 1.0);
        }
}

// Point3f * double (OpenCV's operator*: each product in double, rounded once)
P3 mul_pd(P3 p, double s) { return {(float)(p.x * s), (float)(p.y * s), (float)(p.z * s)}; }

int hamming(const uint8_t* a, const uint8_t* b) {
    int d = 0;
    for (int k = 0; k < 32; k++) d += __builtin_popcount((unsigned)(a[k] ^ b[k]));
    return d;
}

// One map point with its list: `obs` holds list positions in mObservations' order
struct Point {
    const MpKeyframes& kf;
    const MpPoints& mp;
    const MpParams& prm;
    int m, p0;
    std::vector<int> obs;

    int kfo(int j) const { return mp.obs_kf[p0 + j]; }
    int slot(int j) const { return kf.kp_base[kfo(j)] + mp.obs_idx[p0 + j]; }
    int id(int j) const { return kf.kf_id[kfo(j)]; }
    const float* T(int j) const { return kf.Tcw + 16 * kfo(j); }
    P3 view(int j) const { const float* v = kf.view_mp + 3 * slot(j); return {v[0], v[1], v[2]}; }
    void set_view(int j, P3 p, const double* info) {
        float* v = kf.view_mp + 3 * slot(j);
        v[0] = p.x; v[1] = p.y; v[2] = p.z;
        std::memcpy(kf.view_info + 9 * slot(j), info, 9 * sizeof(double));
    }
    void set_null() { mp.null[m] = 1; mp.good_prl[m] = 0; obs.clear(); }

    // MapPoint.cpp:228-292
    void update_main() {
        if (mp.null[m] || obs.empty()) return;
        std::vector<int> vKF;
        for (int j : obs)
            if (!kf.kf_null[kfo(j)]) vKF.push_back(j);
        if (vKF.empty()) return;
        const int N = (int)vKF.size();
        std::vector<float> D((size_t)N * N);
        for (int i = 0; i < N; i++) {
            D[(size_t)i * N + i] = 0;
            for (int j = i + 1; j < N; j++) {
                const int d = hamming(kf.desc + 32 * (size_t)slot(vKF[i]), kf.desc + 32 * (size_t)slot(vKF[j]));
                D[(size_t)i * N + j] = (float)d;
                D[(size_t)j * N + i] = (float)d;
            }
        }
        int bestMedian = INT_MAX, bestIdx = 0;
        for (int i = 0; i < N; i++) {
            std::vector<int> v(D.begin() + (size_t)i * N, D.begin() + (size_t)(i + 1) * N);
            std::sort(v.begin(), v.end());
            const int median = v[(size_t)(0.5 * (N - 1))];
            if (median < bestMedian) { bestMedian = median; bestIdx = i; }
        }
        const int jb = vKF[bestIdx], s = slot(jb);
        std::memcpy(mp.main_desc + 32 * (size_t)m, kf.desc + 32 * (size_t)s, 32);
        mp.main_measure[2 * m] = kf.kp[s].x;
        mp.main_measure[2 * m + 1] = kf.kp[s].y;
        if (mp.main_kf[m] >= 0 && kf.kf_id[mp.main_kf[m]] == id(jb)) return;
        mp.main_kf[m] = kfo(jb);
        const int oct = kf.kp[s].octave;
        mp.main_octave[m] = oct;
        mp.level_scale[m] = prm.scale_factors[oct];
        const float dist = (float)norm3(view(jb));
        mp.max_dist[m] = dist * mp.level_scale[m];
        mp.min_dist[m] = mp.max_dist[m] / prm.scale_factors[prm.nlevels - 1];
    }

    // MapPoint.cpp:124-185 for the entry at list position q; returns true when it abandons the point
    bool update_parallax(int q) {
        if (mp.good_prl[m] || obs.size() <= 2) return false;
        int j0 = -1;
        for (int j : obs) {
            if (id(q) - id(j) > 6) continue;
            if (j0 < 0 || id(j) < id(j0)) j0 = j;
        }
        float P0[12], P1[12];
        projection(prm.K, T(j0), P0);
        projection(prm.K, T(q), P1);
        const float pt0[2] = {kf.kp[slot(j0)].x, kf.kp[slot(j0)].y}, pt1[2] = {kf.kp[slot(q)].x, kf.kp[slot(q)].y};
        float w[3];
        geom_oracle_triangulate1(pt0, pt1, P0, P1, w);
        const P3 posW = {w[0], w[1], w[2]};
        const P3 pos0 = se3map(T(j0), posW), pos1 = se3map(T(q), posW);
        auto accept = [&](float z) { return z >= prm.lower_depth && z <= prm.upper_depth; };   // Config::acceptDepth
        if (accept(pos0.z) && accept(pos1.z)) {
            float Ti0[16], Ti1[16];
            inv4(T(j0), Ti0);
            inv4(T(q), Ti1);
            const float O0[3] = {Ti0[3], Ti0[7], Ti0[11]}, O1[3] = {Ti1[3], Ti1[7], Ti1[11]};
            if (geom_oracle_check_parallax(O0, O1, w, 2)) {
                float* pm = mp.pos + 3 * m;
                pm[0] = posW.x; pm[1] = posW.y; pm[2] = posW.z;
                mp.good_prl[m] = 1;
                double info0[9], info1[9];
                const float p0f[3] = {pos0.x, pos0.y, pos0.z};
                geom_oracle_xyz_info1(p0f, T(j0), T(q), prm.fx, info0, info1);
                set_view(j0, pos0, info0);
                set_view(q, pos1, info1);
                float R0[9], M0[9], tmp[9], W[9];
                for (int i = 0; i < 3; i++)
                    for (int k = 0; k < 3; k++) R0[i * 3 + k] = T(j0)[i * 4 + k];
                for (int e = 0; e < 9; e++) M0[e] = (float)info0[e];
                gemm3_at_b(R0, M0, tmp);                    // Rcw0.t() * toCvMat(xyzinfo0)
                gemm3_fast(tmp, 3, R0, 3, 3, 1.0, W, 3);    // (...) * Rcw0
                for (int j : obs) {
                    if (id(j) == id(q) || id(j) == id(j0)) continue;
                    const P3 pk = se3map(T(j), posW);
                    float Rk[9], t2[9], Wk[9];
                    for (int i = 0; i < 3; i++)
                        for (int k = 0; k < 3; k++) Rk[i * 3 + k] = T(j)[i * 4 + k];
                    gemm3_fast(Rk, 3, W, 3, 3, 1.0, t2, 3);  // Rcwk * xyzinfoW
                    gemm3_a_bt(t2, Rk, Wk);                  // (...) * Rcwk.t()
                    double info[9];
                    for (int e = 0; e < 9; e++) info[e] = (double)Wk[e];   // toMatrix3d
                    set_view(j, pk, info);
                }
            }
        }
        if (id(q) - id(j0) >= 6 && !mp.good_prl[m]) {
            set_null();
            return true;
        }
        return false;
    }

    // MapPoint::addObservation (MapPoint.cpp:104-122) of the entry at list position q
    bool add(int q) {
        const int oldObsSize = (int)obs.size();
        obs.insert(std::lower_bound(obs.begin(), obs.end(), q), q);
        update_main();
        const bool gone = update_parallax(q);
        const P3 newObs = view(q);
        const P3 newNorm = mul_pd(newObs, 1.f / norm3(newObs));
        float* n = mp.normal + 3 * m;
        const float f = 1.f / (float)(oldObsSize + 1);
        n[0] = (n[0] * (float)oldObsSize + newNorm.x) * f;
        n[1] = (n[1] * (float)oldObsSize + newNorm.y) * f;
        n[2] = (n[2] * (float)oldObsSize + newNorm.z) * f;
        if (mp.null[m]) mp.null[m] = 0;
        return gone;
    }

    // MapPoint::eraseObservation (MapPoint.cpp:86-101) of the entry at list position q
    bool erase(int q) {
        const P3 viewPos = view(q);
        const P3 normPos = mul_pd(viewPos, 1.f / norm3(viewPos));
        obs.erase(std::find(obs.begin(), obs.end(), q));
        if (!mp.null[m] && obs.empty()) {
            set_null();
            return true;
        }
        update_main();
        const int size = (int)obs.size();
        float* n = mp.normal + 3 * m;
        const float f = 1.f / (float)size;
        n[0] = (n[0] * (float)(size + 1) - normPos.x) * f;
        n[1] = (n[1] * (float)(size + 1) - normPos.y) * f;
        n[2] = (n[2] * (float)(size + 1) - normPos.z) * f;
        return false;
    }
};

}  // namespace

// add != 0: addObservation, the lists given after every insertion; add == 0: eraseObservation, the lists given before
MP_EXPORT void mp_oracle_updates(int add, const MpKeyframes* kf, const MpPoints* mp, const int* upd_ptr, const int* upd_pos,
                                 const MpParams* prm, uint8_t* abandoned) {
    for (int m = 0; m < mp->n_mp; m++) {
        Point p{*kf, *mp, *prm, m, mp->obs_ptr[m], {}};
        const int L = mp->obs_ptr[m + 1] - p.p0;
        const int* u0 = upd_pos + upd_ptr[m];
        const int* u1 = upd_pos + upd_ptr[m + 1];
        for (int j = 0; j < L; j++)
            if (!add || std::find(u0, u1, j) == u1) p.obs.push_back(j);
        bool gone = false;
        for (const int* u = u0; u < u1; u++) gone |= add ? p.add(*u) : p.erase(*u);
        abandoned[m] = gone;
    }
}

// MapPoint::updateMeasureInKFs (MapPoint.cpp:294-305) for the listed points
MP_EXPORT void mp_oracle_update_measure(const MpKeyframes* kf, const MpPoints* mp, int n, const int* points) {
    for (int i = 0; i < n; i++) {
        const int m = points[i];
        const P3 pos = {mp->pos[3 * m], mp->pos[3 * m + 1], mp->pos[3 * m + 2]};
        for (int j = mp->obs_ptr[m]; j < mp->obs_ptr[m + 1]; j++) {
            const int k = mp->obs_kf[j];
            if (kf->kf_null[k]) continue;
            const P3 p = se3map(kf->Tcw + 16 * k, pos);
            float* v = kf->view_mp + 3 * (kf->kp_base[k] + mp->obs_idx[j]);
            v[0] = p.x; v[1] = p.y; v[2] = p.z;
        }
    }
}

// the pinned OpenCV pieces, one at a time (oracle/pin_mappoint_against_cv2.py)
MP_EXPORT void mp_oracle_gemm3_a_bt(const float* A, const float* B, float* D) { gemm3_a_bt(A, B, D); }
MP_EXPORT void mp_oracle_rt_m_r(const float* R, const float* M, float* D) {
    float t[9];
    gemm3_at_b(R, M, t);
    gemm3_fast(t, 3, R, 3, 3, 1.0, D, 3);
}
MP_EXPORT void mp_oracle_r_m_rt(const float* R, const float* M, float* D) {
    float t[9];
    gemm3_fast(R, 3, M, 3, 3, 1.0, t, 3);
    gemm3_a_bt(t, R, D);
}
MP_EXPORT double mp_oracle_norm3(const float* p) { return norm3({p[0], p[1], p[2]}); }
MP_EXPORT void mp_oracle_mul_pd(const float* p, double s, float* out) {
    const P3 r = mul_pd({p[0], p[1], p[2]}, s);
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
