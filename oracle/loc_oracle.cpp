// CPU oracle (TEST INFRASTRUCTURE ONLY) of the Localizer's own logic (reference src/Localizer.cpp) over the flattened static
// map of se2gpu_loc_map, in the reference's types and containers:
//   UpdatePoseCurr (:614-619)   Se2 in float with glibc's cosf / sinf, cv::Mat 4x4 float products through OpenCV's
//                               small-matrix gemm (float sums left to right)
//   MatchLocalMap's flattening  cvu::se3map and cvu::camprjc (Matx33f * Point3f, float sums from 0) and inImgBound
//   UpdateCovisKFCurr (:675-687) std::set intersection of the observed map points (Map::compareViewMPs)
//   UpdateLocalMap (:631-655)   std::set of keyframes, hops over a snapshot copy, std::set union of getAllObsMPs(true)
//   MatchLoopClose (:658-673)   std::map<int,int> walk, KeyFrame::addObservation skipping null points
// oracle/pyloc.py composes these with the ORB, MatchByProjection and pose-BA oracles into Localizer::run.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <vector>

#define LO_EXPORT extern "C" __attribute__((visibility("default")))

namespace {

// the layout of se2gpu_loc_map (include/se2gpu.h)
struct LocMap {
    int n_kf, n_mp;
    const float* kf_Tcw;
    const int *kf_kp_ptr, *kf_obs_mp, *kf_obs_ptr, *kf_obs, *kf_cov_ptr, *kf_cov;
    const float* mp_pos;
    const uint8_t *mp_null, *mp_good_prl, *mp_desc;
    const int* mp_octave;
};

struct Se2 {
    float x = 0, y = 0, theta = 0;
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
            float t = A[4 * r] * B[c];
            for (int k = 1; k < 4; k++) t = t + A[4 * r + k] * B[4 * k + c];
            out[4 * r + c] = (float)((double)t * 1.0 + 0.0);
        }
    std::memcpy(D, out, sizeof out);
}

std::set<int> all_obs_mps(const LocMap& m, int k, bool check_prl) {  // KeyFrame::getAllObsMPs
    std::set<int> s;
    for (int e = m.kf_obs_ptr[k]; e < m.kf_obs_ptr[k + 1]; e++) {
        const int j = m.kf_obs[e];
        if (m.mp_null[j]) continue;
        if (check_prl && !m.mp_good_prl[j]) continue;
        s.insert(j);
    }
    return s;
}

std::set<int> observed(const int* obs_mp, int n) {  // the current keyframe's mObservations keys
    std::set<int> s;
    for (int i = 0; i < n; i++)
        if (obs_mp[i] >= 0) s.insert(obs_mp[i]);
    return s;
}

}  // namespace

// UpdatePoseCurr: Tcw = cTb * Se2(ref.odom - cur.odom).toCvSE3() * bTc * ref.Tcw
LO_EXPORT void loc_oracle_pose(const float* cTb, const float* bTc, const float* odom, const float* ref_odom, const float* ref_Tcw,
                               float* Tcw) {
    const Se2 cur(odom[0], odom[1], odom[2]), ref(ref_odom[0], ref_odom[1], ref_odom[2]);
    const Se2 d = ref - cur;
    float M[16], T[16];
    Se2(d.x, d.y, d.theta).toCvSE3(M);
    matmul4(cTb, M, T);
    matmul4(T, bTc, T);
    matmul4(T, ref_Tcw, Tcw);
}

// cvu::camprjc(K, cvu::se3map(Tcw, pos[i])) and inImgBound (inclusive) for n points: in[i], uv[2i..]
LO_EXPORT void loc_oracle_project(const float* K, const float* T, int n, const float* pos, const float* bounds, uint8_t* in, float* uv) {
    for (int i = 0; i < n; i++) {
        const float* p = pos + 3 * i;
        float c[3], q[3];
        for (int r = 0; r < 3; r++) {
            float s = 0.f;
            s = s + T[4 * r] * p[0]; s = s + T[4 * r + 1] * p[1]; s = s + T[4 * r + 2] * p[2];
            c[r] = s + T[4 * r + 3];
        }
        for (int r = 0; r < 3; r++) {
            float s = 0.f;
            s = s + K[3 * r] * c[0]; s = s + K[3 * r + 1] * c[1]; s = s + K[3 * r + 2] * c[2];
            q[r] = s;
        }
        const float u = q[0] / q[2], v = q[1] / q[2];
        uv[2 * i] = u; uv[2 * i + 1] = v;
        in[i] = u >= bounds[0] && u <= bounds[1] && v >= bounds[2] && v <= bounds[3];
    }
}

// UpdateCovisKFCurr: cov[k] |= local_kfs[k] && |observed(cur) ∩ mObservations(k)| > 0.1 * getSizeObsMP(); returns how
// many keyframes sat exactly on the threshold (count == 0.1 * n, not added)
LO_EXPORT int loc_oracle_covis(const LocMap* m, const uint8_t* local_kfs, const int* obs_mp, int n, uint8_t* cov) {
    const std::set<int> cur = observed(obs_mp, n);
    const int size = (int)cur.size();
    int edge = 0;
    for (int k = 0; k < m->n_kf; k++) {
        if (!local_kfs[k]) continue;
        std::set<int> common;
        for (int j : cur) {  // Map::compareViewMPs: pKF1->getAllObsMPs(false), pKF2->hasObservation(pMP)
            const int* b = m->kf_obs + m->kf_obs_ptr[k];
            const int* e = m->kf_obs + m->kf_obs_ptr[k + 1];
            for (const int* q = b; q != e; q++)
                if (*q == j) { common.insert(j); break; }
        }
        if (common.size() > 0.1 * size) cov[k] = 1;
        else if ((int)common.size() * 10 == size) edge++;  // the integer boundary, excluded by the strict test
    }
    return edge;
}

// UpdateLocalMap(hops): local_kfs [K] and the ascending local map-point list (returns its full length; at most cap written)
LO_EXPORT int loc_oracle_local_map(const LocMap* m, const uint8_t* cov, int hops, uint8_t* local_kfs, int* list, int cap) {
    std::set<int> kfs;
    for (int k = 0; k < m->n_kf; k++)
        if (cov[k]) kfs.insert(k);
    while (hops > 0) {
        const std::set<int> current = kfs;
        for (int k : current)
            for (int e = m->kf_cov_ptr[k]; e < m->kf_cov_ptr[k + 1]; e++) kfs.insert(m->kf_cov[e]);
        hops--;
    }
    std::set<int> mps;
    for (int k : kfs) {
        const std::set<int> s = all_obs_mps(*m, k, true);
        mps.insert(s.begin(), s.end());
    }
    std::memset(local_kfs, 0, m->n_kf);
    for (int k : kfs) local_kfs[k] = 1;
    int i = 0;
    for (int j : mps) {
        if (i < cap) list[i] = j;
        i++;
    }
    return i;
}

// MatchLoopClose over mapMatchGood (the pairs, walked in ascending idxCurr as std::map orders them): obs_mp updated in
// place; returns how many pairs met a null point (skipped) and, in *bad, how many met a point without good parallax
LO_EXPORT int loc_oracle_loop_close(const LocMap* m, int kf, int n, const int* cur, const int* loop, int* obs_mp, int* bad) {
    std::map<int, int> match;
    for (int e = 0; e < n; e++) match[cur[e]] = loop[e];
    int nulls = 0;
    *bad = 0;
    for (const auto& p : match) {
        const int j = m->kf_obs_mp[m->kf_kp_ptr[kf] + p.second];
        if (j < 0) continue;                       // !mpKFLoop->hasObservation(idxLoop)
        if (m->mp_null[j]) { nulls++; continue; }  // KeyFrame::addObservation returns on a null point
        if (!m->mp_good_prl[j]) (*bad)++;
        obs_mp[p.first] = j;
    }
    return nulls;
}
