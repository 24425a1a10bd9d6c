// Loop-closure ORACLE — TEST INFRASTRUCTURE ONLY.
//
// GlobalMapper::DetectLoopClose / VerifyLoopClose (reference src/GlobalMapper.cpp:201-326) and the Localizer's
// (src/Localizer.cpp:337-431), restated over ordered maps:
//   * loop_oracle_score: DBoW2's L1Scoring::score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68) on std::map<int, double>
//     BowVectors: the two-iterator walk with lower_bound jumps, score += fabs(vi - wi) - fabs(vi) - fabs(wi) at each common
//     word, -score / 2.0 at the end;
//   * loop_oracle_detect: the selection loop of both DetectLoopClose (scoreBest = 0, strict >, keyframes in ascending id
//     order, the id-offset exclusion, the strict threshold), each keyframe's BowVector copied as the reference copies it;
//   * loop_oracle_verify_tail: RemoveKPMatch (:1251-1276) on std::map<int, int> with hasObservation as a std::set<int>,
//     and the verdicts.
// Steps 1-2 of VerifyLoopClose (SearchByBoW, RemoveMatchOutlierRansac) are composed in oracle/pyloop.py from the existing
// SearchByBoW and findFundamentalMat oracles. Only tests/ and tools/ load this.
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <set>

namespace {

using BowVector = std::map<int, double>;

BowVector bow(const int* word, const double* value, int n) {
    BowVector v;
    for (int i = 0; i < n; ++i) v[word[i]] = value[i];
    return v;
}

double l1_score(const BowVector& v1, const BowVector& v2) {
    auto v1_it = v1.begin(), v2_it = v2.begin();
    const auto v1_end = v1.end(), v2_end = v2.end();
    double score = 0;
    while (v1_it != v1_end && v2_it != v2_end) {
        const double vi = v1_it->second, wi = v2_it->second;
        if (v1_it->first == v2_it->first) {
            score += std::fabs(vi - wi) - std::fabs(vi) - std::fabs(wi);
            ++v1_it;
            ++v2_it;
        } else if (v1_it->first < v2_it->first) {
            v1_it = v1.lower_bound(v2_it->first);
        } else {
            v2_it = v2.lower_bound(v1_it->first);
        }
    }
    return -score / 2.0;
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) double loop_oracle_score(const int* w1, const double* v1, int n1, const int* w2,
                                                                const double* v2, int n2) {
    return l1_score(bow(w1, v1, n1), bow(w2, v2, n2));
}

// B queries against N keyframes, BowVectors strided by cap as the device writes them; scores [B*N], loop [B], best [B]
__attribute__((visibility("default"))) void loop_oracle_detect(int B, const int* q_word, const double* q_value, const int* q_n,
                                                               int cap_q, int N, const int* db_word, const double* db_value,
                                                               const int* db_n, int cap_db, const int* q_id, const int* db_id,
                                                               int min_id_offset, double min_score, double* scores, int* loop,
                                                               double* best) {
    std::map<int, BowVector> db;   // Map::getAllKF(): the keyframes in ascending order
    for (int n = 0; n < N; ++n) db[n] = bow(db_word + (size_t)n * cap_db, db_value + (size_t)n * cap_db, db_n[n]);
    for (int b = 0; b < B; ++b) {
        const BowVector cur = bow(q_word + (size_t)b * cap_q, q_value + (size_t)b * cap_q, q_n[b]);
        int kf_best = -1;
        double score_best = 0;
        for (const auto& kv : db) {
            const BowVector v = kv.second;   // DBoW2::BowVector BowVec = pKF->mBowVec;
            const double score = l1_score(cur, v);
            scores[(size_t)b * N + kv.first] = score;
            if (min_id_offset > 0 && std::abs(db_id[kv.first] - q_id[b]) < min_id_offset) continue;
            if (score > score_best) {
                score_best = score;
                kf_best = kv.first;
            }
        }
        loop[b] = (kf_best >= 0 && score_best > min_score) ? kf_best : -1;
        best[b] = score_best;
    }
}

// good [n1] the matches after RemoveMatchOutlierRansac (-1 = none); obs_cur [n1] / obs_loop [n2] hasObservation(idx).
// mp [n1] receives RemoveKPMatch's result (all -1 for the Localizer), counts [3] (raw, good, MP); returns the verdict.
__attribute__((visibility("default"))) int loop_oracle_verify_tail(int n1, const int* raw, const int* good, const uint8_t* obs_cur,
                                                                   int n2, const uint8_t* obs_loop, int localizer, int min_match_mp,
                                                                   int min_match_kp, double ratio_min_match_mp, int num_mps_current,
                                                                   int* mp, int* counts) {
    std::map<int, int> map_raw, map_match;
    std::set<int> dual_cur, dual_loop;   // mDualObservations' keys
    for (int i = 0; i < n1; ++i) {
        if (raw[i] >= 0) map_raw[i] = raw[i];
        if (good[i] >= 0) map_match[i] = good[i];
        if (obs_cur[i]) dual_cur.insert(i);
        mp[i] = -1;
    }
    for (int j = 0; j < n2; ++j)
        if (obs_loop[j]) dual_loop.insert(j);
    const int num_good_match = (int)map_match.size();
    counts[0] = (int)map_raw.size();
    counts[1] = num_good_match;
    if (localizer) {
        counts[2] = 0;
        return num_good_match >= min_match_kp;
    }
    std::map<int, int> map_mp = map_match;   // RemoveKPMatch
    for (auto it = map_match.begin(); it != map_match.end(); ++it)
        if (!(dual_cur.count(it->first) && dual_loop.count(it->second))) map_mp.erase(it->first);
    for (const auto& kv : map_mp) mp[kv.first] = kv.second;
    const int num_good_mp_match = (int)map_mp.size();
    counts[2] = num_good_mp_match;
    const double ratio_mp_matched = num_good_mp_match * 1.0 / num_mps_current;
    return num_good_mp_match >= min_match_mp && num_good_match >= min_match_kp && ratio_mp_matched >= ratio_min_match_mp;
}

}  // extern "C"
