// Pin of the L1 score against the reference's own DBoW2 — TEST INFRASTRUCTURE ONLY.
//
// Linked by oracle/dbow2_ref.mk with the reference's Thirdparty/DBoW2/DBoW2/ScoringObject.cpp and BowVector.cpp, compiled
// from the reference tree into oracle/_ref/libdbow2_l1.so: word / value arrays -> DBoW2::BowVector -> L1Scoring().score.
// oracle/pin_l1_score_against_dbow2.py and tests/test_loop_oracle.py load it when it exists.
#include <chrono>
#include <vector>

#include "BowVector.h"
#include "ScoringObject.h"

extern "C" __attribute__((visibility("default"))) double dbow2_l1_score(const int* w1, const double* v1, int n1, const int* w2,
                                                                         const double* v2, int n2) {
    DBoW2::BowVector a, b;
    for (int i = 0; i < n1; ++i) a[w1[i]] = v1[i];
    for (int i = 0; i < n2; ++i) b[w2[i]] = v2[i];
    return DBoW2::L1Scoring().score(a, b);
}

// DetectLoopClose's loop as the reference runs it, for timing on one core: N keyframes' BowVectors (word / value arrays
// strided by cap, counts db_n) are built once; then, `reps` times, each is copied (DBoW2::BowVector BowVec = pKF->mBowVec)
// and scored against the query. Returns the mean milliseconds per query pass; *best receives the largest score.
extern "C" __attribute__((visibility("default"))) double dbow2_l1_detect_ms(const int* qw, const double* qv, int nq, const int* dw,
                                                                             const double* dv, const int* db_n, int cap, int N,
                                                                             int reps, double* best) {
    DBoW2::BowVector q;
    for (int i = 0; i < nq; ++i) q[qw[i]] = qv[i];
    std::vector<DBoW2::BowVector> db(N);
    for (int n = 0; n < N; ++n)
        for (int i = 0; i < db_n[n]; ++i) db[n][dw[(size_t)n * cap + i]] = dv[(size_t)n * cap + i];
    DBoW2::L1Scoring scoring;
    double score_best = 0;
    const auto t0 = std::chrono::steady_clock::now();
    for (int r = 0; r < reps; ++r) {
        score_best = 0;
        for (int n = 0; n < N; ++n) {
            DBoW2::BowVector v = db[n];
            const double s = scoring.score(q, v);
            if (s > score_best) score_best = s;
        }
    }
    const auto t1 = std::chrono::steady_clock::now();
    *best = score_best;
    return std::chrono::duration<double, std::milli>(t1 - t0).count() / reps;
}
