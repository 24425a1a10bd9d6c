// Loop closure on sm_90a — kernels + C ABI (include/se2gpu.h: se2gpu_detect_loop_device, se2gpu_verify_loop_device).
//
// Replaces GlobalMapper::DetectLoopClose / VerifyLoopClose (reference src/GlobalMapper.cpp:201-326, 1207-1276) and the
// Localizer's (src/Localizer.cpp:337-431) for a batch of query keyframes, on the BowVectors and FeatureVectors
// se2gpu_voc_compute_bow_device writes (DESIGN.md section 2d).
//   k_bow_score     DBoW2's L1Scoring::score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68) of every (query, database
//                   keyframe): one warp per pair, the query's BowVector staged in shared memory. The warp walks the
//                   database keyframe's word list 32 words at a time (coalesced loads) and finds each word in the staged
//                   query by binary search in shared memory; the terms of the common words are then added by every lane
//                   in the same ascending word order, one after the other, in double precision. The result is the
//                   reference's sequential fold bit for bit: its
//                   lower_bound jumps only skip words the other vector lacks. blockIdx.x is the query, so the B CTAs that
//                   read one chunk of database keyframes are adjacent in the launch order and share it through L2.
//   k_loop_select   the selection loop of DetectLoopClose, one CTA per query: the largest score > 0 of the keyframes the id
//                   offset does not exclude, the lowest slot among equal scores (the reference keeps the first on a strict
//                   >), then the strict threshold. Comparisons are exact, so a parallel argmax is exact.
//   verify          SearchByBoW (matcher.cu) -> copy raw -> good -> RemoveMatchOutlierRansac (fundam.cu's
//                   k_remove_outliers_loop) -> k_loop_verdict: RemoveKPMatch, the three counts and the acceptance test,
//                   one CTA per pair.
#include "common.h"

namespace {

using se2gpu::fail;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kDbPerCta = 16;         // database keyframes per score CTA (two per warp)
constexpr int kScoreBytesPerWord = 12; // staged query BowVector: int word + double value

struct ScoreArgs {
    const int* q_word; const double* q_value; const int* q_n; int cap_q;
    const int* db_word; const double* db_value; const int* db_n; int cap_db; int N;
    double* scores;
};

// Dynamic shared memory: double value[cap_q], int word[cap_q].
__global__ void __launch_bounds__(kThreads) k_bow_score(ScoreArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    double* s_val = reinterpret_cast<double*>(smem);
    int* s_word = reinterpret_cast<int*>(s_val + a.cap_q);
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nq = min(max(a.q_n[b], 0), a.cap_q);
    for (int i = threadIdx.x; i < nq; i += kThreads) {
        s_word[i] = a.q_word[(size_t)b * a.cap_q + i];
        s_val[i] = a.q_value[(size_t)b * a.cap_q + i];
    }
    __syncthreads();
    for (int k = warp; k < kDbPerCta; k += kWarps) {
        const int n = blockIdx.y * kDbPerCta + k;
        if (n >= a.N) break;
        const int* dw = a.db_word + (size_t)n * a.cap_db;
        const double* dv = a.db_value + (size_t)n * a.cap_db;
        const int nd = min(max(a.db_n[n], 0), a.cap_db);
        double score = 0.0;
        for (int i0 = 0; i0 < nd; i0 += 32) {
            const int i = i0 + lane;
            bool hit = false;
            double t = 0.0;
            if (i < nd) {
                const int w = dw[i];
                int lo = 0, hi = nq;
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_word[mid] < w) lo = mid + 1; else hi = mid; }
                if (lo < nq && s_word[lo] == w) {
                    const double vi = s_val[lo], wi = dv[i];
                    // fabs(vi - wi) - fabs(vi) - fabs(wi), left to right
                    t = __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi));
                    hit = true;
                }
            }
            // score += t in ascending word order: every lane adds the same terms in the same order
            for (unsigned m = __ballot_sync(0xffffffffu, hit); m; m &= m - 1)
                score = __dadd_rn(score, __shfl_sync(0xffffffffu, t, __ffs(m) - 1));
        }
        if (lane == 0) a.scores[(size_t)b * a.N + n] = __ddiv_rn(-score, 2.0);
    }
}

struct SelectArgs {
    const double* scores; int N;
    const int* q_id; const int* db_id; int min_id_offset; double min_score;
    int* loop; double* best;
};

// (score, slot) a beats (score, slot) b: a is a candidate and b is none, or a's score is larger, or equal with a lower slot
__device__ __forceinline__ bool beats(double sa, int na, double sb, int nb) {
    return na >= 0 && (nb < 0 || sa > sb || (sa == sb && na < nb));
}

__global__ void __launch_bounds__(kThreads) k_loop_select(SelectArgs a) {
    __shared__ double s_s[kWarps];
    __shared__ int s_n[kWarps];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double* sc = a.scores + (size_t)b * a.N;
    const int id = a.min_id_offset > 0 ? a.q_id[b] : 0;
    // scoreBest starts at 0.0 and a keyframe replaces the best only on a strict >; each thread visits its slots in
    // ascending order, so it keeps its first maximum
    double bs = 0.0;
    int bn = -1;
    for (int n = threadIdx.x; n < a.N; n += kThreads) {
        if (a.min_id_offset > 0 && abs(a.db_id[n] - id) < a.min_id_offset) continue;   // omit neighbour keyframes
        const double v = sc[n];
        if (v > bs) { bs = v; bn = n; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, bs, o);
        const int on = __shfl_xor_sync(0xffffffffu, bn, o);
        if (beats(os, on, bs, bn)) { bs = os; bn = on; }
    }
    if (lane == 0) { s_s[warp] = bs; s_n[warp] = bn; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kWarps; ++w)
            if (beats(s_s[w], s_n[w], bs, bn)) { bs = s_s[w]; bn = s_n[w]; }
        a.loop[b] = (bn >= 0 && bs > a.min_score) ? bn : -1;
        a.best[b] = bs;
    }
}

struct VerdictArgs {
    int cap1, cap2; const int* slot2;
    const int* raw; const int* good; int* mp;
    const uint8_t* obs1; const uint8_t* obs2;   // hasObservation(idx) of the current / loop keyframe (GlobalMapper)
    const int* n_mps_cur;
    se2gpu_loop_verify_params p;
    int* counts; uint8_t* verified;
};

__device__ __forceinline__ int block_sum(int v, int* s_red) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
    for (int w = 0; w < kWarps; ++w) t += s_red[w];
    __syncthreads();
    return t;
}

// RemoveKPMatch (GlobalMapper.cpp:1251-1276) and the verdict of VerifyLoopClose, one CTA per pair
__global__ void __launch_bounds__(kThreads) k_loop_verdict(VerdictArgs a) {
    __shared__ int s_red[kWarps];
    const int b = blockIdx.x;
    const int s2 = a.slot2[b];
    const size_t o1 = (size_t)b * a.cap1;
    const bool gm = !a.p.localizer;
    int nraw = 0, ngood = 0, nmp = 0;
    for (int i = threadIdx.x; i < a.cap1; i += kThreads) {
        const int r = a.raw[o1 + i], g = a.good[o1 + i];
        int m = -1;
        // a good match exists only for s2 >= 0 (an empty pair has none), so obs2 is read only at a real slot
        if (gm && g >= 0 && a.obs1[o1 + i] && a.obs2[(size_t)s2 * a.cap2 + g]) m = g;
        a.mp[o1 + i] = m;
        nraw += r >= 0; ngood += g >= 0; nmp += m >= 0;
    }
    nraw = block_sum(nraw, s_red);
    ngood = block_sum(ngood, s_red);
    nmp = block_sum(nmp, s_red);
    if (threadIdx.x == 0) {
        a.counts[3 * b] = nraw; a.counts[3 * b + 1] = ngood; a.counts[3 * b + 2] = nmp;
        bool ok;
        if (gm) {
            // numGoodMPMatch * 1.0 / numMPsCurrent in double: 0 / 0 is NaN and fails, x / 0 is +inf and passes
            const double ratio = __ddiv_rn((double)nmp, (double)a.n_mps_cur[b]);
            ok = nmp >= a.p.min_match_mp && ngood >= a.p.min_match_kp && ratio >= a.p.ratio_min_match_mp;
        } else {
            ok = ngood >= a.p.min_match_kp;
        }
        a.verified[b] = ok ? 1 : 0;
    }
}

// the opt-in shared memory k_bow_score may use on the current device, raised once per device
int score_smem_limit(int* limit) {
    static std::mutex mu;
    static int ready[se2gpu::kMaxDevices] = {};
    int dev = 0, optin = 0;
    SE2_CUDA(cudaGetDevice(&dev));
    SE2_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    *limit = optin;
    std::lock_guard<std::mutex> lk(mu);
    if (dev < se2gpu::kMaxDevices && ready[dev]) return SE2GPU_OK;
    SE2_CUDA(cudaFuncSetAttribute(k_bow_score, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    if (dev < se2gpu::kMaxDevices) ready[dev] = 1;
    return SE2GPU_OK;
}

}  // namespace

extern "C" {

int se2gpu_detect_loop_device(int B, const int* d_q_word, const double* d_q_value, const int* d_q_n, int cap_q, int N,
                              const int* d_db_word, const double* d_db_value, const int* d_db_n, int cap_db, const int* d_q_id,
                              const int* d_db_id, const se2gpu_loop_detect_params* params, double* d_scores, int* d_loop,
                              double* d_best, void* stream) {
    if (!params) return fail(SE2GPU_ERR_INVALID, "null parameters");
    if (B < 0 || N < 0 || cap_q < 0 || cap_db < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (B > 0) {
        const bool ids = params->min_id_offset > 0;
        if (!d_q_n || !d_loop || !d_best || (N && !d_scores) || (cap_q && (!d_q_word || !d_q_value)) ||
            (N && (!d_db_n || (cap_db && (!d_db_word || !d_db_value)))) || (ids && (!d_q_id || (N && !d_db_id))))
            return fail(SE2GPU_ERR_INVALID, "null argument");
    }
    { const int rc = se2gpu::require_device(); if (rc) return rc; }
    if ((long long)N > 65535LL * kDbPerCta)
        return fail(SE2GPU_ERR_CAPACITY, "%d database keyframes exceed %d", N, 65535 * kDbPerCta);
    int smem_limit = 0;
    { const int rc = score_smem_limit(&smem_limit); if (rc) return rc; }
    if ((long long)cap_q * kScoreBytesPerWord > smem_limit)
        return fail(SE2GPU_ERR_CAPACITY, "cap_q = %d exceeds the %d words the query's shared memory holds", cap_q,
                    smem_limit / kScoreBytesPerWord);
    SE2_NVTX("se2gpu.detect_loop");
    if (B == 0) return SE2GPU_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const ScoreArgs sa{d_q_word, d_q_value, d_q_n, cap_q, d_db_word, d_db_value, d_db_n, cap_db, N, d_scores};
    SE2_LAUNCH(k_bow_score, dim3(B, std::max((N + kDbPerCta - 1) / kDbPerCta, 1)), kThreads, (size_t)kScoreBytesPerWord * cap_q,
               s, sa);
    const SelectArgs se{d_scores, N, d_q_id, d_db_id, params->min_id_offset, params->min_score, d_loop, d_best};
    SE2_LAUNCH(k_loop_select, B, kThreads, 0, s, se);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_verify_loop_device(se2gpu_matcher* m, int B, const se2gpu_bow_batch_kf* cur, const se2gpu_bow_batch_kf* map,
                              const int* d_loop, const int* d_n_mps_cur, const se2gpu_loop_verify_params* params, int* d_raw,
                              int* d_good, int* d_mp, int* d_counts, uint8_t* d_verified, void* stream) {
    if (!m || !cur || !map || !params) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (B < 0 || cur->cap < 0 || map->cap < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (cur->cap > se2gpu::kFundamMaxPairs)
        return fail(SE2GPU_ERR_CAPACITY, "cur->cap = %d exceeds the outlier kernel's %d keypoints", cur->cap, se2gpu::kFundamMaxPairs);
    const bool gm = !params->localizer;
    if (B > 0 && (!d_loop || !d_raw || !d_good || !d_mp || !d_counts || !d_verified ||
                  (gm && (!d_n_mps_cur || (cur->cap && !cur->has_mp) || (map->cap && !map->has_mp)))))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    // SearchByBoW(cur, loop, mapMatch, bIfMatchMPOnly = false) with ORBmatcher()'s nnratio 0.6 and orientation check; it
    // checks B and both caps against the matcher and writes nothing when it refuses
    { const int rc = se2gpu_search_by_bow_batch_device(m, B, cur, map, d_loop, 0, 0.6f, 1, d_raw, nullptr, stream); if (rc) return rc; }
    SE2_NVTX("se2gpu.verify_loop");
    if (B == 0) return SE2GPU_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int cap1 = cur->cap, cap2 = map->cap;
    SE2_CUDA(cudaMemcpyAsync(d_good, d_raw, sizeof(int) * (size_t)B * cap1, cudaMemcpyDeviceToDevice, s));
    { const int rc = se2gpu::remove_outliers_loop(B, cur->kp, cap1, map->kp, cap2, d_loop, d_good, s); if (rc) return rc; }
    const VerdictArgs va{cap1, cap2, d_loop, d_raw, d_good, d_mp, cur->has_mp, map->has_mp, d_n_mps_cur, *params, d_counts, d_verified};
    SE2_LAUNCH(k_loop_verdict, B, kThreads, 0, s, va);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

}  // extern "C"
