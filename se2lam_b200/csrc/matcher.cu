// ORB matchers on sm_90a — kernels + C ABI (include/se2gpu.h: se2gpu_hamming_distance, se2gpu_matcher_*,
// se2gpu_match_by_window[_device], se2gpu_match_by_projection[_device], se2gpu_search_by_bow).
//
// Replaces se2lam::ORBmatcher (reference src/ORBmatcher.cpp) and the Frame keypoint grid it queries
// (src/Frame.cpp:64-77, 209-286). A matcher handle owns every device buffer (no allocation per call); the device entry
// points consume the extractor's keypoint / descriptor buffers where they lie in HBM (reference call chain
// Track.cpp:129-132: extract -> MatchByWindow back to back). Three launches per call:
//   k_grid_build   Frame::PosInGrid for every database keypoint and the (column, row, index) order of the grid walk
//   k_candidates   one warp per query: which database keypoints fall in the query's grid window (GetFeaturesInArea
//                  semantics incl. its cell-range rounding and level filter) and their 256-bit Hamming distances
//                  (__popc over 8 x 32 bit == DescriptorDistance :110-126), emitted IN THE REFERENCE'S CANDIDATE ORDER
//   k_resolve      the order-dependent greedy resolution (best / second best with the "already matched better" skip,
//                  steal-back, :308-346, :415-449, :187-246) as SPECULATIVE ROUNDS in one CTA: every query is resolved
//                  in parallel against the claims of the previous round (claims of EARLIER queries only), claims are
//                  rebuilt, and the rounds repeat until no decision changes. A fixed point of that iteration is the
//                  sequential result (induction over the query index: query 0 depends on nothing, query t only on
//                  queries < t), so the output is bit-identical to the reference loop; the number of rounds is the
//                  length of the longest dependency chain (a handful), not the number of queries. The rotation histogram
//                  (:350-372), steal accounting and the vbPrevMatched update run in the same kernel.
//   k_fallback_*   the one-warp sequential loop, kept as the exact fallback when a database keypoint collects more
//                  simultaneous claims than the shared-memory claim table holds (flag set by k_resolve; returns at once
//                  otherwise).
// The device entry points take a batch of B independent frame pairs (se2gpu_match_by_*_batch_device; the single-pair entry
// points are B = 1): the grid and candidate kernels take the pair from blockIdx.y, k_resolve runs one CTA and k_fallback_*
// one warp per pair, and every pair works in its own slice of the context's scratch. The launch count does not depend on B.
// se2gpu_search_by_bow_batch_device puts k_bow_walk in front, one CTA per pair: the node walk of SearchByBoW (:160-247) over
// the two device FeatureVectors, which writes the pair's queries for k_candidates_bow. A negative d_slot2[b] makes pair b empty:
// k_bow_walk gives it no queries, so no later kernel reads its side 2, and the side-2 offsets are formed from slot 0.
#include <climits>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.h"

struct se2gpu_matcher {
    int device = 0;
    int max_q = 0, max_db = 0, max_batch = 1;
    cudaStream_t stream = nullptr;      // host entry points run here
    // device scratch (sized at creation), one slice per frame pair: pair b's slice starts at b * (the size given here)
    int *cell = nullptr, *order = nullptr, *nvalid = nullptr;   // [max_db], [max_db], [1]
    int2* cand = nullptr;               // [max_q][max_db] (index, dist | octave << 16)
    int* ncand = nullptr;               // [max_q]
    int* work = nullptr;                // fallback: [2 * max_db + max_q]
    int* flags = nullptr;               // [0] fallback needed, [1] rounds of the last resolve
    int* nm = nullptr;                  // match count of the last call
    int *bow_q = nullptr, *bow_nq = nullptr;   // SearchByBoW batch: [max_batch][3][max_q] (feature, KF2 range), [max_batch] count
    std::vector<int> seq_flags;         // [max_batch][2] = {1, 0}: the flags of every pair when the sequential kernel runs alone
    int last_batch = 0;                 // pairs of the last resolve
    // device + pinned staging of the host entry points
    se2gpu_keypoint *d_kp1 = nullptr, *d_kp2 = nullptr;
    uint8_t *d_desc1 = nullptr, *d_desc2 = nullptr, *d_u8a = nullptr, *d_u8b = nullptr;
    float *d_f1 = nullptr, *d_f2 = nullptr;
    int *d_i1 = nullptr, *d_i2 = nullptr, *d_i3 = nullptr, *d_i4 = nullptr, *d_out = nullptr;
    se2gpu::PinnedArena pin; size_t pin_bytes = 0;
    se2gpu::DeviceBuffers bufs;
    se2gpu::Profiler prof;
    int resolve_smem_max = 0;
};

namespace {

using se2gpu::count_of;
using se2gpu::fail;
using se2gpu::hamming256;

constexpr int TH_HIGH = 100, TH_LOW = 75, HISTO_LENGTH = 30;   // ORBmatcher.cpp:45-47
constexpr int GRID_ROWS = 48, GRID_COLS = 64;                  // Frame.h:26-27
constexpr int MODE_WINDOW = 0, MODE_PROJ = 1, MODE_BOW = 2;

__global__ void k_hamming_pairs(const uint32_t* a, const uint32_t* b, int n, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = hamming256(a + 8 * (size_t)i, b + 8 * (size_t)i);
}

// Frame::PosInGrid (Frame.cpp:209-220) for every database keypoint and the grid-walk order (cell column, cell row,
// insertion index) of the valid ones by rank counting. Every CTA computes ALL sort keys (cell << 13 | index, INT_MAX for
// keypoints outside the grid) into its shared memory - redundant but cheaper than a grid-wide dependency - and ranks its
// own 128 keypoints against them with broadcast shared-memory reads. CTA 0 also publishes the number of valid keypoints.
// Pair blockIdx.y reads keypoints kp[b * n_cap ..] and count d_n[b], and writes cell / order [b * scr ..] and n_valid[b].
constexpr int GRID_SMEM_KEYS = 8192;
__device__ __forceinline__ int grid_cell_of(const se2gpu_keypoint& p, const se2gpu_grid_params& g) {
    const int px = (int)roundf(__fmul_rn(__fsub_rn(p.x, g.min_x), g.inv_w));
    const int py = (int)roundf(__fmul_rn(__fsub_rn(p.y, g.min_y), g.inv_h));
    return (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? -1 : px * GRID_ROWS + py;
}
__global__ void __launch_bounds__(128) k_grid_build(const se2gpu_keypoint* __restrict__ kp, int n_cap, const int* __restrict__ d_n,
                                                    se2gpu_grid_params g, int* __restrict__ cell, int* __restrict__ order,
                                                    int* __restrict__ n_valid, int scr) {
    __shared__ int keys[GRID_SMEM_KEYS];
    const int b = blockIdx.y;
    kp += (size_t)b * n_cap; cell += (size_t)b * scr; order += (size_t)b * scr; n_valid += b;
    if (d_n) d_n += b;
    const int n = count_of(d_n, n_cap);
    int nv = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int c = grid_cell_of(kp[i], g);
        keys[i] = c < 0 ? INT_MAX : (c << 13) | i;
        nv += c >= 0;
    }
    nv = __syncthreads_count(0) + nv;      // barrier; (count of a false predicate is 0)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int ki = keys[i];
        cell[i] = ki == INT_MAX ? -1 : ki >> 13;
        if (ki != INT_MAX) {
            int r = 0;
            for (int j = 0; j < n; ++j) r += keys[j] < ki;
            order[r] = i;
        }
    }
    if (blockIdx.x == 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(0xffffffffu, nv, o);
        __shared__ int part[4];
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = nv;
        __syncthreads();
        if (threadIdx.x == 0) *n_valid = part[0] + part[1] + part[2] + part[3];
    }
}
// the same for more keypoints than the shared-memory key table holds: cells first, then ranks from global memory
__global__ void k_grid_cell_big(const se2gpu_keypoint* __restrict__ kp, int n_cap, const int* __restrict__ d_n, se2gpu_grid_params g,
                                int* __restrict__ cell, int scr) {
    const int b = blockIdx.y;
    kp += (size_t)b * n_cap; cell += (size_t)b * scr;
    if (d_n) d_n += b;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count_of(d_n, n_cap)) cell[i] = grid_cell_of(kp[i], g);
}
__global__ void k_grid_order_big(const int* __restrict__ cell, int n_cap, const int* __restrict__ d_n, int* __restrict__ order,
                                 int* __restrict__ n_valid, int scr) {
    const int b = blockIdx.y;
    cell += (size_t)b * scr; order += (size_t)b * scr; n_valid += b;
    if (d_n) d_n += b;
    const int n = count_of(d_n, n_cap);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int ci = cell[i];
    if (ci < 0) return;
    int r = 0;
    for (int j = 0; j < n; ++j) { const int cj = cell[j]; r += (cj >= 0) && (cj < ci || (cj == ci && j < i)); }
    order[r] = i;
    atomicAdd(n_valid, 1);
}

struct CandArgs {
    int mode;
    int nq_cap; const int* d_nq;
    // WINDOW: query q = keypoint q of frame 1 searched around vbPrevMatched[q] (ORBmatcher.cpp:292-300)
    const se2gpu_keypoint* kp1; const float* prev; int min_level, max_level, level_offset; int win_size;
    // PROJ: query q = map point q (ORBmatcher.cpp:390-404): mp_valid, predictUV, mMainOctave
    const uint8_t* mp_valid; const float* mp_uv; const int* mp_octave;
    const uint32_t* qdesc;
    // database = keypoints of frame 2 / of the keyframe
    const se2gpu_keypoint* kp; const uint32_t* desc; const int* cell; const int* order; const int* n_valid; const uint8_t* db_skip;
    int db_cap;                       // database items per pair (the pair stride of kp, desc, db_skip)
    se2gpu_grid_params g;
    int cap; int2* cand; int* ncand;  // cap = max_db: row stride of cand, pair stride of cell / order
    int scr_q;                        // max_queries: rows of cand and entries of ncand per pair
};

// pair b's slice of every array (pair-strided inputs, context scratch)
__device__ __forceinline__ void pair_slice(CandArgs& a, int b) {
    const size_t q = (size_t)b * a.nq_cap, d = (size_t)b * a.db_cap;
    if (a.d_nq) a.d_nq += b;
    if (a.mode == MODE_WINDOW) { a.kp1 += q; a.prev += 2 * q; }
    else { a.mp_valid += q; a.mp_uv += 2 * q; a.mp_octave += q; }
    a.qdesc += 8 * q;
    a.kp += d; a.desc += 8 * d;
    if (a.db_skip) a.db_skip += d;
    a.cell += (size_t)b * a.cap; a.order += (size_t)b * a.cap; a.n_valid += b;
    a.cand += (size_t)b * a.scr_q * a.cap; a.ncand += (size_t)b * a.scr_q;
}

// Frame::GetFeaturesInArea (Frame.cpp:222-286) for one query per warp + DescriptorDistance of every hit.
// cand[q*cap + k] = (i2, dist | octave << 16) in the reference's iteration order; ncand[q] = hits. Pair = blockIdx.y.
__global__ void __launch_bounds__(256) k_candidates(CandArgs a) {
    pair_slice(a, blockIdx.y);
    const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nq = count_of(a.d_nq, a.nq_cap);
    if (q >= a.nq_cap) return;
    if (q >= nq) { if (lane == 0) a.ncand[q] = 0; return; }
    int count = 0;
    bool valid;
    float x, y, r;
    int minLevel, maxLevel;
    if (a.mode == MODE_WINDOW) {
        const int l = a.kp1[q].octave;
        valid = !(l > a.max_level || l < a.min_level);
        x = a.prev[2 * q]; y = a.prev[2 * q + 1]; r = (float)a.win_size;
        minLevel = l - a.level_offset > 0 ? l - a.level_offset : 0; maxLevel = l + a.level_offset;
    } else {
        const int pl = a.mp_octave[q];
        valid = a.mp_valid[q] != 0;
        x = a.mp_uv[2 * q]; y = a.mp_uv[2 * q + 1]; r = (float)(pl * a.win_size);
        minLevel = pl > a.level_offset ? pl - a.level_offset : 0; maxLevel = pl + a.level_offset;
    }
    if (valid) {
        const se2gpu_grid_params g = a.g;
        int x0 = (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, g.min_x), r), g.inv_w));
        int x1 = (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, g.min_x), r), g.inv_w));
        int y0 = (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, g.min_y), r), g.inv_h));
        int y1 = (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, g.min_y), r), g.inv_h));
        x0 = max(0, x0); x1 = min(GRID_COLS - 1, x1); y0 = max(0, y0); y1 = min(GRID_ROWS - 1, y1);
        const bool empty = x0 >= GRID_COLS || x1 < 0 || y0 >= GRID_ROWS || y1 < 0;
        const bool check = !(minLevel == -1 && maxLevel == -1);
        const int nv = *a.n_valid;
        const uint32_t* qd = a.qdesc + 8 * (size_t)q;
        if (!empty)
            for (int k0 = 0; k0 < nv; k0 += 32) {
                const int k = k0 + lane;
                bool hit = false;
                int i2 = -1, oct = 0;
                if (k < nv) {
                    i2 = a.order[k];
                    const int c = a.cell[i2], cx = c / GRID_ROWS, cy = c - cx * GRID_ROWS;
                    hit = cx >= x0 && cx <= x1 && cy >= y0 && cy <= y1;
                    if (hit) {
                        const se2gpu_keypoint p = a.kp[i2];
                        oct = p.octave;
                        if (check) hit = p.octave >= minLevel && p.octave <= maxLevel;
                        hit = hit && !(fabsf(__fsub_rn(p.x, x)) > r || fabsf(__fsub_rn(p.y, y)) > r);
                        if (a.db_skip) hit = hit && !a.db_skip[i2];
                    }
                }
                const unsigned bal = __ballot_sync(0xffffffffu, hit);
                if (hit) {
                    const int pos = count + __popc(bal & ((1u << lane) - 1));
                    if (pos < a.cap) a.cand[(size_t)q * a.cap + pos] = make_int2(i2, hamming256(qd, a.desc + 8 * (size_t)i2) | (oct << 16));
                }
                count += __popc(bal);
            }
    }
    if (lane == 0) a.ncand[q] = min(count, a.cap);
}

// SearchByBoW candidates (ORBmatcher.cpp:166-204): query q = feature qidx[q] of KF1 (node-walk order), its candidates are
// the features of the same vocabulary node in KF2, in the node's feature order. Pair = blockIdx.y: KF1 at b * cap1, KF2 at
// slot2[b] * cap2 (slot2 NULL: b), the queries at b * qstride and the candidate rows in the pair's scratch slice.
struct BowCandArgs {
    int nq_cap; const int* d_nq;                       // queries per pair: capacity and device count (NULL: nq_cap)
    const int* qidx; const int* qb0; const int* qb1;   // KF1 feature and its KF2 feat range [qb0, qb1), per query
    int qstride;
    const uint32_t* d1; const uint8_t* mp1; int cap1;
    const int* feat2; const uint32_t* d2; const uint8_t* mp2; int cap2; const int* slot2;
    int mp_only;
    int cap; int2* cand; int* ncand; int scr_q;
};
// side-2 keyframe of pair b; a negative slot (an empty pair) is mapped to 0, whose arrays its kernels then never read
__device__ __forceinline__ int side2_slot(const int* slot2, int b) { return slot2 ? max(slot2[b], 0) : b; }
__device__ __forceinline__ void pair_slice(BowCandArgs& a, int b) {
    const size_t s2 = (size_t)side2_slot(a.slot2, b) * a.cap2, q = (size_t)b * a.qstride;
    if (a.d_nq) a.d_nq += b;
    a.qidx += q; a.qb0 += q; a.qb1 += q;
    a.d1 += 8 * (size_t)b * a.cap1; if (a.mp1) a.mp1 += (size_t)b * a.cap1;
    a.feat2 += s2; a.d2 += 8 * s2; if (a.mp2) a.mp2 += s2;
    a.cand += (size_t)b * a.scr_q * a.cap; a.ncand += (size_t)b * a.scr_q;
}
__global__ void __launch_bounds__(256) k_candidates_bow(BowCandArgs a) {
    pair_slice(a, blockIdx.y);
    const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (q >= count_of(a.d_nq, a.nq_cap)) return;
    const int idx1 = a.qidx[q];
    int count = 0;
    if (!(a.mp_only && !a.mp1[idx1])) {
        const int b0 = a.qb0[q], b1 = a.qb1[q];
        for (int k0 = b0; k0 < b1; k0 += 32) {
            const int k = k0 + lane;
            bool hit = false;
            int idx2 = -1;
            if (k < b1) { idx2 = a.feat2[k]; hit = !(a.mp_only && !a.mp2[idx2]); }
            const unsigned bal = __ballot_sync(0xffffffffu, hit);
            if (hit) {
                const int pos = count + __popc(bal & ((1u << lane) - 1));
                if (pos < a.cap) a.cand[(size_t)q * a.cap + pos] = make_int2(idx2, hamming256(a.d1 + 8 * (size_t)idx1, a.d2 + 8 * (size_t)idx2));
            }
            count += __popc(bal);
        }
    }
    if (lane == 0) a.ncand[q] = min(count, a.cap);
}

// The two-iterator walk of SearchByBoW over the ascending node ids (:160-247) for pair blockIdx.x, on the FeatureVectors
// se2gpu_voc_compute_bow_device writes: every KF1 node is looked up in KF2's node list by binary search (both lists are
// ascending and free of repeats, so a node is common exactly when the walk stops on it), and the features of the common
// nodes become the queries, numbered in walk order by an exclusive sum over the nodes in ascending order.
struct BowWalkArgs {
    const int* node1; const int* ptr1; const int* feat1; const int* n_node1; int cap1;
    const int* node2; const int* ptr2; const int* n_node2; int cap2; const int* slot2;
    int* qidx; int* qb0; int* qb1; int qstride; int* nq;
};
__global__ void __launch_bounds__(256) k_bow_walk(BowWalkArgs a) {
    __shared__ int s_warp[32];
    const int b = blockIdx.x, s2 = side2_slot(a.slot2, b);
    const bool empty = a.slot2 && a.slot2[b] < 0;
    const int* node1 = a.node1 + (size_t)b * a.cap1; const int* ptr1 = a.ptr1 + (size_t)b * (a.cap1 + 1);
    const int* feat1 = a.feat1 + (size_t)b * a.cap1;
    const int* node2 = a.node2 + (size_t)s2 * a.cap2; const int* ptr2 = a.ptr2 + (size_t)s2 * (a.cap2 + 1);
    const int n1 = min(max(a.n_node1[b], 0), a.cap1), n2 = empty ? 0 : min(max(a.n_node2[s2], 0), a.cap2);
    const size_t qo = (size_t)b * a.qstride;
    int *qidx = a.qidx + qo, *qb0 = a.qb0 + qo, *qb1 = a.qb1 + qo;
    int base = 0;
    for (int a0 = 0; a0 < n1; a0 += blockDim.x) {
        const int i = a0 + threadIdx.x;
        int c = 0, j = -1;
        if (i < n1) {
            const int nd = node1[i];
            int lo = 0, hi = n2;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (node2[mid] < nd) lo = mid + 1; else hi = mid; }
            if (lo < n2 && node2[lo] == nd) { j = lo; c = ptr1[i + 1] - ptr1[i]; }
        }
        int total;
        const int off = base + se2gpu::block_exclusive_sum(c, total, s_warp);
        if (c > 0) {
            const int p1 = ptr1[i], b0 = ptr2[j], b1 = ptr2[j + 1];
            for (int k = 0; k < c && off + k < a.cap1; ++k) { qidx[off + k] = feat1[p1 + k]; qb0[off + k] = b0; qb1[off + k] = b1; }
        }
        base += total;
    }
    if (threadIdx.x == 0) a.nq[b] = min(base, a.cap1);
}

__device__ void three_maxima(const int* hist, int& ind1, int& ind2, int& ind3) {  // ORBmatcher.cpp:64-105
    int max1 = 0, max2 = 0, max3 = 0;
    ind1 = ind2 = ind3 = -1;
    for (int i = 0; i < HISTO_LENGTH; i++) {
        const int s = hist[i];
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if (max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if (max3 < 0.1f * (float)max1) { ind3 = -1; }
}

__device__ __forceinline__ int rot_bin(float a1, float a2) {
    const float factor = (float)HISTO_LENGTH / 360.0f;
    float rot = __fsub_rn(a1, a2);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.f);
    int bin = (int)roundf(__fmul_rn(rot, factor));
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

struct ResolveArgs {
    int nq_cap; const int* d_nq;      // queries (frame-1 keypoints / map points / KF1 features in walk order)
    int n2_cap; const int* d_n2;      // database items
    int cap; const int2* cand; const int* ncand;
    float nnratio;
    int K;                            // claim slots per database item in shared memory
    // rotation histogram inputs (angle of query q at ang1[qid(q) * stride1], of database item j at ang2[j * stride2])
    const float* ang1; int stride1; const float* ang2; int stride2; int check_ori;
    const int* qid;                   // BOW: feature index of query q (pair stride qstride); null: q
    int qstride;
    const int* slot2;                 // BOW batch: pair b's database is slot2[b] of the side-2 arrays; null: b
    const se2gpu_keypoint* kp2;       // WINDOW: database keypoints (vbPrevMatched update)
    int* out; int n_out;              // WINDOW: matches12[n1]; PROJ: vMatchesIdxMP[n_kf]; BOW: matches12[n1]
    float* prev;                      // WINDOW: vbPrevMatched, updated in place
    int* nmatches; int* flags;
    int scr_q;                        // max_queries: per-pair rows of cand (each `cap` wide) and entries of ncand
};

// pair b's slice: queries and database items are strided by nq_cap / n2_cap (BOW: the angles are per feature and nq_cap
// is KF1's feature capacity), outputs by n_out, the context scratch by its capacities; work is the fallback's
// [2 * cap + scr_q] per pair
__device__ __forceinline__ void pair_slice(ResolveArgs& a, int b) {
    const size_t q = (size_t)b * a.nq_cap, d = (size_t)side2_slot(a.slot2, b) * a.n2_cap;
    if (a.qid) a.qid += (size_t)b * a.qstride;
    if (a.d_nq) a.d_nq += b;
    if (a.d_n2) a.d_n2 += b;
    a.cand += (size_t)b * a.scr_q * a.cap; a.ncand += (size_t)b * a.scr_q;
    if (a.ang1) { a.ang1 += q * a.stride1; a.ang2 += d * a.stride2; }
    if (a.kp2) a.kp2 += d;
    if (a.prev) a.prev += 2 * q;
    a.out += (size_t)b * a.n_out; a.nmatches += b; a.flags += 2 * b;
}
__device__ __forceinline__ int* work_slice(const ResolveArgs& a, int* work, int b) { return work + (size_t)b * (2 * (size_t)a.cap + a.scr_q); }

// Greedy resolution as speculative rounds, one CTA per pair (see the file header). Per-query decision = (chosen database item or
// -1, its distance). Claim table: for every database item the (query, distance) pairs of the queries that currently
// choose it; a query evaluates a candidate j against min{distance of claims by EARLIER queries} == vMatchesDistance[j]
// at its turn of the sequential loop (the distance of successive claims on one item is strictly decreasing), in BOW
// mode against "claimed by an earlier query at all" == vbMatched2[j].
template <int MODE>
__global__ void __launch_bounds__(1024) k_resolve(ResolveArgs a) {
    extern __shared__ int smi[];
    __shared__ int hist[HISTO_LENGTH];
    __shared__ int s_over, s_nm, s_top[3];
    // pair 0 needs no offsets; skipping them keeps a single pair's prologue as short as it was (one CTA on one SM runs the
    // whole resolve, so every per-thread instruction before the rounds is on the critical path)
    if (blockIdx.x != 0 || (MODE == MODE_BOW && a.slot2)) pair_slice(a, blockIdx.x);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int nq = count_of(a.d_nq, a.nq_cap), n2 = count_of(a.d_n2, a.n2_cap);
    const int K = a.K;
    int* cnt = smi;                                   // [n2_cap]
    int* lastc = cnt + a.n2_cap;                      // [n2_cap]
    unsigned* slot = reinterpret_cast<unsigned*>(lastc + a.n2_cap);   // [n2_cap][K]: query << 16 | distance
    int* ch = reinterpret_cast<int*>(slot + (size_t)a.n2_cap * K);   // [nq_cap] chosen item or -1
    int* cd = ch + a.nq_cap;                          // [nq_cap] its distance (later: its rotation bin)
    for (int q = tid; q < nq; q += nt) { ch[q] = -1; cd[q] = 0; }
    if (tid == 0) { s_over = 0; s_nm = 0; }
    if (tid < HISTO_LENGTH) hist[tid] = 0;
    __syncthreads();
    int rounds = 0;
    while (true) {
        for (int j = tid; j < n2; j += nt) cnt[j] = 0;
        __syncthreads();
        for (int q = tid; q < nq; q += nt) {
            const int j = ch[q];
            if (j >= 0) {
                const int pos = atomicAdd(&cnt[j], 1);
                if (pos < K) slot[(size_t)j * K + pos] = ((unsigned)q << 16) | (unsigned)cd[q];
                else s_over = 1;
            }
        }
        __syncthreads();
        if (s_over) break;
        int changed = 0;
        for (int q = tid; q < nq; q += nt) {
            const int nc = a.ncand[q];
            int best = INT_MAX, best2 = INT_MAX, bj = -1, lvl = -1, lvl2 = -1;
            const int2* cq = a.cand + (size_t)q * a.cap;
            for (int k = 0; k < nc; ++k) {
                const int2 c = cq[k];
                const int j = c.x, dist = c.y & 0xffff;
                const int cn = cnt[j];
                bool skip = false;
                for (int u = 0; u < cn; ++u) {
                    const unsigned e = slot[(size_t)j * K + u];
                    if ((int)(e >> 16) < q) skip = skip || (MODE == MODE_BOW) || ((int)(e & 0xffffu) <= dist);
                }
                if (skip) continue;
                if (dist < best) { best2 = best; lvl2 = lvl; best = dist; lvl = c.y >> 16; bj = j; }
                else if (dist < best2) { best2 = dist; lvl2 = c.y >> 16; }
            }
            bool acc;
            if (MODE == MODE_WINDOW) acc = best <= TH_LOW && (float)best < (float)best2 * a.nnratio;            // :329-330
            else if (MODE == MODE_PROJ) acc = best <= TH_HIGH && !(lvl == lvl2 && (float)best > a.nnratio * (float)best2);   // :435-437
            else acc = best < TH_LOW && (float)best < a.nnratio * (float)best2;                                   // :206-208
            const int nj = acc ? bj : -1, nd = acc ? best : 0;
            if (nj != ch[q] || nd != cd[q]) { ch[q] = nj; cd[q] = nd; changed = 1; }
        }
        ++rounds;
        if (!__syncthreads_or(changed)) break;
    }
    if (s_over) {                       // claim table too small for this input: the sequential kernel takes over
        if (tid == 0) { a.flags[0] = 1; a.flags[1] = rounds; }
        return;
    }
    // ---- epilogue: last claimant of every item keeps it (every later claim steals, :331-334 / :438-441), histogram, output
    for (int j = tid; j < n2; j += nt) lastc[j] = -1;
    if (MODE == MODE_BOW) for (int i = tid; i < a.n_out; i += nt) a.out[i] = -1;
    __syncthreads();
    const bool use_hist = MODE == MODE_WINDOW || (MODE == MODE_BOW && a.check_ori);
    for (int q = tid; q < nq; q += nt) {
        const int j = ch[q];
        if (j < 0) continue;
        atomicMax(&lastc[j], q);
        if (use_hist) {
            const int id = a.qid ? a.qid[q] : q;
            const int bin = rot_bin(a.ang1[(size_t)id * a.stride1], a.ang2[(size_t)j * a.stride2]);
            cd[q] = bin;
            atomicAdd(&hist[bin], 1);
        }
    }
    __syncthreads();
    if (tid == 0) {
        int i1 = -1, i2 = -1, i3 = -1;
        if (use_hist) three_maxima(hist, i1, i2, i3);
        s_top[0] = i1; s_top[1] = i2; s_top[2] = i3;
    }
    __syncthreads();
    int mine = 0;
    if (MODE == MODE_PROJ) {
        for (int j = tid; j < a.n_out; j += nt) { const int m = j < n2 ? lastc[j] : -1; a.out[j] = m; mine += m >= 0; }
    } else {
        const int lim = MODE == MODE_WINDOW ? a.n_out : nq;
        for (int q = tid; q < lim; q += nt) {
            int m = -1;
            if (q < nq && ch[q] >= 0 && lastc[ch[q]] == q) {
                m = ch[q];
                if (use_hist) { const int b = cd[q]; if (b != s_top[0] && b != s_top[1] && b != s_top[2]) m = -1; }
            }
            if (MODE == MODE_WINDOW) {
                a.out[q] = m;
                if (m >= 0) { a.prev[2 * q] = a.kp2[m].x; a.prev[2 * q + 1] = a.kp2[m].y; }       // :375-377
            } else if (m >= 0) {
                a.out[a.qid[q]] = m;
            }
            mine += m >= 0;
        }
    }
    if (mine) atomicAdd(&s_nm, mine);
    __syncthreads();
    if (tid == 0) { *a.nmatches = s_nm; a.flags[1] = rounds; }
}

struct Top2 { int d1, p1, d2, p2; };  // two smallest (dist, position) pairs, lexicographic
__device__ __forceinline__ void top2_push(Top2& t, int dist, int pos) {
    if (dist < t.d1 || (dist == t.d1 && pos < t.p1)) { t.d2 = t.d1; t.p2 = t.p1; t.d1 = dist; t.p1 = pos; }
    else if (dist < t.d2 || (dist == t.d2 && pos < t.p2)) { t.d2 = dist; t.p2 = pos; }
}
__device__ __forceinline__ Top2 top2_warp(Top2 t) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Top2 u;
        u.d1 = __shfl_xor_sync(0xffffffffu, t.d1, o); u.p1 = __shfl_xor_sync(0xffffffffu, t.p1, o);
        u.d2 = __shfl_xor_sync(0xffffffffu, t.d2, o); u.p2 = __shfl_xor_sync(0xffffffffu, t.p2, o);
        top2_push(t, u.d1, u.p1);
        top2_push(t, u.d2, u.p2);
    }
    return t;
}

// Exact sequential fallbacks (one warp per pair, queries in order); a warp returns at once unless its pair's flags[0] is set.
// work: [n2] vMatchesDistance, [n2] vnMatches21, [n1] bin_of
__global__ void __launch_bounds__(32) k_fallback_window(ResolveArgs a, const se2gpu_keypoint* __restrict__ kp1, int* __restrict__ work) {
    const int b = blockIdx.x;
    if (a.flags[2 * b] == 0) return;
    pair_slice(a, b);
    kp1 += (size_t)b * a.nq_cap; work = work_slice(a, work, b);
    __shared__ int hist[HISTO_LENGTH];
    const int lane = threadIdx.x;
    const int n1 = count_of(a.d_nq, a.nq_cap), n2 = count_of(a.d_n2, a.n2_cap);
    int* vdist = work; int* m21 = work + a.n2_cap; int* bin_of = work + 2 * a.n2_cap;
    for (int i = lane; i < n2; i += 32) { vdist[i] = INT_MAX; m21[i] = -1; }
    for (int i = lane; i < a.n_out; i += 32) a.out[i] = -1;
    for (int i = lane; i < n1; i += 32) bin_of[i] = -1;
    if (lane < HISTO_LENGTH) hist[lane] = 0;
    __syncwarp();
    int nmatches = 0;
    for (int i1 = 0; i1 < n1; ++i1) {
        const int nc = a.ncand[i1];
        if (nc == 0) continue;
        Top2 t{INT_MAX, INT_MAX, INT_MAX, INT_MAX};
        for (int k = lane; k < nc; k += 32) {
            const int2 c = a.cand[(size_t)i1 * a.cap + k];
            const int dist = c.y & 0xffff;
            if (vdist[c.x] <= dist) continue;
            top2_push(t, dist, k);
        }
        t = top2_warp(t);
        if (t.d1 <= TH_LOW && (float)t.d1 < (float)t.d2 * a.nnratio) {
            const int bestIdx2 = a.cand[(size_t)i1 * a.cap + t.p1].x;
            if (lane == 0) {
                if (m21[bestIdx2] >= 0) { a.out[m21[bestIdx2]] = -1; nmatches--; }
                a.out[i1] = bestIdx2; m21[bestIdx2] = i1; vdist[bestIdx2] = t.d1; nmatches++;
                const int bin = rot_bin(kp1[i1].angle, a.kp2[bestIdx2].angle);
                bin_of[i1] = bin; hist[bin]++;
            }
            __syncwarp();
        }
    }
    __syncwarp();
    if (lane == 0) {
        int i1, i2, i3;
        three_maxima(hist, i1, i2, i3);
        for (int k = 0; k < n1; ++k) {
            const int b = bin_of[k];
            if (b < 0 || b == i1 || b == i2 || b == i3) continue;
            if (a.out[k] >= 0) { a.out[k] = -1; nmatches--; }
        }
        *a.nmatches = nmatches;
    }
    __syncwarp();
    for (int k = lane; k < n1; k += 32)
        if (a.out[k] >= 0) { a.prev[2 * k] = a.kp2[a.out[k]].x; a.prev[2 * k + 1] = a.kp2[a.out[k]].y; }
}

// MatchByProjection's sequential loop (:415-449). work: [n] vMatchesDistance
__global__ void __launch_bounds__(32) k_fallback_projection(ResolveArgs a, int* __restrict__ work) {
    const int b = blockIdx.x;
    if (a.flags[2 * b] == 0) return;
    pair_slice(a, b);
    work = work_slice(a, work, b);
    const int lane = threadIdx.x;
    const int nmp = count_of(a.d_nq, a.nq_cap), n = count_of(a.d_n2, a.n2_cap);
    for (int i = lane; i < n; i += 32) work[i] = INT_MAX;
    for (int i = lane; i < a.n_out; i += 32) a.out[i] = -1;
    __syncwarp();
    int nmatches = 0;
    for (int i = 0; i < nmp; ++i) {
        const int nc = a.ncand[i];
        if (nc == 0) continue;
        Top2 t{INT_MAX, INT_MAX, INT_MAX, INT_MAX};
        for (int k = lane; k < nc; k += 32) {
            const int2 c = a.cand[(size_t)i * a.cap + k];
            const int dist = c.y & 0xffff;
            if (work[c.x] <= dist) continue;
            top2_push(t, dist, k);
        }
        t = top2_warp(t);
        if (t.d1 <= TH_HIGH) {
            const int2 cb = a.cand[(size_t)i * a.cap + t.p1];
            const int bestLevel = cb.y >> 16;
            const int bestLevel2 = (t.d2 == INT_MAX) ? -1 : (a.cand[(size_t)i * a.cap + t.p2].y >> 16);
            if (bestLevel == bestLevel2 && (float)t.d1 > a.nnratio * (float)t.d2) continue;
            if (lane == 0) {
                if (a.out[cb.x] >= 0) { a.out[cb.x] = -1; nmatches--; }
                a.out[cb.x] = i; work[cb.x] = t.d1; nmatches++;
            }
            __syncwarp();
        }
    }
    if (lane == 0) *a.nmatches = nmatches;
}

// SearchByBoW's sequential loop (:166-246) over the precomputed candidate lists. work: [n2] vbMatched2, [nq] bin_of
__global__ void __launch_bounds__(32) k_fallback_bow(ResolveArgs a, int* __restrict__ work) {
    const int b = blockIdx.x;
    if (a.flags[2 * b] == 0) return;
    pair_slice(a, b);
    work = work_slice(a, work, b);
    __shared__ int hist[HISTO_LENGTH];
    const int lane = threadIdx.x;
    const int nq = count_of(a.d_nq, a.nq_cap), n2 = a.n2_cap;
    int* matched2 = work; int* bin_of = work + n2;
    for (int i = lane; i < n2; i += 32) matched2[i] = 0;
    for (int i = lane; i < a.n_out; i += 32) a.out[i] = -1;
    for (int i = lane; i < nq; i += 32) bin_of[i] = -1;
    if (lane < HISTO_LENGTH) hist[lane] = 0;
    __syncwarp();
    int nmatches = 0;
    for (int q = 0; q < nq; ++q) {
        const int nc = a.ncand[q];
        Top2 t{INT_MAX, INT_MAX, INT_MAX, INT_MAX};
        for (int k = lane; k < nc; k += 32) {
            const int2 c = a.cand[(size_t)q * a.cap + k];
            if (matched2[c.x]) continue;
            top2_push(t, c.y & 0xffff, k);
        }
        t = top2_warp(t);
        if (t.d1 < TH_LOW && (float)t.d1 < a.nnratio * (float)t.d2) {
            const int j = a.cand[(size_t)q * a.cap + t.p1].x;
            if (lane == 0) {
                a.out[a.qid[q]] = j; matched2[j] = 1;
                if (a.check_ori) { const int bin = rot_bin(a.ang1[(size_t)a.qid[q] * a.stride1], a.ang2[(size_t)j * a.stride2]); bin_of[q] = bin; hist[bin]++; }
                nmatches++;
            }
            __syncwarp();
        }
    }
    __syncwarp();
    if (lane == 0) {
        if (a.check_ori) {
            int i1, i2, i3;
            three_maxima(hist, i1, i2, i3);
            for (int q = 0; q < nq; ++q) {
                const int bb = bin_of[q];
                if (bb < 0 || bb == i1 || bb == i2 || bb == i3) continue;
                a.out[a.qid[q]] = -1; nmatches--;
            }
        }
        *a.nmatches = nmatches;
    }
}

__global__ void k_kp_to_xy(const se2gpu_keypoint* __restrict__ kp, int n_cap, const int* __restrict__ d_n, float* __restrict__ xy) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count_of(d_n, n_cap)) { xy[2 * i] = kp[i].x; xy[2 * i + 1] = kp[i].y; }
}

// the grids of B databases of n (capacity) keypoints each, pair b's at d_kp + b * n
int launch_grid(se2gpu_matcher* m, int B, const se2gpu_keypoint* d_kp, int n, const int* d_n, se2gpu_grid_params grid, cudaStream_t s) {
    const dim3 blocks((n + 127) / 128, B);
    m->prof.begin(0, s);
    if (n <= GRID_SMEM_KEYS) {
        SE2_LAUNCH(k_grid_build, blocks, 128, 0, s, d_kp, n, d_n, grid, m->cell, m->order, m->nvalid, m->max_db);
    } else {
        SE2_CUDA(cudaMemsetAsync(m->nvalid, 0, sizeof(int) * B, s));
        SE2_LAUNCH(k_grid_cell_big, blocks, 128, 0, s, d_kp, n, d_n, grid, m->cell, m->max_db);
        SE2_LAUNCH(k_grid_order_big, blocks, 128, 0, s, m->cell, n, d_n, m->order, m->nvalid, m->max_db);
    }
    m->prof.end(s);
    return SE2GPU_OK;
}

size_t resolve_smem(int nq, int n2, int K) { return ((size_t)n2 * (2 + K) + 2 * (size_t)nq) * sizeof(int); }

int pick_K(int smem_max, int nq, int n2) {
    for (int K = 16; K >= 2; K -= 2)
        if (resolve_smem(nq, n2, K) <= (size_t)smem_max) return K;
    return 0;
}

// common tail of the device paths for B pairs: resolve + guarded fallback. K depends on the caps only,
// so it is the same for every pair.
template <int MODE>
int launch_resolve(se2gpu_matcher* m, int B, ResolveArgs ra, const se2gpu_keypoint* kp1, cudaStream_t s) {
    const int K = (ra.nq_cap < 65536) ? pick_K(m->resolve_smem_max, ra.nq_cap, ra.n2_cap) : 0;
    ra.scr_q = m->max_q;
    m->last_batch = B;
    SE2_CUDA(cudaMemsetAsync(m->flags, 0, 2 * sizeof(int) * B, s));
    m->prof.begin(2, s);
    if (K >= 2) {
        ra.K = K;
        SE2_LAUNCH(k_resolve<MODE>, B, 1024, resolve_smem(ra.nq_cap, ra.n2_cap, K), s, ra);
    } else {                     // inputs too large for the shared-memory claim table: sequential kernel directly
        SE2_CUDA(cudaMemcpyAsync(m->flags, m->seq_flags.data(), 2 * sizeof(int) * B, cudaMemcpyHostToDevice, s));
    }
    m->prof.end(s);
    m->prof.begin(3, s);
    if (MODE == MODE_WINDOW) SE2_LAUNCH(k_fallback_window, B, 32, 0, s, ra, kp1, m->work);
    else if (MODE == MODE_PROJ) SE2_LAUNCH(k_fallback_projection, B, 32, 0, s, ra, m->work);
    else SE2_LAUNCH(k_fallback_bow, B, 32, 0, s, ra, m->work);
    m->prof.end(s);
    return SE2GPU_OK;
}

std::mutex g_default_mutex;
se2gpu_matcher* g_default[se2gpu::kMaxDevices] = {};

}  // namespace

// the dynamic shared memory k_resolve may use on `device` (what se2gpu_matcher_create_batch opts into)
static int resolve_smem_limit(int device) {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    return optin > 0 ? optin - 2048 : 46 * 1024;
}

bool se2gpu::matcher_window_capturable(int device, int cap1, int cap2) {
    return cap1 < 65536 && pick_K(resolve_smem_limit(device), cap1, cap2) >= 2;
}

extern "C" {

se2gpu_matcher* se2gpu_matcher_create(int max_queries, int max_db, int device) {
    return se2gpu_matcher_create_batch(max_queries, max_db, 1, device);
}

se2gpu_matcher* se2gpu_matcher_create_batch(int max_queries, int max_db, int max_batch, int device) {
    if (max_queries <= 0 || max_db <= 0 || max_batch <= 0) { fail(SE2GPU_ERR_INVALID, "bad capacities"); return nullptr; }
    if (max_batch > 65535) { fail(SE2GPU_ERR_CAPACITY, "%d pairs per call: at most 65535 (the grid's y dimension)", max_batch); return nullptr; }
    if ((size_t)max_queries * max_db * sizeof(int2) > (((size_t)4 << 30) / max_batch)) {
        fail(SE2GPU_ERR_CAPACITY, "candidate table %d x %d x %d too large", max_batch, max_queries, max_db);
        return nullptr;
    }
    if (se2gpu::select_device(device) != SE2GPU_OK) return nullptr;
    se2gpu_matcher* m = new se2gpu_matcher;
    m->device = device; m->max_q = max_queries; m->max_db = max_db; m->max_batch = max_batch;
    m->seq_flags.assign(2 * (size_t)max_batch, 0);
    for (int b = 0; b < max_batch; ++b) m->seq_flags[2 * b] = 1;
    const size_t Q = max_queries, D = max_db, N = std::max(Q, D), P = max_batch;
    bool ok = true;
    auto A = [&](auto** p, size_t count) { ok = ok && m->bufs.alloc(p, count) == cudaSuccess; };
    A(&m->cell, P * D); A(&m->order, P * D); A(&m->nvalid, P);
    A(&m->cand, P * Q * D); A(&m->ncand, P * Q); A(&m->work, P * (2 * D + Q)); A(&m->flags, 2 * P); A(&m->nm, P);
    A(&m->bow_q, P * 3 * Q); A(&m->bow_nq, P);
    A(&m->d_kp1, N); A(&m->d_kp2, N); A(&m->d_desc1, N * 32); A(&m->d_desc2, N * 32);
    A(&m->d_u8a, N); A(&m->d_u8b, N); A(&m->d_f1, 2 * N); A(&m->d_f2, 2 * N);
    A(&m->d_i1, N + 1); A(&m->d_i2, N + 1); A(&m->d_i3, N + 1); A(&m->d_i4, N + 1); A(&m->d_out, N);
    // pinned staging: both keypoint sets + descriptors + per-item side arrays + outputs
    m->pin_bytes = N * (2 * (sizeof(se2gpu_keypoint) + 32) + 2 + 16 + 5 * sizeof(int) + 8) + 4096;
    ok = ok && m->pin.reserve(m->pin_bytes);
    ok = ok && cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) == cudaSuccess;
    if (ok) {
        m->resolve_smem_max = resolve_smem_limit(device);
        ok = cudaFuncSetAttribute(k_resolve<MODE_WINDOW>, cudaFuncAttributeMaxDynamicSharedMemorySize, m->resolve_smem_max) == cudaSuccess &&
             cudaFuncSetAttribute(k_resolve<MODE_PROJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, m->resolve_smem_max) == cudaSuccess &&
             cudaFuncSetAttribute(k_resolve<MODE_BOW>, cudaFuncAttributeMaxDynamicSharedMemorySize, m->resolve_smem_max) == cudaSuccess;
    }
    if (!ok) { fail(SE2GPU_ERR_CUDA, "matcher allocation failed: %s", cudaGetErrorString(cudaGetLastError())); se2gpu_matcher_destroy(m); return nullptr; }
    return m;
}

void se2gpu_matcher_destroy(se2gpu_matcher* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m;
}

int se2gpu_matcher_profile(se2gpu_matcher* m, int enable) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(m->device));
    m->prof.enable(enable != 0);
    return SE2GPU_OK;
}

int se2gpu_matcher_profile_read(se2gpu_matcher* m, double* ms, int* launches) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(m->device));
    m->prof.flush();
    for (int g = 0; g < SE2GPU_MATCHER_PROFILE_GROUPS; ++g) { if (ms) ms[g] = m->prof.ms[g]; if (launches) launches[g] = m->prof.launches[g]; }
    return SE2GPU_OK;
}

int se2gpu_matcher_last_rounds(se2gpu_matcher* m, int* rounds, int* used_fallback) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(m->device));
    int f[2] = {0, 0};
    SE2_CUDA(cudaMemcpy(f, m->flags, sizeof f, cudaMemcpyDeviceToHost));
    if (used_fallback) *used_fallback = f[0];
    if (rounds) *rounds = f[1];
    return SE2GPU_OK;
}

int se2gpu_matcher_last_rounds_batch(se2gpu_matcher* m, int B, int* rounds, int* used_fallback) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (B < 0 || B > m->last_batch) return fail(SE2GPU_ERR_INVALID, "%d pairs asked for, the last resolve had %d", B, m->last_batch);
    if (B == 0) return SE2GPU_OK;
    SE2_CUDA(cudaSetDevice(m->device));
    std::vector<int> f(2 * (size_t)B);
    SE2_CUDA(cudaMemcpy(f.data(), m->flags, sizeof(int) * f.size(), cudaMemcpyDeviceToHost));
    for (int b = 0; b < B; ++b) {
        if (used_fallback) used_fallback[b] = f[2 * b];
        if (rounds) rounds[b] = f[2 * b + 1];
    }
    return SE2GPU_OK;
}

int se2gpu_keypoints_to_points_device(const se2gpu_keypoint* d_kp, int n, const int* d_n, float* d_xy, void* stream) {
    if (n < 0 || (n && (!d_kp || !d_xy))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = se2gpu::require_device(); if (rc) return rc; }
    if (n == 0) return SE2GPU_OK;
    SE2_LAUNCH(k_kp_to_xy, (n + 255) / 256, 256, 0, (cudaStream_t)stream, d_kp, n, d_n, d_xy);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_match_by_window_device(se2gpu_matcher* m, const se2gpu_keypoint* d_kp1, const uint8_t* d_desc1, int n1, const int* d_n1,
                                  const se2gpu_keypoint* d_kp2, const uint8_t* d_desc2, int n2, const int* d_n2, float* d_prev,
                                  se2gpu_grid_params grid, int win_size, int level_offset, int min_level, int max_level, float nnratio,
                                  int* d_matches12, int* d_nmatches, void* stream) {
    return se2gpu_match_by_window_batch_device(m, 1, d_kp1, d_desc1, n1, d_n1, d_kp2, d_desc2, n2, d_n2, d_prev, grid, win_size, level_offset,
                                               min_level, max_level, nnratio, d_matches12, d_nmatches, stream);
}

int se2gpu_match_by_window_batch_device(se2gpu_matcher* m, int B, const se2gpu_keypoint* d_kp1, const uint8_t* d_desc1, int cap1,
                                        const int* d_n1, const se2gpu_keypoint* d_kp2, const uint8_t* d_desc2, int cap2, const int* d_n2,
                                        float* d_prev, se2gpu_grid_params grid, int win_size, int level_offset, int min_level,
                                        int max_level, float nnratio, int* d_matches12, int* d_nmatches, void* stream) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (B < 0 || cap1 < 0 || cap2 < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (B > m->max_batch || cap1 > m->max_q || cap2 > m->max_db)
        return fail(SE2GPU_ERR_CAPACITY, "%d pairs of %d x %d exceed the matcher's capacity %d pairs of %d x %d", B, cap1, cap2, m->max_batch, m->max_q, m->max_db);
    SE2_NVTX("se2gpu.match_by_window");
    if (B == 0) return SE2GPU_OK;
    if (cap1 && (!d_kp1 || !d_desc1 || !d_prev || !d_matches12)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (cap2 && (!d_kp2 || !d_desc2)) return fail(SE2GPU_ERR_INVALID, "null argument");
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)stream;
    int* nm = d_nmatches ? d_nmatches : m->nm;
    if (cap1 == 0 || cap2 == 0) {
        if (cap1) SE2_CUDA(cudaMemsetAsync(d_matches12, 0xff, sizeof(int) * cap1 * B, s));
        SE2_CUDA(cudaMemsetAsync(nm, 0, sizeof(int) * B, s));
        return SE2GPU_OK;
    }
    { const int rc = launch_grid(m, B, d_kp2, cap2, d_n2, grid, s); if (rc != SE2GPU_OK) return rc; }
    CandArgs ca{};
    ca.mode = MODE_WINDOW; ca.nq_cap = cap1; ca.d_nq = d_n1; ca.kp1 = d_kp1; ca.prev = d_prev; ca.min_level = min_level; ca.max_level = max_level;
    ca.level_offset = level_offset; ca.win_size = win_size; ca.qdesc = reinterpret_cast<const uint32_t*>(d_desc1);
    ca.kp = d_kp2; ca.desc = reinterpret_cast<const uint32_t*>(d_desc2); ca.cell = m->cell; ca.order = m->order; ca.n_valid = m->nvalid; ca.db_skip = nullptr;
    ca.db_cap = cap2; ca.g = grid; ca.cap = m->max_db; ca.cand = m->cand; ca.ncand = m->ncand; ca.scr_q = m->max_q;
    m->prof.begin(1, s);
    SE2_LAUNCH(k_candidates, dim3((cap1 * 32 + 255) / 256, B), 256, 0, s, ca);
    m->prof.end(s);
    ResolveArgs ra{};
    ra.nq_cap = cap1; ra.d_nq = d_n1; ra.n2_cap = cap2; ra.d_n2 = d_n2; ra.cap = m->max_db; ra.cand = m->cand; ra.ncand = m->ncand; ra.nnratio = nnratio;
    ra.ang1 = &d_kp1->angle; ra.stride1 = sizeof(se2gpu_keypoint) / 4; ra.ang2 = &d_kp2->angle; ra.stride2 = sizeof(se2gpu_keypoint) / 4; ra.check_ori = 1;
    ra.qid = nullptr; ra.kp2 = d_kp2; ra.out = d_matches12; ra.n_out = cap1; ra.prev = d_prev; ra.nmatches = nm; ra.flags = m->flags;
    return launch_resolve<MODE_WINDOW>(m, B, ra, d_kp1, s);
}

int se2gpu_match_by_projection_device(se2gpu_matcher* m, const se2gpu_keypoint* d_kf_kp, const uint8_t* d_kf_desc, int n_kf, const int* d_n_kf,
                                      const uint8_t* d_kf_observed, const uint8_t* d_mp_valid, const float* d_mp_uv, int n_mp,
                                      const int* d_mp_octave, const uint8_t* d_mp_desc, se2gpu_grid_params grid, int win_size,
                                      int level_offset, float nnratio, int* d_matches_idx_mp, int* d_nmatches, void* stream) {
    return se2gpu_match_by_projection_batch_device(m, 1, d_kf_kp, d_kf_desc, n_kf, d_n_kf, d_kf_observed, d_mp_valid, d_mp_uv, n_mp, d_mp_octave,
                                                   d_mp_desc, grid, win_size, level_offset, nnratio, d_matches_idx_mp, d_nmatches, stream);
}

int se2gpu_match_by_projection_batch_device(se2gpu_matcher* m, int B, const se2gpu_keypoint* d_kf_kp, const uint8_t* d_kf_desc, int cap_kf,
                                            const int* d_n_kf, const uint8_t* d_kf_observed, const uint8_t* d_mp_valid, const float* d_mp_uv,
                                            int cap_mp, const int* d_mp_octave, const uint8_t* d_mp_desc, se2gpu_grid_params grid,
                                            int win_size, int level_offset, float nnratio, int* d_matches_idx_mp, int* d_nmatches,
                                            void* stream) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (B < 0 || cap_kf < 0 || cap_mp < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (B > m->max_batch || cap_mp > m->max_q || cap_kf > m->max_db)
        return fail(SE2GPU_ERR_CAPACITY, "%d pairs of %d x %d exceed the matcher's capacity %d pairs of %d x %d", B, cap_mp, cap_kf, m->max_batch, m->max_q, m->max_db);
    SE2_NVTX("se2gpu.match_by_projection");
    if (B == 0) return SE2GPU_OK;
    if (cap_kf && (!d_kf_kp || !d_kf_desc || !d_kf_observed || !d_matches_idx_mp)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (cap_mp && (!d_mp_valid || !d_mp_uv || !d_mp_octave || !d_mp_desc)) return fail(SE2GPU_ERR_INVALID, "null argument");
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)stream;
    int* nm = d_nmatches ? d_nmatches : m->nm;
    if (cap_kf == 0 || cap_mp == 0) {
        if (cap_kf) SE2_CUDA(cudaMemsetAsync(d_matches_idx_mp, 0xff, sizeof(int) * cap_kf * B, s));
        SE2_CUDA(cudaMemsetAsync(nm, 0, sizeof(int) * B, s));
        return SE2GPU_OK;
    }
    { const int rc = launch_grid(m, B, d_kf_kp, cap_kf, d_n_kf, grid, s); if (rc != SE2GPU_OK) return rc; }
    CandArgs ca{};
    ca.mode = MODE_PROJ; ca.nq_cap = cap_mp; ca.d_nq = nullptr; ca.mp_valid = d_mp_valid; ca.mp_uv = d_mp_uv; ca.mp_octave = d_mp_octave;
    ca.level_offset = level_offset; ca.win_size = win_size; ca.qdesc = reinterpret_cast<const uint32_t*>(d_mp_desc);
    ca.kp = d_kf_kp; ca.desc = reinterpret_cast<const uint32_t*>(d_kf_desc); ca.cell = m->cell; ca.order = m->order; ca.n_valid = m->nvalid; ca.db_skip = d_kf_observed;
    ca.db_cap = cap_kf; ca.g = grid; ca.cap = m->max_db; ca.cand = m->cand; ca.ncand = m->ncand; ca.scr_q = m->max_q;
    m->prof.begin(1, s);
    SE2_LAUNCH(k_candidates, dim3((cap_mp * 32 + 255) / 256, B), 256, 0, s, ca);
    m->prof.end(s);
    ResolveArgs ra{};
    ra.nq_cap = cap_mp; ra.d_nq = nullptr; ra.n2_cap = cap_kf; ra.d_n2 = d_n_kf; ra.cap = m->max_db; ra.cand = m->cand; ra.ncand = m->ncand; ra.nnratio = nnratio;
    ra.check_ori = 0; ra.out = d_matches_idx_mp; ra.n_out = cap_kf; ra.nmatches = nm; ra.flags = m->flags;
    return launch_resolve<MODE_PROJ>(m, B, ra, nullptr, s);
}

int se2gpu_search_by_bow_batch_device(se2gpu_matcher* m, int B, const se2gpu_bow_batch_kf* kf1, const se2gpu_bow_batch_kf* kf2,
                                      const int* d_slot2, int mp_only, float nnratio, int check_orientation, int* d_matches12,
                                      int* d_nmatches, void* stream) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (!kf1 || !kf2) return fail(SE2GPU_ERR_INVALID, "null keyframe side");
    const int cap1 = kf1->cap, cap2 = kf2->cap;
    if (B < 0 || cap1 < 0 || cap2 < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (B > m->max_batch || cap1 > m->max_q || cap2 > m->max_db)
        return fail(SE2GPU_ERR_CAPACITY, "%d pairs of %d x %d exceed the matcher's capacity %d pairs of %d x %d", B, cap1, cap2, m->max_batch, m->max_q, m->max_db);
    SE2_NVTX("se2gpu.search_by_bow_batch");
    if (B == 0) return SE2GPU_OK;
    auto missing = [&](const se2gpu_bow_batch_kf* k) {
        return !k->kp || !k->desc || (mp_only && !k->has_mp) || !k->node || !k->ptr || !k->feat || !k->n_node;
    };
    if ((cap1 && (missing(kf1) || !d_matches12)) || (cap2 && missing(kf2))) return fail(SE2GPU_ERR_INVALID, "null argument");
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)stream;
    int* nm = d_nmatches ? d_nmatches : m->nm;
    if (cap1 == 0 || cap2 == 0) {
        if (cap1) SE2_CUDA(cudaMemsetAsync(d_matches12, 0xff, sizeof(int) * cap1 * B, s));
        SE2_CUDA(cudaMemsetAsync(nm, 0, sizeof(int) * B, s));
        return SE2GPU_OK;
    }
    // pair b's queries at b * 3 max_q of bow_q: features, then the starts and ends of their KF2 ranges
    const int qstride = 3 * m->max_q;
    int *qidx = m->bow_q, *qb0 = qidx + m->max_q, *qb1 = qidx + 2 * m->max_q;
    BowWalkArgs wa{kf1->node, kf1->ptr, kf1->feat, kf1->n_node, cap1, kf2->node, kf2->ptr, kf2->n_node, cap2, d_slot2,
                   qidx, qb0, qb1, qstride, m->bow_nq};
    BowCandArgs ca{};
    ca.nq_cap = cap1; ca.d_nq = m->bow_nq; ca.qidx = qidx; ca.qb0 = qb0; ca.qb1 = qb1; ca.qstride = qstride;
    ca.d1 = reinterpret_cast<const uint32_t*>(kf1->desc); ca.mp1 = kf1->has_mp; ca.cap1 = cap1;
    ca.feat2 = kf2->feat; ca.d2 = reinterpret_cast<const uint32_t*>(kf2->desc); ca.mp2 = kf2->has_mp; ca.cap2 = cap2; ca.slot2 = d_slot2;
    ca.mp_only = mp_only; ca.cap = m->max_db; ca.cand = m->cand; ca.ncand = m->ncand; ca.scr_q = m->max_q;
    m->prof.begin(1, s);
    SE2_LAUNCH(k_bow_walk, B, 256, 0, s, wa);
    SE2_LAUNCH(k_candidates_bow, dim3((cap1 * 32 + 255) / 256, B), 256, 0, s, ca);
    m->prof.end(s);
    ResolveArgs ra{};
    ra.nq_cap = cap1; ra.d_nq = m->bow_nq; ra.n2_cap = cap2; ra.d_n2 = nullptr; ra.cap = m->max_db; ra.cand = m->cand; ra.ncand = m->ncand;
    ra.nnratio = nnratio; ra.ang1 = &kf1->kp->angle; ra.stride1 = sizeof(se2gpu_keypoint) / 4; ra.ang2 = &kf2->kp->angle;
    ra.stride2 = sizeof(se2gpu_keypoint) / 4; ra.check_ori = check_orientation; ra.qid = qidx; ra.qstride = qstride; ra.slot2 = d_slot2;
    ra.out = d_matches12; ra.n_out = cap1; ra.nmatches = nm; ra.flags = m->flags;
    return launch_resolve<MODE_BOW>(m, B, ra, nullptr, s);
}

}  // extern "C"

namespace {

se2gpu_matcher* default_matcher(int device, int nq, int ndb) {
    if (device < 0 || device >= se2gpu::kMaxDevices) { fail(SE2GPU_ERR_INVALID, "device %d out of range", device); return nullptr; }
    se2gpu_matcher*& m = g_default[device];
    if (m && (m->max_q < nq || m->max_db < ndb)) { se2gpu_matcher_destroy(m); m = nullptr; }
    if (!m) m = se2gpu_matcher_create(std::max(nq, 2048), std::max(ndb, 2048), device);
    return m;
}

}  // namespace

extern "C" {

int se2gpu_hamming_distance(const uint8_t* a, const uint8_t* b, int n, int* out, int device) {
    if (n < 0 || (n && (!a || !b || !out))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (n == 0) return SE2GPU_OK;
    const uint32_t* da = st.upload(reinterpret_cast<const uint32_t*>(a), (size_t)n * 8);
    const uint32_t* db = st.upload(reinterpret_cast<const uint32_t*>(b), (size_t)n * 8);
    int* dout = st.output(out, n);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_hamming_pairs, (n + 255) / 256, 256, 0, nullptr, da, db, n, dout);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

int se2gpu_matcher_match_by_window(se2gpu_matcher* m, const se2gpu_keypoint* kp1, const uint8_t* desc1, int n1, const se2gpu_keypoint* kp2,
                                   const uint8_t* desc2, int n2, float* prev, se2gpu_grid_params grid, int win_size, int level_offset,
                                   int min_level, int max_level, float nnratio, int* matches12) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (n1 < 0 || n2 < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (n1 && (!kp1 || !desc1 || !prev || !matches12)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (n2 && (!kp2 || !desc2)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (n1 == 0) return 0;
    if (n2 == 0) { for (int i = 0; i < n1; ++i) matches12[i] = -1; return 0; }
    if (n1 > m->max_q || n2 > m->max_db) return fail(SE2GPU_ERR_CAPACITY, "%d x %d exceeds the matcher's capacity %d x %d", n1, n2, m->max_q, m->max_db);
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = m->stream;
    se2gpu::PinnedArena& st = m->pin;
    st.reserve(m->pin_bytes);
    if (st.up(m->d_kp1, kp1, n1, s) || st.up(m->d_kp2, kp2, n2, s) || st.up(m->d_desc1, desc1, (size_t)n1 * 32, s) ||
        st.up(m->d_desc2, desc2, (size_t)n2 * 32, s) || st.up(m->d_f1, prev, (size_t)2 * n1, s))
        return SE2GPU_ERR_CUDA;
    int rc = se2gpu_match_by_window_device(m, m->d_kp1, m->d_desc1, n1, nullptr, m->d_kp2, m->d_desc2, n2, nullptr, m->d_f1, grid, win_size,
                                           level_offset, min_level, max_level, nnratio, m->d_out, m->nm, s);
    if (rc != SE2GPU_OK) return rc;
    int* h_m = st.alloc<int>(n1); float* h_prev = st.alloc<float>((size_t)2 * n1); int* h_nm = st.alloc<int>(1);
    if (!h_m || !h_prev || !h_nm) return fail(SE2GPU_ERR_CAPACITY, "staging exhausted");
    SE2_CUDA(cudaMemcpyAsync(h_m, m->d_out, sizeof(int) * n1, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaMemcpyAsync(h_prev, m->d_f1, sizeof(float) * 2 * n1, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaMemcpyAsync(h_nm, m->nm, sizeof(int), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    memcpy(matches12, h_m, sizeof(int) * n1); memcpy(prev, h_prev, sizeof(float) * 2 * n1);
    return *h_nm;
}

int se2gpu_matcher_match_by_projection(se2gpu_matcher* m, const se2gpu_keypoint* kf_kp, const uint8_t* kf_desc, int n_kf,
                                       const uint8_t* kf_observed, const uint8_t* mp_valid, const float* mp_uv, int n_mp,
                                       const int* mp_octave, const uint8_t* mp_desc, se2gpu_grid_params grid, int win_size,
                                       int level_offset, float nnratio, int* matches_idx_mp) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (n_kf < 0 || n_mp < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    if (n_kf && (!kf_kp || !kf_desc || !kf_observed || !matches_idx_mp)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (n_mp && (!mp_valid || !mp_uv || !mp_octave || !mp_desc)) return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int i = 0; i < n_kf; ++i) matches_idx_mp[i] = -1;
    if (n_kf == 0 || n_mp == 0) return 0;
    if (n_mp > m->max_q || n_kf > m->max_db) return fail(SE2GPU_ERR_CAPACITY, "%d x %d exceeds the matcher's capacity %d x %d", n_mp, n_kf, m->max_q, m->max_db);
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = m->stream;
    se2gpu::PinnedArena& st = m->pin;
    st.reserve(m->pin_bytes);
    if (st.up(m->d_kp2, kf_kp, n_kf, s) || st.up(m->d_desc2, kf_desc, (size_t)n_kf * 32, s) || st.up(m->d_desc1, mp_desc, (size_t)n_mp * 32, s) ||
        st.up(m->d_u8a, kf_observed, n_kf, s) || st.up(m->d_u8b, mp_valid, n_mp, s) || st.up(m->d_f1, mp_uv, (size_t)2 * n_mp, s) ||
        st.up(m->d_i1, mp_octave, n_mp, s))
        return SE2GPU_ERR_CUDA;
    int rc = se2gpu_match_by_projection_device(m, m->d_kp2, m->d_desc2, n_kf, nullptr, m->d_u8a, m->d_u8b, m->d_f1, n_mp, m->d_i1, m->d_desc1, grid,
                                               win_size, level_offset, nnratio, m->d_out, m->nm, s);
    if (rc != SE2GPU_OK) return rc;
    int* h_m = st.alloc<int>(n_kf); int* h_nm = st.alloc<int>(1);
    if (!h_m || !h_nm) return fail(SE2GPU_ERR_CAPACITY, "staging exhausted");
    SE2_CUDA(cudaMemcpyAsync(h_m, m->d_out, sizeof(int) * n_kf, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaMemcpyAsync(h_nm, m->nm, sizeof(int), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    memcpy(matches_idx_mp, h_m, sizeof(int) * n_kf);
    return *h_nm;
}

int se2gpu_matcher_search_by_bow(se2gpu_matcher* m, const se2gpu_bow_kf* k1, const se2gpu_bow_kf* k2, int mp_only, float nnratio,
                                 int check_orientation, int* matches12) {
    if (!m) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (!k1 || !k2 || k1->n < 0 || k2->n < 0 || (k1->n && !matches12)) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    for (int i = 0; i < k1->n; ++i) matches12[i] = -1;
    if (k1->n == 0 || k2->n == 0 || k1->n_node == 0 || k2->n_node == 0) return 0;
    SE2_NVTX("se2gpu.search_by_bow");
    // the two-iterator walk over the ascending node ids (:160-247) visits the common nodes; the queries are KF1's
    // features of those nodes in walk order, each with the feature range of the same node in KF2
    std::vector<int> qidx, qb0, qb1;
    int maxlist = 0;
    for (int a = 0, b = 0; a < k1->n_node && b < k2->n_node;) {
        const int na = k1->node[a], nb = k2->node[b];
        if (na == nb) {
            for (int i = k1->ptr[a]; i < k1->ptr[a + 1]; ++i) { qidx.push_back(k1->feat[i]); qb0.push_back(k2->ptr[b]); qb1.push_back(k2->ptr[b + 1]); }
            maxlist = std::max(maxlist, k2->ptr[b + 1] - k2->ptr[b]);
            ++a; ++b;
        } else if (na < nb) ++a;
        else ++b;
    }
    const int nq = (int)qidx.size(), nf2 = k2->ptr[k2->n_node];
    if (nq == 0) return 0;
    for (int i = 0; i < nq; ++i) if (qidx[i] < 0 || qidx[i] >= k1->n) return fail(SE2GPU_ERR_INVALID, "feature index out of range");
    if (nq > m->max_q || k1->n > m->max_q || k2->n > m->max_db || nf2 > m->max_db || maxlist > m->max_db)
        return fail(SE2GPU_ERR_CAPACITY, "BoW problem (%d queries, %d x %d features) exceeds the matcher's capacity %d x %d", nq, k1->n, k2->n, m->max_q, m->max_db);
    SE2_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = m->stream;
    se2gpu::PinnedArena& st = m->pin;
    st.reserve(m->pin_bytes);
    if (st.up(m->d_desc1, k1->desc, (size_t)k1->n * 32, s) || st.up(m->d_desc2, k2->desc, (size_t)k2->n * 32, s) ||
        st.up(m->d_u8a, k1->has_mp, k1->n, s) || st.up(m->d_u8b, k2->has_mp, k2->n, s) || st.up(m->d_f1, k1->angle, k1->n, s) ||
        st.up(m->d_f2, k2->angle, k2->n, s) || st.up(m->d_i1, qidx.data(), nq, s) || st.up(m->d_i2, qb0.data(), nq, s) ||
        st.up(m->d_i3, qb1.data(), nq, s) || st.up(m->d_i4, k2->feat, nf2, s))
        return SE2GPU_ERR_CUDA;
    BowCandArgs ca{};
    ca.nq_cap = nq; ca.d_nq = nullptr; ca.qidx = m->d_i1; ca.qb0 = m->d_i2; ca.qb1 = m->d_i3;
    ca.d1 = reinterpret_cast<const uint32_t*>(m->d_desc1); ca.mp1 = m->d_u8a; ca.feat2 = m->d_i4;
    ca.d2 = reinterpret_cast<const uint32_t*>(m->d_desc2); ca.mp2 = m->d_u8b;
    ca.mp_only = mp_only; ca.cap = m->max_db; ca.cand = m->cand; ca.ncand = m->ncand; ca.scr_q = m->max_q;
    m->prof.begin(1, s);
    SE2_LAUNCH(k_candidates_bow, (nq * 32 + 255) / 256, 256, 0, s, ca);
    m->prof.end(s);
    ResolveArgs ra{};
    ra.nq_cap = nq; ra.d_nq = nullptr; ra.n2_cap = k2->n; ra.d_n2 = nullptr; ra.cap = m->max_db; ra.cand = m->cand; ra.ncand = m->ncand; ra.nnratio = nnratio;
    ra.ang1 = m->d_f1; ra.stride1 = 1; ra.ang2 = m->d_f2; ra.stride2 = 1; ra.check_ori = check_orientation;
    ra.qid = m->d_i1; ra.out = m->d_out; ra.n_out = k1->n; ra.nmatches = m->nm; ra.flags = m->flags;
    int rc = launch_resolve<MODE_BOW>(m, 1, ra, nullptr, s);
    if (rc != SE2GPU_OK) return rc;
    int* h_m = st.alloc<int>(k1->n); int* h_nm = st.alloc<int>(1);
    if (!h_m || !h_nm) return fail(SE2GPU_ERR_CAPACITY, "staging exhausted");
    SE2_CUDA(cudaMemcpyAsync(h_m, m->d_out, sizeof(int) * k1->n, cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaMemcpyAsync(h_nm, m->nm, sizeof(int), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    memcpy(matches12, h_m, sizeof(int) * k1->n);
    return *h_nm;
}

// handle-less entry points: a matcher per device is created on first use and kept (no allocation per call)
int se2gpu_match_by_window(const se2gpu_keypoint* kp1, const uint8_t* desc1, int n1, const se2gpu_keypoint* kp2,
                           const uint8_t* desc2, int n2, float* prev, se2gpu_grid_params grid, int win_size,
                           int level_offset, int min_level, int max_level, float nnratio, int* matches12, int device) {
    int rc = se2gpu::select_device(device);
    if (rc != SE2GPU_OK) return rc;
    std::lock_guard<std::mutex> lock(g_default_mutex);
    se2gpu_matcher* m = default_matcher(device, n1, n2);
    if (!m) return SE2GPU_ERR_CUDA;
    return se2gpu_matcher_match_by_window(m, kp1, desc1, n1, kp2, desc2, n2, prev, grid, win_size, level_offset, min_level, max_level, nnratio, matches12);
}

int se2gpu_match_by_projection(const se2gpu_keypoint* kf_kp, const uint8_t* kf_desc, int n_kf, const uint8_t* kf_observed,
                               const uint8_t* mp_valid, const float* mp_uv, int n_mp, const int* mp_octave,
                               const uint8_t* mp_desc, se2gpu_grid_params grid, int win_size, int level_offset,
                               float nnratio, int* matches_idx_mp, int device) {
    int rc = se2gpu::select_device(device);
    if (rc != SE2GPU_OK) return rc;
    std::lock_guard<std::mutex> lock(g_default_mutex);
    se2gpu_matcher* m = default_matcher(device, n_mp, n_kf);
    if (!m) return SE2GPU_ERR_CUDA;
    return se2gpu_matcher_match_by_projection(m, kf_kp, kf_desc, n_kf, kf_observed, mp_valid, mp_uv, n_mp, mp_octave, mp_desc, grid, win_size,
                                              level_offset, nnratio, matches_idx_mp);
}

int se2gpu_search_by_bow(const se2gpu_bow_kf* k1, const se2gpu_bow_kf* k2, int mp_only, float nnratio, int check_orientation,
                         int* matches12, int device) {
    if (!k1 || !k2) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    int rc = se2gpu::select_device(device);
    if (rc != SE2GPU_OK) return rc;
    std::lock_guard<std::mutex> lock(g_default_mutex);
    se2gpu_matcher* m = default_matcher(device, std::max(k1->n, k1->n_node ? k1->ptr[k1->n_node] : 0), std::max(k2->n, k2->n_node ? k2->ptr[k2->n_node] : 0));
    if (!m) return SE2GPU_ERR_CUDA;
    return se2gpu_matcher_search_by_bow(m, k1, k2, mp_only, nnratio, check_orientation, matches12);
}

}  // extern "C"
