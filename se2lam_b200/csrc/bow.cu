// Bag-of-words front end on sm_90a (SURVEY.md section 8f N4) - same popcount kernel family as the matchers:
//   se2gpu_voc_transform       DBoW2 TemplatedVocabulary::transform(feature, word_id, weight, nid, levelsup)
//                              (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1220-1262): every descriptor descends
//                              the k-ary vocabulary tree, at each level taking the child with the smallest Hamming distance
//                              (first child wins ties: the reference compares with a strict <). One warp per descriptor,
//                              lanes over the children of the current node, lexicographic (distance, child order) warp min.
//                              KeyFrame::ComputeBoW (src/KeyFrame.cpp:244-254) calls it for all descriptors of a keyframe with
//                              levelsup = 4.
//   se2gpu_voc_compute_bow_device
//                              transform(features, v, fv, levelsup) (:1150-1216) as KeyFrame::ComputeBoW calls it, for B
//                              keyframes per call: the descent above over B x cap descriptor slots, then k_bow_assemble, one
//                              CTA per keyframe, builds the BowVector (TF_IDF weights summed per word in feature order, L1
//                              normalised in word order) and the FeatureVector (ascending nodes, ascending feature lists) by
//                              stable rank counting in shared memory (DESIGN.md "Bag-of-words assembly on the device").
//   se2gpu_median_descriptor   MapPoint::updateMainKFandDescriptor (src/MapPoint.cpp:228-272): among the descriptors of a map
//                              point's observations pick the one with the least median Hamming distance to the others.
//                              One CTA per map point, distance matrix in shared memory, rank-counting selection of the
//                              element std::sort would put at index int(0.5*(N-1)).
#include <climits>
#include <vector>

#include "common.h"
#include "median_desc.h"

struct se2gpu_voc {
    int device = 0;
    int n_nodes = 0, levels = 0, max_children = 0;
    uint32_t* desc = nullptr;     // [n_nodes][8]
    int* child_ptr = nullptr;     // [n_nodes+1]
    int* children = nullptr;      // [child_ptr[n_nodes]]
    int* word_id = nullptr;       // [n_nodes]  (-1 = inner node)
    double* weight = nullptr;     // [n_nodes]
    // se2gpu_voc_compute_bow_device's per-descriptor triples [slots]; grown only when a call needs more slots than any before
    int* t_word = nullptr; double* t_weight = nullptr; int* t_node = nullptr;
    size_t slots = 0;
    int assemble_smem_max = 0;    // dynamic shared memory k_bow_assemble may use on this device
    se2gpu::DeviceBuffers bufs;
};

namespace {

using se2gpu::fail;

// one warp per feature slot; root = node 0. Slot f belongs to keyframe f / cap and is used when f % cap < d_n[f / cap]
// (d_n NULL: every slot of the n = B * cap).
__global__ void __launch_bounds__(256) k_voc_transform(const uint32_t* __restrict__ feat, int n, int cap, const int* __restrict__ d_n,
                                                       const uint32_t* __restrict__ ndesc,
                                                       const int* __restrict__ child_ptr, const int* __restrict__ children,
                                                       const int* __restrict__ word_of, const double* __restrict__ weight_of, int levels,
                                                       int levelsup, int* __restrict__ word_id, double* __restrict__ weight,
                                                       int* __restrict__ node_id) {
    const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (f >= n) return;
    if (d_n && f % cap >= se2gpu::count_of(d_n + f / cap, cap)) return;
    const uint4 q0 = *reinterpret_cast<const uint4*>(feat + 8 * (size_t)f), q1 = *reinterpret_cast<const uint4*>(feat + 8 * (size_t)f + 4);
    const int nid_level = levels - levelsup;
    int nid = (nid_level <= 0) ? 0 : -1;          // :1231 root; -1: the leaf is shallower than the requested level (the reference leaves *nid unset)
    int cur = 0, level = 0;
    while (true) {
        const int c0 = child_ptr[cur], c1 = child_ptr[cur + 1];
        if (c1 <= c0) break;                       // leaf
        ++level;
        int best = INT_MAX, bpos = INT_MAX;
        for (int k = c0 + lane; k < c1; k += 32) {
            const uint32_t* nd = ndesc + 8 * (size_t)children[k];
            const uint4 b0 = *reinterpret_cast<const uint4*>(nd), b1 = *reinterpret_cast<const uint4*>(nd + 4);
            const int d = __popc(q0.x ^ b0.x) + __popc(q0.y ^ b0.y) + __popc(q0.z ^ b0.z) + __popc(q0.w ^ b0.w) +
                          __popc(q1.x ^ b1.x) + __popc(q1.y ^ b1.y) + __popc(q1.z ^ b1.z) + __popc(q1.w ^ b1.w);
            if (d < best) { best = d; bpos = k; }  // ascending k per lane: the earliest child of the minimum stays
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int ob = __shfl_xor_sync(0xffffffffu, best, o), op = __shfl_xor_sync(0xffffffffu, bpos, o);
            if (ob < best || (ob == best && op < bpos)) { best = ob; bpos = op; }
        }
        cur = children[bpos];
        if (level == nid_level) nid = cur;         // :1253-1254
    }
    if (lane == 0) {
        word_id[f] = word_of[cur]; weight[f] = weight_of[cur];
        if (node_id) node_id[f] = nid;
    }
}

// transform(features, v, fv, levelsup)'s assembly (TemplatedVocabulary.h:1170-1190, BowVector::normalize L1 :62-84) for
// keyframe blockIdx.x from its descent triples at b * cap. A feature takes part when its weight is > 0 (:1181). Both maps
// come from one stable rank count over (key, feature index) packed into 64 bits, so equal words and equal nodes keep
// ascending feature order: the word value is then summed by one thread in feature order (v.addWeight, :1183) and the
// norm by one thread in ascending word order, as the reference's std::map walks do - double addition is not associative.
// Node -1 (the leaf above the requested level) is a key like any other and sorts first.
// Shared memory: 36 bytes per slot (bow_assemble_smem).
constexpr int ASSEMBLE_THREADS = 256;
__host__ __device__ constexpr size_t bow_assemble_smem(int cap) { return (size_t)cap * (8 + 8 + 8 + 4 + 4 + 4); }
__global__ void __launch_bounds__(ASSEMBLE_THREADS) k_bow_assemble(int cap, const int* __restrict__ d_n, const int* __restrict__ t_word,
                                                                   const double* __restrict__ t_weight, const int* __restrict__ t_node,
                                                                   int* __restrict__ bow_word, double* __restrict__ bow_value,
                                                                   int* __restrict__ bow_n, int* __restrict__ fv_node, int* __restrict__ fv_ptr,
                                                                   int* __restrict__ fv_feat, int* __restrict__ fv_n) {
    extern __shared__ __align__(16) unsigned char smem[];
    long long* kw = reinterpret_cast<long long*>(smem);           // [cap] word * 2^32 + i, LLONG_MAX when stopped
    long long* kn = kw + cap;                                     // [cap] node * 2^32 + i
    double* val = reinterpret_cast<double*>(kn + cap);           // [cap] word sums in word order
    int* ow = reinterpret_cast<int*>(val + cap);                  // [cap] feature at word rank r
    int* on = ow + cap;                                           // [cap] feature at node rank r
    int* run = on + cap;                                          // [cap] run starts, then the run index of a start
    __shared__ int s_warp[32], s_nv;
    __shared__ double s_norm;
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const size_t o = (size_t)b * cap;
    const int n = se2gpu::count_of(d_n ? d_n + b : nullptr, cap);
    t_word += o; t_weight += o; t_node += o;
    if (tid == 0) s_nv = 0;
    __syncthreads();
    int mine = 0;
    for (int i = tid; i < n; i += nt) {
        const bool used = t_weight[i] > 0;                         // :1181 "not stopped"
        kw[i] = used ? (long long)t_word[i] * 4294967296LL + i : LLONG_MAX;
        kn[i] = used ? (long long)t_node[i] * 4294967296LL + i : LLONG_MAX;
        mine += used;
    }
    if (mine) atomicAdd(&s_nv, mine);
    __syncthreads();
    const int nv = s_nv;
    for (int i = tid; i < n; i += nt) {
        const long long ki = kw[i], ni = kn[i];
        if (ki == LLONG_MAX) continue;
        int rw = 0, rn = 0;
        for (int j = 0; j < n; ++j) { rw += kw[j] < ki; rn += kn[j] < ni; }
        ow[rw] = i; on[rn] = i;
    }
    __syncthreads();
    // the ranks of one thread: a contiguous chunk, so that one exclusive sum numbers the runs in rank order
    const int per = (nv + nt - 1) / nt, lo = min(nv, tid * per), hi = min(nv, lo + per);
    auto key_at = [](const long long* k, const int* ord, int r) { return (int)(k[ord[r]] >> 32); };
    // FeatureVector: fv.addFeature(nid, i) (:1184), nodes ascending
    {
        int starts = 0;
        for (int r = lo; r < hi; ++r) starts += r == 0 || key_at(kn, on, r) != key_at(kn, on, r - 1);
        int total;
        int idx = se2gpu::block_exclusive_sum(starts, total, s_warp);
        fv_node += o; fv_ptr += (size_t)b * (cap + 1); fv_feat += o;
        for (int r = lo; r < hi; ++r) {
            if (r == 0 || key_at(kn, on, r) != key_at(kn, on, r - 1)) { fv_node[idx] = key_at(kn, on, r); fv_ptr[idx] = r; ++idx; }
            fv_feat[r] = on[r];
        }
        if (tid == 0) { fv_ptr[total] = nv; fv_n[b] = total; }
    }
    if (!bow_word) return;
    // BowVector: v.addWeight(id, w) in feature order (:1183), then normalize(L1)
    int starts = 0;
    for (int r = lo; r < hi; ++r) starts += r == 0 || key_at(kw, ow, r) != key_at(kw, ow, r - 1);
    int nw;
    int idx = se2gpu::block_exclusive_sum(starts, nw, s_warp);
    for (int r = lo; r < hi; ++r)
        if (r == 0 || key_at(kw, ow, r) != key_at(kw, ow, r - 1)) run[idx++] = r;
    __syncthreads();
    bow_word += o; bow_value += o;
    for (int k = tid; k < nw; k += nt) {
        const int r0 = run[k], r1 = k + 1 < nw ? run[k + 1] : nv;
        double v = t_weight[ow[r0]];
        for (int r = r0 + 1; r < r1; ++r) v = __dadd_rn(v, t_weight[ow[r]]);
        val[k] = v;
        bow_word[k] = key_at(kw, ow, r0);
    }
    __syncthreads();
    if (tid == 0) {                                               // BowVector.cpp:66-69: one ordered sum of |v|
        double norm = 0.0;
#pragma unroll 8
        for (int k = 0; k < nw; ++k) norm = __dadd_rn(norm, fabs(val[k]));
        s_norm = norm;
        bow_n[b] = nw;
    }
    __syncthreads();
    const double norm = s_norm;
    for (int k = tid; k < nw; k += nt) bow_value[k] = norm > 0.0 ? __ddiv_rn(val[k], norm) : val[k];
}

// one CTA per map point; dist [N*N] uint16 in dynamic shared memory
__global__ void __launch_bounds__(128) k_median_descriptor(const uint32_t* __restrict__ desc, const int* __restrict__ ptr, int M,
                                                           int* __restrict__ best_idx, int* __restrict__ best_median) {
    extern __shared__ unsigned short dist[];
    __shared__ int s_best;
    const int m = blockIdx.x;
    if (m >= M) return;
    const int p0 = ptr[m], N = ptr[m + 1] - p0;
    if (N <= 0) { if (threadIdx.x == 0) { best_idx[m] = -1; if (best_median) best_median[m] = INT_MAX; } return; }
    se2gpu::hamming_matrix(desc, [p0](int i) { return p0 + i; }, N, dist, threadIdx.x, blockDim.x);
    if (threadIdx.x == 0) s_best = INT_MAX;
    __syncthreads();
    const int kth = (int)(0.5 * (N - 1));          // vDists[0.5*(N-1)] after std::sort (MapPoint.cpp:263)
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int median = se2gpu::rank_select(dist + (size_t)i * N, N, kth);
        atomicMin(&s_best, (median << 16) | i);    // lexicographic (median, index): the first index of the least median (:264-267)
    }
    __syncthreads();
    if (threadIdx.x == 0) { best_idx[m] = s_best & 0xffff; if (best_median) best_median[m] = s_best >> 16; }
}

}  // namespace

extern "C" {

se2gpu_voc* se2gpu_voc_create(int n_nodes, const uint8_t* node_desc, const int* child_ptr, const int* children,
                              const int* word_id, const double* weight, int levels, int device) {
    if (n_nodes <= 0 || !node_desc || !child_ptr || !children || !word_id || !weight || levels <= 0) { fail(SE2GPU_ERR_INVALID, "bad vocabulary"); return nullptr; }
    if (child_ptr[0] != 0) { fail(SE2GPU_ERR_INVALID, "child_ptr[0] must be 0"); return nullptr; }
    int max_children = 0;
    for (int i = 0; i < n_nodes; ++i) {
        const int c = child_ptr[i + 1] - child_ptr[i];
        if (c < 0) { fail(SE2GPU_ERR_INVALID, "child_ptr must be non-decreasing"); return nullptr; }
        max_children = std::max(max_children, c);
        if (c == 0 && word_id[i] < 0) { fail(SE2GPU_ERR_INVALID, "leaf %d has no word id", i); return nullptr; }
    }
    const int nc = child_ptr[n_nodes];
    for (int k = 0; k < nc; ++k) if (children[k] <= 0 || children[k] >= n_nodes) { fail(SE2GPU_ERR_INVALID, "child index out of range"); return nullptr; }
    if (se2gpu::select_device(device) != SE2GPU_OK) return nullptr;
    se2gpu_voc* v = new se2gpu_voc;
    v->device = device; v->n_nodes = n_nodes; v->levels = levels; v->max_children = max_children;
    bool ok = v->bufs.alloc(&v->desc, (size_t)n_nodes * 8) == cudaSuccess && v->bufs.alloc(&v->child_ptr, (size_t)n_nodes + 1) == cudaSuccess &&
              v->bufs.alloc(&v->children, (size_t)nc) == cudaSuccess && v->bufs.alloc(&v->word_id, (size_t)n_nodes) == cudaSuccess &&
              v->bufs.alloc(&v->weight, (size_t)n_nodes) == cudaSuccess;
    ok = ok && cudaMemcpy(v->desc, node_desc, (size_t)n_nodes * 32, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->child_ptr, child_ptr, sizeof(int) * ((size_t)n_nodes + 1), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->children, children, sizeof(int) * (size_t)nc, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->word_id, word_id, sizeof(int) * (size_t)n_nodes, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->weight, weight, sizeof(double) * (size_t)n_nodes, cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        int optin = 0;
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        v->assemble_smem_max = std::max(optin - 2048, 46 * 1024);
        ok = cudaFuncSetAttribute(k_bow_assemble, cudaFuncAttributeMaxDynamicSharedMemorySize, v->assemble_smem_max) == cudaSuccess;
    }
    if (!ok) { fail(SE2GPU_ERR_CUDA, "vocabulary upload failed: %s", cudaGetErrorString(cudaGetLastError())); se2gpu_voc_destroy(v); return nullptr; }
    return v;
}

void se2gpu_voc_destroy(se2gpu_voc* v) {
    if (!v) return;
    cudaSetDevice(v->device);
    delete v;
}

int se2gpu_voc_transform_device(se2gpu_voc* v, const uint8_t* d_desc, int n, int levelsup, int* d_word_id, double* d_weight,
                                int* d_node_id, void* stream) {
    if (!v) return fail(SE2GPU_ERR_INVALID, "null vocabulary");
    if (n < 0 || (n && (!d_desc || !d_word_id || !d_weight))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n == 0) return SE2GPU_OK;
    SE2_NVTX("se2gpu.voc_transform");
    SE2_CUDA(cudaSetDevice(v->device));
    SE2_LAUNCH(k_voc_transform, (n * 32 + 255) / 256, 256, 0, (cudaStream_t)stream, reinterpret_cast<const uint32_t*>(d_desc), n, n, nullptr, v->desc,
               v->child_ptr, v->children, v->word_id, v->weight, v->levels, levelsup, d_word_id, d_weight, d_node_id);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_voc_compute_bow_device(se2gpu_voc* v, int B, const uint8_t* d_desc, int cap, const int* d_n, int levelsup, int* d_bow_word,
                                  double* d_bow_value, int* d_bow_n, int* d_fv_node, int* d_fv_ptr, int* d_fv_feat, int* d_fv_n,
                                  void* stream) {
    if (!v) return fail(SE2GPU_ERR_INVALID, "null vocabulary");
    if (B < 0 || cap < 0) return fail(SE2GPU_ERR_INVALID, "negative sizes");
    const int nbow = !!d_bow_word + !!d_bow_value + !!d_bow_n;
    if (nbow != 0 && nbow != 3) return fail(SE2GPU_ERR_INVALID, "the BowVector outputs are all given or all NULL");
    if (B == 0) return SE2GPU_OK;
    if (!d_fv_node || !d_fv_ptr || !d_fv_feat || !d_fv_n || (cap && !d_desc)) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (bow_assemble_smem(cap) > (size_t)v->assemble_smem_max)
        return fail(SE2GPU_ERR_CAPACITY, "%d features per keyframe: at most %d fit the assembly's shared memory", cap,
                    (int)(v->assemble_smem_max / bow_assemble_smem(1)));
    if ((size_t)B * cap * 32 > (size_t)INT_MAX) return fail(SE2GPU_ERR_CAPACITY, "%d keyframes of %d features: too many descriptor slots", B, cap);
    SE2_NVTX("se2gpu.voc_compute_bow");
    SE2_CUDA(cudaSetDevice(v->device));
    const size_t slots = (size_t)B * cap;
    if (slots > v->slots) {          // the first call of a larger batch; cudaFree waits for the calls still reading them
        if (v->bufs.regrow(&v->t_word, slots) != cudaSuccess || v->bufs.regrow(&v->t_weight, slots) != cudaSuccess ||
            v->bufs.regrow(&v->t_node, slots) != cudaSuccess) {
            v->slots = 0;
            return fail(SE2GPU_ERR_CUDA, "vocabulary scratch for %zu descriptors: %s", slots, cudaGetErrorString(cudaGetLastError()));
        }
        v->slots = slots;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (slots)
        SE2_LAUNCH(k_voc_transform, (int)((slots * 32 + 255) / 256), 256, 0, s, reinterpret_cast<const uint32_t*>(d_desc), (int)slots, cap, d_n,
                   v->desc, v->child_ptr, v->children, v->word_id, v->weight, v->levels, levelsup, v->t_word, v->t_weight, v->t_node);
    SE2_LAUNCH(k_bow_assemble, B, ASSEMBLE_THREADS, bow_assemble_smem(cap), s, cap, d_n, v->t_word, v->t_weight, v->t_node, d_bow_word,
               d_bow_value, d_bow_n, d_fv_node, d_fv_ptr, d_fv_feat, d_fv_n);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_voc_transform(se2gpu_voc* v, const uint8_t* desc, int n, int levelsup, int* word_id, double* weight, int* node_id) {
    if (!v) return fail(SE2GPU_ERR_INVALID, "null vocabulary");
    if (n < 0 || (n && (!desc || !word_id || !weight))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n == 0) return SE2GPU_OK;
    se2gpu::HostStage st(v->device);
    const uint8_t* d_in = st.upload(desc, (size_t)n * 32);
    int* d_word = st.output(word_id, n);
    double* d_w = st.output(weight, n);
    int* d_node = node_id ? st.output(node_id, n) : st.scratch<int>(n);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_voc_transform_device(v, d_in, n, levelsup, d_word, d_w, d_node, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_median_descriptor(const uint8_t* desc, const int* ptr, int M, int* best_idx, int* best_median, int device) {
    if (M < 0 || (M && (!desc || !ptr || !best_idx))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (M == 0) return SE2GPU_OK;
    int maxN = 0;
    for (int m = 0; m < M; ++m) { if (ptr[m + 1] < ptr[m]) return fail(SE2GPU_ERR_INVALID, "ptr must be non-decreasing"); maxN = std::max(maxN, ptr[m + 1] - ptr[m]); }
    const size_t smem = (size_t)maxN * maxN * sizeof(unsigned short);
    if (maxN > 320) return fail(SE2GPU_ERR_CAPACITY, "a map point with %d observations exceeds this build's limit of 320", maxN);
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    const size_t total = (size_t)ptr[M];
    const uint32_t* d_desc = st.upload(reinterpret_cast<const uint32_t*>(desc), total * 8);
    const int* d_ptr = st.upload(ptr, (size_t)M + 1);
    int* d_idx = st.output(best_idx, M);
    int* d_med = best_median ? st.output(best_median, M) : st.scratch<int>(M);
    if (smem > 48 * 1024) st.check(cudaFuncSetAttribute(k_median_descriptor, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute");
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_median_descriptor, M, 128, smem, 0, d_desc, d_ptr, M, d_idx, d_med);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

}  // extern "C"
