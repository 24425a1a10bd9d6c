// Bag-of-words front end on sm_90a (SURVEY.md section 8f N4) - same popcount kernel family as the matchers:
//   se2gpu_voc_transform       DBoW2 TemplatedVocabulary::transform(feature, word_id, weight, nid, levelsup)
//                              (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1220-1262): every descriptor descends
//                              the k-ary vocabulary tree, at each level taking the child with the smallest Hamming distance
//                              (first child wins ties: the reference compares with a strict <). One warp per descriptor,
//                              lanes over the children of the current node, lexicographic (distance, child order) warp min.
//                              KeyFrame::ComputeBoW (src/KeyFrame.cpp:244-254) calls it for all descriptors of a keyframe with
//                              levelsup = 4.
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
    se2gpu::DeviceBuffers bufs;
};

namespace {

using se2gpu::fail;

// one warp per feature; root = node 0
__global__ void __launch_bounds__(256) k_voc_transform(const uint32_t* __restrict__ feat, int n, const uint32_t* __restrict__ ndesc,
                                                       const int* __restrict__ child_ptr, const int* __restrict__ children,
                                                       const int* __restrict__ word_of, const double* __restrict__ weight_of, int levels,
                                                       int levelsup, int* __restrict__ word_id, double* __restrict__ weight,
                                                       int* __restrict__ node_id) {
    const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (f >= n) return;
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
    SE2_LAUNCH(k_voc_transform, (n * 32 + 255) / 256, 256, 0, (cudaStream_t)stream, reinterpret_cast<const uint32_t*>(d_desc), n, v->desc, v->child_ptr,
               v->children, v->word_id, v->weight, v->levels, levelsup, d_word_id, d_weight, d_node_id);
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
