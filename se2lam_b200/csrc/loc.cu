// Localizer::run (reference src/Localizer.cpp:32-176) for a batch of camera streams against a static map kept on the
// device (DESIGN.md section 15). The map goes up once at create. The device part of a step (extraction, MatchLocalMap,
// DoLocalBA, UpdateCovisKFCurr, UpdateLocalMap(1) and the record) is one CUDA graph per (B, w, h); UpdatePoseCurr runs
// here on the host with the tracker's Se2 arithmetic, so the pose a step starts from is the reference's bit for bit.
// The relocalization (the verified branch of Localizer::run) runs the same kernels by direct launches.
//
// Stream b's per-step work is selected by mode[b] (1: tracked), which the kernels read from the step's staging copy; the
// local map of a stream that does not run is left as it is. No kernel here uses atomics: set membership is written as
// byte stores of 1, and lists are compacted with warp ballots in ascending order.
#include <cmath>

#include "common.h"
#include "fround.h"
#include "se2_host.h"

using namespace se2gpu;

namespace {

constexpr int kBlock = 256;
// the step's device block, 4-byte words: Tcw [16 S] | mode [S] | aux [S] | record [kRec S]
enum Rec { R_KP, R_MATCHED, R_OBS, R_SKIP, R_STATUS, R_ITERS, R_NKF, R_NMP, R_EDGES, kRec };

struct Map {
    int K = 0, M = 0;
    const int *kp_ptr, *kf_obs_mp, *obs_ptr, *obs, *cov_ptr, *cov, *mp_oct;
    const float* mp_pos;
    const uint8_t *mp_use, *mp_null, *mp_desc;
};

// ---------------------------------------------------------------------------------------------- kernels
// ReadFrameInfo: the new keyframe of every stream b < B starts with no observation (mObservations, mDualObservations)
__global__ void __launch_bounds__(kBlock) k_loc_begin(int cap, int M, int* __restrict__ obs_mp, uint8_t* __restrict__ kf_obsd,
                                                      uint8_t* __restrict__ has_mp) {
    const int b = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(cap, M); i += gridDim.x * blockDim.x) {
        if (i < cap) { obs_mp[(size_t)b * cap + i] = -1; kf_obsd[(size_t)b * cap + i] = 0; }
        if (i < M) has_mp[(size_t)b * M + i] = 0;
    }
}

// MatchLocalMap's flattening (ORBmatcher::MatchByProjection, ORBmatcher.cpp:390-400) for slot j of stream b's local list:
// valid = !isNull && isGoodPrl && !hasObservation(pMP) && inImgBound(camprjc(K, se3map(Tcw, pos))), inclusive bounds
__global__ void __launch_bounds__(kBlock) k_loc_project(Map m, const float* __restrict__ Tcw_all, const int* __restrict__ mode,
                                                        const int* __restrict__ n_local, const int* __restrict__ local, int cap_mp,
                                                        const uint8_t* __restrict__ has_mp, const float* __restrict__ K, float x0,
                                                        float x1, float y0, float y1, uint8_t* __restrict__ valid,
                                                        float* __restrict__ uv, int* __restrict__ octave, uint4* __restrict__ desc) {
    const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= cap_mp) return;
    const size_t k = (size_t)b * cap_mp + j;
    uint8_t ok = 0;
    if (mode[b] && j < min(n_local[b], cap_mp)) {
        const int mp = local[k];
        if (m.mp_use[mp] && !has_mp[(size_t)b * m.M + mp]) {
            float T[16];
#pragma unroll
            for (int q = 0; q < 16; q++) T[q] = Tcw_all[16 * b + q];
            const F3 p = se3map(T, {m.mp_pos[3 * (size_t)mp], m.mp_pos[3 * (size_t)mp + 1], m.mp_pos[3 * (size_t)mp + 2]});
            float u, v;
            camprjc(K, p, &u, &v);
            if (u >= x0 && u <= x1 && v >= y0 && v <= y1) {
                ok = 1;
                uv[2 * k] = u; uv[2 * k + 1] = v;
                octave[k] = m.mp_oct[mp];
                const uint4* d = reinterpret_cast<const uint4*>(m.mp_desc) + 2 * (size_t)mp;
                desc[2 * k] = d[0]; desc[2 * k + 1] = d[1];
            }
        }
    }
    valid[k] = ok;
}

// MatchLocalMap's KeyFrame::addObservation(vpMPLocal[idx], i) for every matched keypoint i of a running stream
__global__ void __launch_bounds__(kBlock) k_loc_apply(int M, const int* __restrict__ mode, const int* __restrict__ n_kp, int cap,
                                                      const int* __restrict__ matches, const int* __restrict__ local, int cap_mp,
                                                      int* __restrict__ obs_mp, uint8_t* __restrict__ kf_obsd,
                                                      uint8_t* __restrict__ has_mp) {
    const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!mode[b] || i >= count_of(n_kp + b, cap)) return;
    const size_t k = (size_t)b * cap + i;
    const int q = matches[k];
    if (q < 0 || q >= cap_mp) return;
    const int mp = local[(size_t)b * cap_mp + q];
    obs_mp[k] = mp; kf_obsd[k] = 1;
    has_mp[(size_t)b * M + mp] = 1;
}

// UpdateCovisKFCurr (Localizer.cpp:675-687): one warp per (stream, keyframe); keyframe k of the previous local set becomes
// covisible when the map points it shares with the current keyframe (Map::compareViewMPs) are more than 0.1 * getSizeObsMP()
__global__ void __launch_bounds__(kBlock) k_loc_covis(Map m, const int* __restrict__ mode, const int* __restrict__ n_obs,
                                                      const uint8_t* __restrict__ has_mp, const uint8_t* __restrict__ kf_local,
                                                      uint8_t* __restrict__ kf_cov) {
    const int b = blockIdx.y, lane = threadIdx.x & 31;
    const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= m.K) return;
    const size_t bk = (size_t)b * m.K + k;
    const bool in = mode[b] && kf_local[bk];
    int c = 0;
    if (in)
        for (int e = m.obs_ptr[k] + lane; e < m.obs_ptr[k + 1]; e += 32) c += has_mp[(size_t)b * m.M + m.obs[e]];
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) kf_cov[bk] = in && (double)c > 0.1 * (double)n_obs[b];
}

// the relocalization's setPose / addCovisibleKF(kfLoop): covisible = {aux[b]} for the streams it runs
__global__ void __launch_bounds__(kBlock) k_loc_seed(int K, const int* __restrict__ mode, const int* __restrict__ aux,
                                                     uint8_t* __restrict__ kf_cov) {
    const int b = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
    if (mode[b] && k < K) kf_cov[(size_t)b * K + k] = k == aux[b];
}

// UpdateLocalMap(hops) (Localizer.cpp:631-655) and DetectIfLost, one CTA per running stream: the local keyframes are the
// covisible set, expanded `hops` times through the covisibility lists (each hop from a snapshot of the set, as the
// reference iterates a copy); the local map points are the union of their getAllObsMPs(true) (not null, good parallax),
// listed in ascending map-point index. At most cap_mp are written; n_mp gets the full count.
__global__ void __launch_bounds__(1024) k_loc_local_map(Map m, const int* __restrict__ mode, int hops, const uint8_t* __restrict__ kf_cov,
                                                        uint8_t* __restrict__ kf_local, uint8_t* __restrict__ kf_tmp,
                                                        uint8_t* __restrict__ mark, int* __restrict__ local, int cap_mp,
                                                        int* __restrict__ n_kf_out, int* __restrict__ n_mp_out) {
    __shared__ int s_w[32];
    __shared__ int s_base;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    if (!mode[b]) return;
    const size_t ko = (size_t)b * m.K, mo = (size_t)b * m.M;
    for (int k = tid; k < m.K; k += blockDim.x) kf_local[ko + k] = kf_cov[ko + k];
    for (int j = tid; j < m.M; j += blockDim.x) mark[mo + j] = 0;
    __syncthreads();
    for (int h = 0; h < hops; h++) {
        for (int k = tid; k < m.K; k += blockDim.x) kf_tmp[ko + k] = kf_local[ko + k];
        __syncthreads();
        for (int k = warp; k < m.K; k += nw)
            if (kf_tmp[ko + k])
                for (int e = m.cov_ptr[k] + lane; e < m.cov_ptr[k + 1]; e += 32) kf_local[ko + m.cov[e]] = 1;
        __syncthreads();
    }
    int nk = 0;
    for (int k = warp; k < m.K; k += nw) {       // one warp per local keyframe walks its observation list
        if (!kf_local[ko + k]) continue;
        nk += lane == 0;
        for (int e = m.obs_ptr[k] + lane; e < m.obs_ptr[k + 1]; e += 32) {
            const int j = m.obs[e];
            if (m.mp_use[j]) mark[mo + j] = 1;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) nk += __shfl_xor_sync(0xffffffffu, nk, o);
    if (lane == 0) s_w[warp] = nk;
    if (tid == 0) s_base = 0;
    __syncthreads();
    if (tid == 0) {
        int t = 0;
        for (int v = 0; v < nw; v++) t += s_w[v];
        n_kf_out[b] = t;
    }
    __syncthreads();
    for (int j0 = 0; j0 < m.M; j0 += blockDim.x) {
        const int j = j0 + tid;
        const bool take = j < m.M && mark[mo + j];
        const unsigned bal = __ballot_sync(0xffffffffu, take);
        if (lane == 0) s_w[warp] = __popc(bal);
        __syncthreads();
        int off = s_base;
        for (int v = 0; v < warp; v++) off += s_w[v];
        off += __popc(bal & ((1u << lane) - 1));
        if (take && off < cap_mp) local[(size_t)b * cap_mp + off] = j;
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int v = 0; v < nw; v++) t += s_w[v];
            s_base += t;
        }
        __syncthreads();
    }
    if (tid == 0) n_mp_out[b] = s_base;
}

// MatchLoopClose (Localizer.cpp:658-673) for the pairs (stream, idxCurr, idxLoop): the keyframe aux[stream]'s map point at
// idxLoop, when there is one and it is not null (KeyFrame::addObservation), becomes the observation of idxCurr
__global__ void __launch_bounds__(kBlock) k_loc_loop_close(Map m, int n, const int* __restrict__ pairs, const int* __restrict__ aux,
                                                           int cap, int* __restrict__ obs_mp, uint8_t* __restrict__ kf_obsd,
                                                           uint8_t* __restrict__ has_mp) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int b = pairs[3 * e], ic = pairs[3 * e + 1], il = pairs[3 * e + 2];
    const int mp = m.kf_obs_mp[m.kp_ptr[aux[b]] + il];
    if (mp < 0 || m.mp_null[mp]) return;
    const size_t k = (size_t)b * cap + ic;
    obs_mp[k] = mp; kf_obsd[k] = 1;
    has_mp[(size_t)b * m.M + mp] = 1;
}

struct StreamState {
    bool has_frame = false, first = false, tracked = false, overflow = false;
    bool lost_branch = false;   // the last step began with mbIsTracked false and ran Localizer::run's else branch
    Se2 odom{0, 0, 0};
    float Tcw[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
};

bool params_ok(const se2gpu_loc_params* p) {
    if (!p || p->nfeatures <= 0 || p->nlevels <= 0 || p->nlevels > 16 || !(p->scale_factor > 1.f) || p->max_local_mps <= 0 ||
        p->ba.iterations < 0)
        return false;
    return p->ndist == 0 || p->ndist == 4 || p->ndist == 5 || p->ndist == 8 || p->ndist == 12;
}

// a CSR over n rows into [0, range): ptr[0] == 0, monotone; with `strict`, every row strictly ascending
bool csr_ok(int n, const int* ptr, const int* idx, int range, bool strict) {
    if (!ptr || ptr[0] != 0) return false;
    for (int r = 0; r < n; r++) {
        if (ptr[r + 1] < ptr[r]) return false;
        if (ptr[r + 1] > ptr[r] && !idx) return false;
        for (int e = ptr[r]; e < ptr[r + 1]; e++) {
            if (idx[e] < (strict ? 0 : -1) || idx[e] >= range) return false;
            if (strict && e > ptr[r] && idx[e] <= idx[e - 1]) return false;
        }
    }
    return true;
}

int map_ok(const se2gpu_loc_map* m, int nlevels) {
    if (!m || m->n_kf < 0 || m->n_mp < 0) return fail(SE2GPU_ERR_INVALID, "bad map sizes");
    const int K = m->n_kf, M = m->n_mp;
    if (K && !m->kf_Tcw) return fail(SE2GPU_ERR_INVALID, "null keyframe poses");
    if (M && (!m->mp_pos || !m->mp_null || !m->mp_good_prl || !m->mp_desc || !m->mp_octave)) return fail(SE2GPU_ERR_INVALID, "null map-point arrays");
    if (!csr_ok(K, m->kf_kp_ptr, m->kf_obs_mp, M, false)) return fail(SE2GPU_ERR_INVALID, "keypoint slots: bad CSR or map-point index");
    if (!csr_ok(K, m->kf_obs_ptr, m->kf_obs, M, true)) return fail(SE2GPU_ERR_INVALID, "observations: bad CSR or map-point index");
    if (!csr_ok(K, m->kf_cov_ptr, m->kf_cov, K, true)) return fail(SE2GPU_ERR_INVALID, "covisibility: bad CSR or keyframe index");
    for (int j = 0; j < M; j++)
        if (m->mp_octave[j] < 0 || m->mp_octave[j] >= nlevels) return fail(SE2GPU_ERR_INVALID, "map point %d: octave %d", j, m->mp_octave[j]);
    return SE2GPU_OK;
}

// UpdatePoseCurr (Localizer.cpp:614-619): Tcw = cTb * Se2(ref.odom - cur.odom).toCvSE3() * bTc * ref.Tcw
void host_pose(const se2gpu_loc_params& p, const Se2& odom, const Se2& ref_odom, const float* ref_Tcw, float* Tcw) {
    float Tcr[16];
    cam_motion(p.cTb, p.bTc, se2_minus(ref_odom, odom), Tcr);
    gemm4(Tcr, ref_Tcw, Tcw);
}

Se2 odo3(const float* o) { return se2(o[0], o[1], o[2]); }

}  // namespace

struct se2gpu_loc {
    int device = 0, S = 0, C = 0, Q = 0, max_w = 0, max_h = 0;
    se2gpu_loc_params p{};
    Map map;
    std::vector<float> kf_Tcw;
    std::vector<int> kf_nkp;
    se2gpu_orb* orb = nullptr;
    se2gpu_matcher* matcher = nullptr;
    cudaStream_t s = nullptr;
    DeviceBuffers bufs;
    uint8_t* d_frames = nullptr;
    se2gpu_keypoint* d_kp = nullptr;
    uint8_t *d_desc = nullptr, *d_kf_obsd = nullptr, *d_has_mp = nullptr, *d_mark = nullptr;
    uint8_t *d_kf_cov = nullptr, *d_kf_local = nullptr, *d_kf_tmp = nullptr;
    int *d_obs_mp = nullptr, *d_local = nullptr, *d_matches = nullptr, *d_best = nullptr, *d_pairs = nullptr;
    uint8_t *d_valid = nullptr, *d_mpdesc = nullptr;
    float *d_uv = nullptr, *d_exyz = nullptr, *d_euv = nullptr, *d_ew = nullptr, *d_K = nullptr, *d_isig = nullptr;
    int* d_oct = nullptr;
    uint32_t* d_io = nullptr;   // Tcw | mode | aux | record
    PinnedArena pin;
    uint32_t* h_io = nullptr;
    int* h_pairs = nullptr;
    cudaGraphExec_t exec = nullptr;
    int gB = 0, gw = 0, gh = 0, g_kernels = 0, g_nodes = 0;
    bool eager = false;
    std::vector<StreamState> st;

    float* Tcw(uint32_t* io) const { return reinterpret_cast<float*>(io); }
    int* mode(uint32_t* io) const { return reinterpret_cast<int*>(io + 16 * (size_t)S); }
    int* aux(uint32_t* io) const { return reinterpret_cast<int*>(io + 17 * (size_t)S); }
    int* rec(uint32_t* io, int f) const { return reinterpret_cast<int*>(io + (18 + (size_t)f) * S); }
    size_t up_words() const { return 18 * (size_t)S; }
    size_t io_words() const { return (18 + (size_t)kRec) * S; }

    ~se2gpu_loc() {
        if (device >= 0) cudaSetDevice(device);
        if (s) cudaStreamSynchronize(s);
        if (exec) cudaGraphExecDestroy(exec);
        if (s) cudaStreamDestroy(s);
        se2gpu_matcher_destroy(matcher);
        se2gpu_orb_destroy(orb);
    }
};

namespace {

// MatchLocalMap for the streams with mode set, B streams wide: the projection, MatchByProjection(mpKFCurr, local, 15, 2)
// with nnratio 0.9 and the observations it adds
int enqueue_match(se2gpu_loc* h, int B) {
    const int S = h->S, C = h->C, Q = h->Q;
    const se2gpu_loc_params& p = h->p;
    SE2_LAUNCH(k_loc_project, dim3((Q + kBlock - 1) / kBlock, B), kBlock, 0, h->s, h->map, h->Tcw(h->d_io), h->mode(h->d_io),
               h->rec(h->d_io, R_NMP), h->d_local, Q, h->d_has_mp, h->d_K, p.min_x, p.max_x, p.min_y, p.max_y, h->d_valid, h->d_uv,
               h->d_oct, reinterpret_cast<uint4*>(h->d_mpdesc));
    SE2_CUDA(cudaGetLastError());
    int rc = se2gpu_match_by_projection_batch_device(h->matcher, B, h->d_kp, h->d_desc, C, h->rec(h->d_io, R_KP), h->d_kf_obsd, h->d_valid,
                                                     h->d_uv, Q, h->d_oct, h->d_mpdesc, p.grid, 15, 2, 0.9f, h->d_matches,
                                                     h->rec(h->d_io, R_MATCHED), h->s);
    if (rc) return rc;
    SE2_LAUNCH(k_loc_apply, dim3((C + kBlock - 1) / kBlock, B), kBlock, 0, h->s, h->map.M, h->mode(h->d_io), h->rec(h->d_io, R_KP), C,
               h->d_matches, h->d_local, Q, h->d_obs_mp, h->d_kf_obsd, h->d_has_mp);
    SE2_CUDA(cudaGetLastError());
    (void)S;
    return SE2GPU_OK;
}

// DoLocalBA for the streams with mode set (min_obs >= 0: only above that many observations)
int enqueue_ba(se2gpu_loc* h, int B, int min_obs) {
    return loc_local_ba(B, h->d_kp, h->C, h->rec(h->d_io, R_KP), h->d_obs_mp, h->map.M, h->map.mp_pos, h->map.mp_use, h->d_isig, h->p.nlevels,
                        h->mode(h->d_io), min_obs, h->d_best, h->d_exyz, h->d_euv, h->d_ew, h->rec(h->d_io, R_EDGES),
                        h->rec(h->d_io, R_SKIP), h->rec(h->d_io, R_OBS), h->Tcw(h->d_io), &h->p.ba, h->rec(h->d_io, R_ITERS),
                        h->rec(h->d_io, R_STATUS), h->s);
}

int enqueue_local_map(se2gpu_loc* h, int B, int hops) {
    SE2_LAUNCH(k_loc_local_map, B, 1024, 0, h->s, h->map, h->mode(h->d_io), hops, h->d_kf_cov, h->d_kf_local, h->d_kf_tmp, h->d_mark,
               h->d_local, h->Q, h->rec(h->d_io, R_NKF), h->rec(h->d_io, R_NMP));
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

// the device work of one step for streams 0 .. B-1, capturable: the frames are in d_frames, the poses and modes in h_io
int enqueue_step(se2gpu_loc* h, int B, int w, int hgt) {
    const int C = h->C;
    cudaStream_t s = h->s;
    SE2_CUDA(cudaMemcpyAsync(h->d_io, h->h_io, sizeof(uint32_t) * h->up_words(), cudaMemcpyHostToDevice, s));
    int rc = se2gpu_orb_extract_device(h->orb, h->d_frames, B, w, hgt, w, (size_t)w * hgt, h->d_kp, h->d_desc, h->rec(h->d_io, R_KP), s);
    if (rc) return rc;
    SE2_LAUNCH(k_loc_begin, dim3((std::max(C, h->map.M) + kBlock - 1) / kBlock, B), kBlock, 0, s, C, h->map.M, h->d_obs_mp, h->d_kf_obsd,
               h->d_has_mp);
    SE2_CUDA(cudaGetLastError());
    if ((rc = enqueue_match(h, B))) return rc;
    if ((rc = enqueue_ba(h, B, 30))) return rc;
    if (h->map.K) {
        SE2_LAUNCH(k_loc_covis, dim3((h->map.K * 32 + kBlock - 1) / kBlock, B), kBlock, 0, s, h->map, h->mode(h->d_io), h->rec(h->d_io, R_OBS),
                   h->d_has_mp, h->d_kf_local, h->d_kf_cov);
        SE2_CUDA(cudaGetLastError());
    }
    if ((rc = enqueue_local_map(h, B, 1))) return rc;
    SE2_CUDA(cudaMemcpyAsync(h->h_io, h->d_io, sizeof(uint32_t) * h->io_words(), cudaMemcpyDeviceToHost, s));
    return SE2GPU_OK;
}

int ensure_graph(se2gpu_loc* h, int B, int w, int hgt) {
    if (h->exec && h->gB == B && h->gw == w && h->gh == hgt) return SE2GPU_OK;
    if (int rc = orb_prepare_shape(h->orb, w, hgt, h->s)) return rc;
    SE2_CUDA(cudaStreamSynchronize(h->s));
    if (h->exec) { cudaGraphExecDestroy(h->exec); h->exec = nullptr; }
    h->gB = h->gw = h->gh = 0;
    SE2_CUDA(cudaStreamBeginCapture(h->s, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue_step(h, B, w, hgt);
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(h->s, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (e != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "capturing the step failed: %s", cudaGetErrorString(e));
    size_t n = 0;
    cudaGraphGetNodes(graph, nullptr, &n);
    std::vector<cudaGraphNode_t> nodes(n);
    int kernels = 0;
    if (n) cudaGraphGetNodes(graph, nodes.data(), &n);
    for (cudaGraphNode_t nd : nodes) {
        cudaGraphNodeType ty;
        if (cudaGraphNodeGetType(nd, &ty) == cudaSuccess && ty == cudaGraphNodeTypeKernel) kernels++;
    }
    const cudaError_t ei = cudaGraphInstantiate(&h->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ei != cudaSuccess) { h->exec = nullptr; return fail(SE2GPU_ERR_CUDA, "instantiating the step graph failed: %s", cudaGetErrorString(ei)); }
    h->gB = B; h->gw = w; h->gh = hgt; h->g_kernels = kernels; h->g_nodes = (int)n;
    return SE2GPU_OK;
}

// one stream's result from the record in h_io after a call that ran it (ran: mode was set)
void fill_result(se2gpu_loc* h, int b, bool ran, se2gpu_loc_result& r) {
    StreamState& ss = h->st[b];
    std::memset(&r, 0, sizeof r);
    r.first = ss.first;
    r.n_keypoints = h->rec(h->h_io, R_KP)[b];
    r.ba_status = SE2GPU_POSE_BA_NO_EDGES;
    if (ran) {
        r.n_matched = h->rec(h->h_io, R_MATCHED)[b];
        r.n_obs_mp = h->rec(h->h_io, R_OBS)[b];
        r.ba_status = h->rec(h->h_io, R_STATUS)[b];
        r.ba_iterations = h->rec(h->h_io, R_ITERS)[b];
        r.n_local_kfs = h->rec(h->h_io, R_NKF)[b];
        r.n_local_mps = h->rec(h->h_io, R_NMP)[b];
        std::memcpy(ss.Tcw, h->Tcw(h->h_io) + 16 * b, sizeof ss.Tcw);
        ss.tracked = r.n_local_kfs > 0;                  // DetectIfLost
        ss.overflow = r.n_local_mps > h->Q;
    }
    r.tracked = ss.tracked;
    r.overflow = ss.overflow;
    std::memcpy(r.Tcw, ss.Tcw, sizeof r.Tcw);
}

}  // namespace

extern "C" {

se2gpu_loc* se2gpu_loc_create(int max_streams, int max_w, int max_h, const se2gpu_loc_params* params, const se2gpu_loc_map* map,
                              int device) {
    if (max_streams <= 0 || max_w <= 0 || max_h <= 0 || !params_ok(params)) { fail(SE2GPU_ERR_INVALID, "bad arguments"); return nullptr; }
    if (max_streams > 65535) { fail(SE2GPU_ERR_CAPACITY, "%d streams: at most 65535", max_streams); return nullptr; }
    if (map_ok(map, params->nlevels)) return nullptr;
    if (select_device(device) != SE2GPU_OK) return nullptr;
    if (!matcher_window_capturable(device, params->max_local_mps, params->nfeatures)) {
        fail(SE2GPU_ERR_CAPACITY, "%d local map points x %d features are too many for the matcher's shared-memory resolve",
             params->max_local_mps, params->nfeatures);
        return nullptr;
    }
    se2gpu_loc* h = new se2gpu_loc;
    h->device = device; h->S = max_streams; h->C = params->nfeatures; h->Q = params->max_local_mps; h->max_w = max_w; h->max_h = max_h;
    h->p = *params;
    h->st.resize(max_streams);
    const int K = map->n_kf, M = map->n_mp;
    h->kf_Tcw.assign(map->kf_Tcw, map->kf_Tcw + 16 * (size_t)K);
    h->kf_nkp.resize(K);
    for (int k = 0; k < K; k++) h->kf_nkp[k] = map->kf_kp_ptr[k + 1] - map->kf_kp_ptr[k];
    auto bad = [&](const char* what) { fail(SE2GPU_ERR_CUDA, "localizer: %s", what); delete h; return (se2gpu_loc*)nullptr; };
    h->orb = se2gpu_orb_create(params->nfeatures, params->scale_factor, params->nlevels, params->fast_th, max_w, max_h, max_streams, device);
    if (!h->orb) { delete h; return nullptr; }
    if (se2gpu_orb_set_undistort(h->orb, params->ndist ? params->K : nullptr, params->dist, params->ndist) != SE2GPU_OK) { delete h; return nullptr; }
    h->matcher = se2gpu_matcher_create_batch(h->Q, h->C, max_streams, device);
    if (!h->matcher) { delete h; return nullptr; }
    const size_t S = max_streams, C = h->C, Q = h->Q, Kn = std::max(K, 1), Mn = std::max(M, 1);
    const size_t nkp = std::max(map->kf_kp_ptr[K], 1), nobs = std::max(map->kf_obs_ptr[K], 1), ncov = std::max(map->kf_cov_ptr[K], 1);
    bool ok = true;
    auto A = [&](auto** p, size_t count) { ok = ok && h->bufs.alloc(p, count) == cudaSuccess; };
    int *kp_ptr, *kf_obs_mp, *obs_ptr, *obs, *cov_ptr, *cov, *mp_oct;
    float* mp_pos;
    uint8_t *mp_use, *mp_null, *mp_desc;
    A(&kp_ptr, Kn + 1); A(&kf_obs_mp, nkp); A(&obs_ptr, Kn + 1); A(&obs, nobs); A(&cov_ptr, Kn + 1); A(&cov, ncov);
    A(&mp_oct, Mn); A(&mp_pos, 3 * Mn); A(&mp_use, Mn); A(&mp_null, Mn); A(&mp_desc, 32 * Mn);
    A(&h->d_frames, S * max_w * max_h);
    A(&h->d_kp, S * C); A(&h->d_desc, S * C * 32); A(&h->d_kf_obsd, S * C); A(&h->d_obs_mp, S * C); A(&h->d_matches, S * C);
    A(&h->d_has_mp, S * Mn); A(&h->d_mark, S * Mn); A(&h->d_best, S * Mn);
    A(&h->d_kf_cov, S * Kn); A(&h->d_kf_local, S * Kn); A(&h->d_kf_tmp, S * Kn);
    A(&h->d_local, S * Q); A(&h->d_valid, S * Q); A(&h->d_uv, 2 * S * Q); A(&h->d_oct, S * Q); A(&h->d_mpdesc, 32 * S * Q);
    A(&h->d_exyz, 3 * S * C); A(&h->d_euv, 2 * S * C); A(&h->d_ew, S * C); A(&h->d_K, 9); A(&h->d_isig, 16);
    A(&h->d_pairs, 3 * S * C); A(&h->d_io, h->io_words());
    if (!ok) return bad("device allocation failed");
    ok = h->pin.reserve(sizeof(uint32_t) * h->io_words() + sizeof(int) * 3 * S * C + 2 * 64);
    if (ok) {
        h->h_io = h->pin.alloc<uint32_t>(h->io_words());
        h->h_pairs = h->pin.alloc<int>(3 * S * C);
        ok = h->h_io && h->h_pairs;
    }
    if (!ok) return bad("page-locked allocation failed");
    std::memset(h->h_io, 0, sizeof(uint32_t) * h->io_words());
    std::vector<uint8_t> use(Mn, 0);
    for (int j = 0; j < M; j++) use[j] = !map->mp_null[j] && map->mp_good_prl[j];
    if (cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking) != cudaSuccess) return bad("stream creation failed");
    auto up = [&](void* d, const void* src, size_t bytes) {
        ok = ok && (!bytes || cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, h->s) == cudaSuccess);
    };
    up(kp_ptr, map->kf_kp_ptr, sizeof(int) * (K + 1)); up(kf_obs_mp, map->kf_obs_mp, sizeof(int) * map->kf_kp_ptr[K]);
    up(obs_ptr, map->kf_obs_ptr, sizeof(int) * (K + 1)); up(obs, map->kf_obs, sizeof(int) * map->kf_obs_ptr[K]);
    up(cov_ptr, map->kf_cov_ptr, sizeof(int) * (K + 1)); up(cov, map->kf_cov, sizeof(int) * map->kf_cov_ptr[K]);
    up(mp_oct, map->mp_octave, sizeof(int) * M); up(mp_pos, map->mp_pos, sizeof(float) * 3 * M); up(mp_use, use.data(), M);
    up(mp_null, map->mp_null, M); up(mp_desc, map->mp_desc, 32 * (size_t)M);
    up(h->d_K, params->K, sizeof(float) * 9); up(h->d_isig, params->inv_level_sigma2, sizeof(float) * 16);
    // every array a stream's state exposes is defined from here on
    ok = ok && cudaMemsetAsync(h->d_io, 0, sizeof(uint32_t) * h->io_words(), h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_kp, 0, sizeof(se2gpu_keypoint) * S * C, h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_desc, 0, 32 * S * C, h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_obs_mp, 0xff, sizeof(int) * S * C, h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_kf_obsd, 0, S * C, h->s) == cudaSuccess && cudaMemsetAsync(h->d_has_mp, 0, S * Mn, h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_kf_cov, 0, S * Kn, h->s) == cudaSuccess && cudaMemsetAsync(h->d_kf_local, 0, S * Kn, h->s) == cudaSuccess &&
         cudaMemsetAsync(h->d_local, 0xff, sizeof(int) * S * Q, h->s) == cudaSuccess && cudaStreamSynchronize(h->s) == cudaSuccess;
    if (!ok) return bad("initialisation failed");
    h->map.K = K; h->map.M = M; h->map.kp_ptr = kp_ptr; h->map.kf_obs_mp = kf_obs_mp; h->map.obs_ptr = obs_ptr; h->map.obs = obs;
    h->map.cov_ptr = cov_ptr; h->map.cov = cov; h->map.mp_oct = mp_oct; h->map.mp_pos = mp_pos; h->map.mp_use = mp_use;
    h->map.mp_null = mp_null; h->map.mp_desc = mp_desc;
    return h;
}

void se2gpu_loc_destroy(se2gpu_loc* h) { delete h; }

int se2gpu_loc_step(se2gpu_loc* h, int B, const uint8_t* frames, int on_device, int w, int hgt, int stride, size_t frame_stride,
                    const float* odom, se2gpu_loc_result* out) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (B <= 0) return fail(SE2GPU_ERR_INVALID, "%d streams", B);
    if (B > h->S) return fail(SE2GPU_ERR_CAPACITY, "%d streams exceed the handle's %d", B, h->S);
    if (!frames || !odom || !out) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (w <= 0 || hgt <= 0 || stride < w) return fail(SE2GPU_ERR_INVALID, "bad frame geometry %dx%d, stride %d", w, hgt, stride);
    if (w > h->max_w || hgt > h->max_h) return fail(SE2GPU_ERR_CAPACITY, "frame %dx%d exceeds %dx%d", w, hgt, h->max_w, h->max_h);
    if (B > 1 && frame_stride < (size_t)stride * (hgt - 1) + w) return fail(SE2GPU_ERR_INVALID, "frames overlap");
    for (int b = 0; b < B; b++)
        if (h->st[b].overflow) return fail(SE2GPU_ERR_CAPACITY, "stream %d: its local map exceeded %d map points", b, h->Q);
    SE2_CUDA(cudaSetDevice(h->device));
    SE2_NVTX("se2gpu.loc.step");
    // ReadFrameInfo's Tcw = cTb for a first frame, UpdatePoseCurr for the others; mode = mbIsTracked
    float* T = h->Tcw(h->h_io);
    int* mode = h->mode(h->h_io);
    std::vector<float> pose(16 * (size_t)B);
    for (int b = 0; b < B; b++) {
        const StreamState& ss = h->st[b];
        if (ss.has_frame) host_pose(h->p, odo3(odom + 3 * b), ss.odom, ss.Tcw, &pose[16 * b]);
        else std::memcpy(&pose[16 * b], h->p.cTb, 16 * sizeof(float));
        mode[b] = ss.has_frame && ss.tracked;
    }
    for (int b = 0; b < h->S; b++) if (b >= B) mode[b] = 0;
    std::memcpy(T, pose.data(), sizeof(float) * 16 * B);
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (frame_stride == (size_t)stride * hgt)
        SE2_CUDA(cudaMemcpy2DAsync(h->d_frames, w, frames, stride, w, (size_t)hgt * B, kind, h->s));
    else
        for (int b = 0; b < B; b++)
            SE2_CUDA(cudaMemcpy2DAsync(h->d_frames + (size_t)b * w * hgt, w, frames + b * frame_stride, stride, w, hgt, kind, h->s));
    if (h->eager) {
        if (int rc = orb_prepare_shape(h->orb, w, hgt, h->s)) return rc;
        if (int rc = enqueue_step(h, B, w, hgt)) return rc;
    } else {
        if (int rc = ensure_graph(h, B, w, hgt)) return rc;
        SE2_CUDA(cudaGraphLaunch(h->exec, h->s));
        ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    SE2_CUDA(cudaStreamSynchronize(h->s));
    for (int b = 0; b < B; b++) {
        StreamState& ss = h->st[b];
        const bool ran = mode[b] != 0;
        ss.first = !ss.has_frame;
        ss.lost_branch = ss.has_frame && !ran;
        if (!ran) std::memcpy(ss.Tcw, &pose[16 * b], sizeof ss.Tcw);
        fill_result(h, b, ran, out[b]);
        ss.has_frame = true;
        ss.odom = odo3(odom + 3 * b);
    }
    return SE2GPU_OK;
}

int se2gpu_loc_relocalize(se2gpu_loc* h, int n, const int* streams, const int* kf_loop, const int* match_ptr, const int* match_curr,
                          const int* match_loop, se2gpu_loc_result* out, float* Tcw_first) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (n < 0 || (n && (!streams || !kf_loop || !match_ptr || !out))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n == 0) return SE2GPU_OK;
    if (match_ptr[0] != 0) return fail(SE2GPU_ERR_INVALID, "match_ptr[0] must be 0");
    std::vector<uint8_t> seen(h->S, 0);
    int Bm = 0;
    for (int j = 0; j < n; j++) {
        const int b = streams[j];
        if (b < 0 || b >= h->S) return fail(SE2GPU_ERR_INVALID, "stream %d out of range", b);
        if (seen[b]++) return fail(SE2GPU_ERR_INVALID, "stream %d listed twice", b);
        const StreamState& ss = h->st[b];
        if (ss.overflow) return fail(SE2GPU_ERR_CAPACITY, "stream %d: its local map exceeded %d map points", b, h->Q);
        // DetectLoopClose runs only in the else branch: a stream that was tracked when its last step began waits a frame
        if (!ss.lost_branch || ss.tracked)
            return fail(SE2GPU_ERR_INVALID, "stream %d: its last step did not begin lost (or it relocalized already)", b);
        if (kf_loop[j] < 0 || kf_loop[j] >= h->map.K) return fail(SE2GPU_ERR_INVALID, "keyframe %d out of range", kf_loop[j]);
        if (match_ptr[j + 1] < match_ptr[j] || match_ptr[j + 1] - match_ptr[j] > h->C) return fail(SE2GPU_ERR_INVALID, "bad match_ptr at %d", j);
        const int nk = h->rec(h->h_io, R_KP)[b];
        for (int e = match_ptr[j]; e < match_ptr[j + 1]; e++) {
            if (!match_curr || !match_loop) return fail(SE2GPU_ERR_INVALID, "null match arrays");
            if (match_curr[e] < 0 || match_curr[e] >= nk || (e > match_ptr[j] && match_curr[e] <= match_curr[e - 1]))
                return fail(SE2GPU_ERR_INVALID, "stream %d: idxCurr %d out of range or not ascending", b, match_curr[e]);
            if (match_loop[e] < 0 || match_loop[e] >= h->kf_nkp[kf_loop[j]])
                return fail(SE2GPU_ERR_INVALID, "stream %d: idxLoop %d out of range", b, match_loop[e]);
        }
        Bm = std::max(Bm, b + 1);
    }
    SE2_CUDA(cudaSetDevice(h->device));
    SE2_NVTX("se2gpu.loc.relocalize");
    SE2_CUDA(cudaStreamSynchronize(h->s));
    // setPose(kfLoop->getPose()) and the streams to run; the record of the other streams is kept
    std::vector<uint32_t> keep(h->io_words());
    std::memcpy(keep.data(), h->h_io, sizeof(uint32_t) * h->io_words());
    int* mode = h->mode(h->h_io);
    int* aux = h->aux(h->h_io);
    for (int b = 0; b < h->S; b++) {
        mode[b] = 0;
        std::memcpy(h->Tcw(h->h_io) + 16 * b, h->st[b].Tcw, sizeof(float) * 16);
    }
    int np = 0;
    for (int j = 0; j < n; j++) {
        const int b = streams[j];
        mode[b] = 1; aux[b] = kf_loop[j];
        std::memcpy(h->Tcw(h->h_io) + 16 * b, &h->kf_Tcw[16 * (size_t)kf_loop[j]], sizeof(float) * 16);
        for (int e = match_ptr[j]; e < match_ptr[j + 1]; e++, np++) {
            h->h_pairs[3 * np] = b; h->h_pairs[3 * np + 1] = match_curr[e]; h->h_pairs[3 * np + 2] = match_loop[e];
        }
    }
    cudaStream_t s = h->s;
    SE2_CUDA(cudaMemcpyAsync(h->d_io, h->h_io, sizeof(uint32_t) * h->up_words(), cudaMemcpyHostToDevice, s));
    if (np) SE2_CUDA(cudaMemcpyAsync(h->d_pairs, h->h_pairs, sizeof(int) * 3 * np, cudaMemcpyHostToDevice, s));
    SE2_LAUNCH(k_loc_seed, dim3((h->map.K + kBlock - 1) / kBlock, Bm), kBlock, 0, s, h->map.K, h->mode(h->d_io), h->aux(h->d_io), h->d_kf_cov);
    SE2_CUDA(cudaGetLastError());
    if (int rc = enqueue_local_map(h, Bm, 3)) return rc;
    if (np) {
        SE2_LAUNCH(k_loc_loop_close, (np + kBlock - 1) / kBlock, kBlock, 0, s, h->map, np, h->d_pairs, h->aux(h->d_io), h->C, h->d_obs_mp,
                   h->d_kf_obsd, h->d_has_mp);
        SE2_CUDA(cudaGetLastError());
    }
    if (int rc = enqueue_ba(h, Bm, -1)) return rc;
    std::vector<float> first(16 * (size_t)Bm);
    SE2_CUDA(cudaMemcpyAsync(h->h_io, h->d_io, sizeof(uint32_t) * h->io_words(), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    std::memcpy(first.data(), h->Tcw(h->h_io), sizeof(float) * first.size());
    if (int rc = enqueue_match(h, Bm)) return rc;
    if (int rc = enqueue_ba(h, Bm, -1)) return rc;
    SE2_CUDA(cudaMemcpyAsync(h->h_io, h->d_io, sizeof(uint32_t) * h->io_words(), cudaMemcpyDeviceToHost, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    int rc = SE2GPU_OK;
    for (int j = 0; j < n; j++) {
        const int b = streams[j];
        fill_result(h, b, true, out[j]);
        if (Tcw_first) std::memcpy(Tcw_first + 16 * j, &first[16 * b], sizeof(float) * 16);
        if (out[j].overflow) rc = fail(SE2GPU_ERR_CAPACITY, "stream %d: its local map has %d map points, more than %d", b, out[j].n_local_mps, h->Q);
    }
    // the host copy of the record stays that of the last step for the streams that did not run
    for (int b = 0; b < h->S; b++)
        if (!seen[b])
            for (int f = 0; f < kRec; f++) h->rec(h->h_io, f)[b] = reinterpret_cast<int*>(keep.data() + (18 + (size_t)f) * h->S)[b];
    return rc;
}

int se2gpu_loc_state(se2gpu_loc* h, int b, se2gpu_loc_stream_state* out) {
    if (!h || !out) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (b < 0 || b >= h->S) return fail(SE2GPU_ERR_INVALID, "stream %d out of range", b);
    SE2_CUDA(cudaSetDevice(h->device));
    SE2_CUDA(cudaStreamSynchronize(h->s));
    const size_t C = h->C, k = (size_t)b * C;
    out->d_kp = h->d_kp + k; out->d_desc = h->d_desc + 32 * k; out->d_n = h->rec(h->d_io, R_KP) + b;
    out->d_obs_mp = h->d_obs_mp + k;
    out->d_local_mps = h->d_local + (size_t)b * h->Q; out->d_n_local_mps = h->rec(h->d_io, R_NMP) + b;
    out->d_local_kfs = h->d_kf_local + (size_t)b * std::max(h->map.K, 1); out->d_covis_kfs = h->d_kf_cov + (size_t)b * std::max(h->map.K, 1);
    const StreamState& ss = h->st[b];
    std::memcpy(out->Tcw, ss.Tcw, sizeof ss.Tcw);
    out->has_frame = ss.has_frame; out->tracked = ss.tracked; out->overflow = ss.overflow;
    return SE2GPU_OK;
}

int se2gpu_loc_graph_nodes(se2gpu_loc* h, int* kernels, int* nodes) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (kernels) *kernels = h->g_kernels;
    if (nodes) *nodes = h->g_nodes;
    return SE2GPU_OK;
}

int se2gpu_loc_debug_eager(se2gpu_loc* h, int eager) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    h->eager = eager != 0;
    return SE2GPU_OK;
}

int se2gpu_loc_host_pose(const se2gpu_loc_params* p, const float* odom, const float* ref_odom, const float* ref_Tcw, float* Tcw) {
    if (!p || !odom || !ref_odom || !ref_Tcw || !Tcw) return fail(SE2GPU_ERR_INVALID, "null argument");
    host_pose(*p, odo3(odom), odo3(ref_odom), ref_Tcw, Tcw);
    return SE2GPU_OK;
}

}  // extern "C"
