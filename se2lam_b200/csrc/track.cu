// Track::mTrack (reference src/Track.cpp:105-204, :346-376) for a batch of camera streams with the tracking state kept on the
// device (DESIGN.md section 14). The device part of a step (extraction, MatchByWindow, removeOutliers, doTriangulate and
// the counts record) is one CUDA graph per (B, w, h); updateFramePose, the pre-integration and needNewKF run here on the
// host in the reference's float / double arithmetic, so Tcr and the decisions are those of glibc's cosf / sinf.
#include <cmath>

#include "common.h"
#include "se2_host.h"

using namespace se2gpu;

namespace {

constexpr int kBlock = 256;
constexpr int kRecFields = 5;          // counts record: nMatched [S], nInlier [S], {nTrackedOld, nGoodPrl} [2S], N [S]

// ------------------------------------------------------------------------------------------ host part (float / double)
// Eigen's coefficient-based 3x3 product: coefficient (i, j) is the unrolled sum x0 + (x1 + x2)
void mul3(const double* A, const double* B, double* C, bool bt) {   // column-major, C = A * (bt ? B^T : B)
    double R[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double x[3];
            for (int k = 0; k < 3; k++) x[k] = A[i + 3 * k] * (bt ? B[j + 3 * k] : B[k + 3 * j]);
            R[i + 3 * j] = x[0] + (x[1] + x[2]);
        }
    std::memcpy(C, R, sizeof R);
}

// updateFramePose (src/Track.cpp:162-188): Tcr and the pre-integration of preSE2
void host_pose(const se2gpu_tracker_params& p, const Se2& odom, const Se2& kf_odom, const Se2& last, float* Tcr, double* meas,
               double* cov) {
    cam_motion(p.cTb, p.bTc, se2_minus(kf_odom, odom), Tcr);
    const Se2 odok = se2_minus(odom, last);
    const double ox = odok.x, oy = odok.y;
    const double c = std::cos(meas[2]), s = std::sin(meas[2]);   // Rotation2Dd(meas[2]).toRotationMatrix()
    const double Phi[4] = {c, -s, s, c};                          // row-major 2x2
    meas[0] += Phi[0] * ox + Phi[1] * oy;
    meas[1] += Phi[2] * ox + Phi[3] * oy;
    meas[2] += odok.theta;
    double A[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Bk[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, V[9] = {0};   // column-major
    A[6] = Phi[0] * -oy + Phi[1] * ox;
    A[7] = Phi[2] * -oy + Phi[3] * ox;
    Bk[0] = Phi[0]; Bk[3] = Phi[1]; Bk[1] = Phi[2]; Bk[4] = Phi[3];
    for (int k = 0; k < 3; k++) V[4 * k] = p.odo_noise[k] * p.odo_noise[k];
    double t1[9], t2[9], P1[9], P2[9];
    mul3(A, cov, t1, false); mul3(t1, A, P1, true);
    mul3(Bk, V, t2, false); mul3(t2, Bk, P2, true);
    for (int k = 0; k < 9; k++) cov[k] = P1[k] + P2[k];
}

// needNewKF (src/Track.cpp:346-376) with mbUseOdometry
void host_decide(const se2gpu_tracker_params& p, int dframes, int n_tracked_old, int n_old_kp, int n_good_prl, int n_matched,
                 const Se2& odom, const Se2& kf_odom, bool accept, int* new_kf, int* abort_ba) {
    const bool c0 = dframes > p.min_frames;
    const bool c1 = (float)n_tracked_old <= (float)n_old_kp * 0.5f;
    const bool c2 = n_good_prl > 40;
    const bool c3 = dframes > p.max_frames;
    const bool c4 = n_matched < 0.1f * p.nfeatures || n_matched < 20;
    bool need = c0 && ((c1 && c2) || c3 || c4);
    const Se2 d = se2_minus(odom, kf_odom);
    const bool c5 = std::fabs(d.theta) >= 0.0349f;
    float cTc[16];
    cam_motion(p.cTb, p.bTc, se2(d.x, d.y, d.theta), cTc);
    double sq = 0;                                                 // cv::norm of the 3x1 float translation
    for (int k = 0; k < 3; k++) sq += (double)cTc[4 * k + 3] * (double)cTc[4 * k + 3];
    const bool c6 = std::sqrt(sq) >= (0.0523f * p.upper_depth * 0.1f);
    const bool by_odo = c5 || c6;
    need = need && by_odo;
    *new_kf = accept ? need : 0;
    *abort_ba = !accept && c0 && (c4 || c3) && by_odo;
}

bool params_ok(const se2gpu_tracker_params* p) {
    if (!p || p->nfeatures <= 0 || p->nlevels <= 0 || !(p->scale_factor > 1.f) || p->min_frames < 0 || p->max_frames < 0) return false;
    return p->ndist == 0 || p->ndist == 4 || p->ndist == 5 || p->ndist == 8 || p->ndist == 12;
}

// ------------------------------------------------------------------------------------------ device part
// per-step inputs, one page-locked copy: Tcr, the nMinFrames gate and the keyframe arrays of every stream
struct StepPar {
    float* Tcr; int* gate; const uint8_t** observed; const float** view_mp;
};
size_t step_par_bytes(int S) { return (size_t)S * (16 * sizeof(float) + sizeof(int) + 2 * sizeof(void*)); }
StepPar step_par(void* base, int S) {
    uint8_t* b = (uint8_t*)base;
    StepPar p;
    p.observed = (const uint8_t**)b; p.view_mp = (const float**)(b + S * sizeof(void*));
    p.Tcr = (float*)(b + 2 * S * sizeof(void*)); p.gate = (int*)(p.Tcr + 16 * (size_t)S);
    return p;
}

// resetLocalTrack for the streams list[0 .. n-1] (blockIdx.y): the current frame becomes the reference frame, mPrevMatched
// its keypoints, mLocalMPs the keyframe's mViewMPs up to its count and (-1,-1,-1) past it (Track.cpp:28), mMatchIdx -1
__global__ void __launch_bounds__(kBlock) k_track_reset(const int* __restrict__ list, const float* const* __restrict__ view_mp, int cap,
                                                        const se2gpu_keypoint* __restrict__ cur_kp, const uint4* __restrict__ cur_desc,
                                                        const int* __restrict__ cur_n, se2gpu_keypoint* __restrict__ ref_kp,
                                                        uint4* __restrict__ ref_desc, int* __restrict__ ref_n, float* __restrict__ prev,
                                                        float* __restrict__ local_mps, int* __restrict__ matches) {
    const int b = list[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = count_of(cur_n + b, cap);
    if (i == 0) ref_n[b] = n;
    if (i >= cap) return;
    const size_t k = (size_t)b * cap + i;
    matches[k] = -1;
    if (i < n) {
        const se2gpu_keypoint kp = cur_kp[k];
        ref_kp[k] = kp;
        ref_desc[2 * k] = cur_desc[2 * k]; ref_desc[2 * k + 1] = cur_desc[2 * k + 1];
        prev[2 * k] = kp.x; prev[2 * k + 1] = kp.y;
        const float* v = view_mp[blockIdx.y];
        local_mps[3 * k] = v[3 * i]; local_mps[3 * k + 1] = v[3 * i + 1]; local_mps[3 * k + 2] = v[3 * i + 2];
    } else {
        local_mps[3 * k] = -1.f; local_mps[3 * k + 1] = -1.f; local_mps[3 * k + 2] = -1.f;
    }
}

// mLocalMPs as Track::Track makes it (Track.cpp:28): MaxFtrNumber entries of (-1,-1,-1)
__global__ void __launch_bounds__(kBlock) k_fill(float* __restrict__ p, size_t n, float v) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

struct StreamState {
    int next_id = 0;          // Frame::nextId of this stream
    int frame_id = -1;        // mFrame.id, -1 before the first frame
    int kf_id = 0;            // mpKF->id
    bool has_ref = false;
    Se2 last_odom{0, 0, 0};   // lastOdom
    float Tcr[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    double meas[3] = {0, 0, 0}, cov[9] = {0};
    int n_good_prl = 0;
};

}  // namespace

struct se2gpu_tracker {
    int device = 0, S = 0, cap = 0, max_w = 0, max_h = 0;
    se2gpu_tracker_params p{};
    se2gpu_orb* orb = nullptr;
    se2gpu_matcher* matcher = nullptr;
    cudaStream_t s = nullptr;
    cudaEvent_t ev_reset = nullptr;
    DeviceBuffers bufs;
    uint8_t* d_frames = nullptr;
    se2gpu_keypoint *d_ref_kp = nullptr, *d_cur_kp = nullptr;
    uint8_t *d_ref_desc = nullptr, *d_cur_desc = nullptr;
    int *d_ref_n = nullptr, *d_rec = nullptr, *d_matches = nullptr;
    float *d_prev = nullptr, *d_local = nullptr, *d_K = nullptr;
    uint8_t* d_good = nullptr;
    void* d_par = nullptr;
    int* d_reset_list = nullptr;
    const float** d_reset_vmp = nullptr;
    PinnedArena pin;
    void* h_par = nullptr;
    int* h_rec = nullptr;
    int* h_reset_list = nullptr;
    const float** h_reset_vmp = nullptr;
    cudaGraphExec_t exec = nullptr;
    int gB = 0, gw = 0, gh = 0, g_kernels = 0, g_nodes = 0;
    bool eager = false;
    std::vector<StreamState> st;

    ~se2gpu_tracker() {
        if (device >= 0) cudaSetDevice(device);
        if (exec) cudaGraphExecDestroy(exec);
        if (ev_reset) cudaEventDestroy(ev_reset);
        if (s) cudaStreamDestroy(s);
        se2gpu_matcher_destroy(matcher);
        se2gpu_orb_destroy(orb);
    }
};

namespace {

// the device work of one step for streams 0 .. B-1 on t->s, capturable: the frames are already in t->d_frames and the
// per-step inputs in t->h_par
int enqueue_step(se2gpu_tracker* t, int B, int w, int hgt) {
    const int S = t->S, cap = t->cap;
    cudaStream_t s = t->s;
    int* rec_n = t->d_rec + 4 * S;
    SE2_CUDA(cudaMemcpyAsync(t->d_par, t->h_par, step_par_bytes(S), cudaMemcpyHostToDevice, s));
    int rc = se2gpu_orb_extract_device(t->orb, t->d_frames, B, w, hgt, w, (size_t)w * hgt, t->d_cur_kp, t->d_cur_desc, rec_n, s);
    if (rc) return rc;
    const se2gpu_grid_params& g = t->p.grid;
    rc = se2gpu_match_by_window_batch_device(t->matcher, B, t->d_ref_kp, t->d_ref_desc, cap, t->d_ref_n, t->d_cur_kp, t->d_cur_desc, cap,
                                             rec_n, t->d_prev, g, 20, 1, 0, 8, 0.9f, t->d_matches, t->d_rec, s);
    if (rc) return rc;
    rc = se2gpu_remove_outliers_device(B, t->d_ref_kp, t->d_ref_n, cap, t->d_cur_kp, rec_n, cap, t->d_matches, t->d_rec + S, nullptr,
                                       nullptr, s);
    if (rc) return rc;
    const StepPar dp = step_par(t->d_par, S);
    TrackTriArgs a{};
    a.kp_kf = t->d_ref_kp; a.cap = cap; a.d_n = t->d_ref_n; a.kp_fr = t->d_cur_kp; a.cap_fr = cap; a.matches = t->d_matches;
    a.observed_tab = dp.observed; a.view_mp_tab = dp.view_mp; a.Tcr = dp.Tcr; a.gate = dp.gate; a.K = t->d_K;
    a.lower = t->p.lower_depth; a.upper = t->p.upper_depth; a.min_cos = track_min_cos(2);
    a.local_mps = t->d_local; a.good_prl = t->d_good; a.counts = t->d_rec + 2 * S;
    rc = track_triangulate_launch(a, B, s);
    if (rc) return rc;
    SE2_CUDA(cudaMemcpyAsync(t->h_rec, t->d_rec, sizeof(int) * kRecFields * S, cudaMemcpyDeviceToHost, s));
    return SE2GPU_OK;
}

// a graph for (B, w, hgt): the set-up that cannot be captured runs first, then one capture of enqueue_step
int ensure_graph(se2gpu_tracker* t, int B, int w, int hgt) {
    if (t->exec && t->gB == B && t->gw == w && t->gh == hgt) return SE2GPU_OK;
    if (int rc = orb_prepare_shape(t->orb, w, hgt, t->s)) return rc;
    if (int rc = fundam_prepare()) return rc;
    SE2_CUDA(cudaStreamSynchronize(t->s));
    if (t->exec) { cudaGraphExecDestroy(t->exec); t->exec = nullptr; }
    t->gB = t->gw = t->gh = 0;
    SE2_CUDA(cudaStreamBeginCapture(t->s, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue_step(t, B, w, hgt);
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(t->s, &graph);
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
    const cudaError_t ei = cudaGraphInstantiate(&t->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ei != cudaSuccess) { t->exec = nullptr; return fail(SE2GPU_ERR_CUDA, "instantiating the step graph failed: %s", cudaGetErrorString(ei)); }
    t->gB = B; t->gw = w; t->gh = hgt; t->g_kernels = kernels; t->g_nodes = (int)n;
    return SE2GPU_OK;
}

// Se2(x, y, theta), as Track::run builds the odometry reading (the angle normalised)
Se2 odo3(const float* o) { return se2(o[0], o[1], o[2]); }

int run_step(se2gpu_tracker* t, int B, const uint8_t* frames, int on_device, int w, int hgt, int stride, size_t frame_stride,
             const float* odom, const se2gpu_track_kf* kf, se2gpu_track_result* out, bool first) {
    if (!t) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (B <= 0) return fail(SE2GPU_ERR_INVALID, "%d streams", B);
    if (B > t->S) return fail(SE2GPU_ERR_CAPACITY, "%d streams exceed the tracker's %d", B, t->S);
    if (!frames || !odom || !out) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (w <= 0 || hgt <= 0 || stride < w) return fail(SE2GPU_ERR_INVALID, "bad frame geometry %dx%d, stride %d", w, hgt, stride);
    if (w > t->max_w || hgt > t->max_h) return fail(SE2GPU_ERR_CAPACITY, "frame %dx%d exceeds %dx%d", w, hgt, t->max_w, t->max_h);
    if (B > 1 && frame_stride < (size_t)stride * (hgt - 1) + w) return fail(SE2GPU_ERR_INVALID, "frames overlap");
    for (int b = 0; b < B; b++)
        if (!first && t->st[b].has_ref && (!kf || !kf[b].d_observed || !kf[b].d_view_mp))
            return fail(SE2GPU_ERR_INVALID, "stream %d tracks and needs its keyframe arrays", b);
    SE2_CUDA(cudaSetDevice(t->device));
    if (first) {                                 // streams 0 .. B-1 lose their reference frame and restart their frame ids
        for (int b = 0; b < B; b++) { t->st[b].has_ref = false; t->st[b].next_id = 0; }
        SE2_CUDA(cudaMemsetAsync(t->d_ref_n, 0, sizeof(int) * B, t->s));
    }
    SE2_NVTX("se2gpu.tracker.step");
    // the staging buffers are free: the last step and reset were waited for
    SE2_CUDA(cudaEventSynchronize(t->ev_reset));
    // updateFramePose on the host (it needs odometry only), the nMinFrames gate and the keyframe arrays
    StepPar hp = step_par(t->h_par, t->S);
    std::vector<int> fid(B);
    for (int b = 0; b < B; b++) {
        StreamState& ss = t->st[b];
        fid[b] = ss.next_id;
        hp.gate[b] = 0; hp.observed[b] = nullptr; hp.view_mp[b] = nullptr;
        if (ss.has_ref) {
            host_pose(t->p, odo3(odom + 3 * b), odo3(kf[b].odom), ss.last_odom, ss.Tcr, ss.meas, ss.cov);
            hp.gate[b] = !(fid[b] - ss.kf_id < t->p.min_frames);
            hp.observed[b] = kf[b].d_observed; hp.view_mp[b] = kf[b].d_view_mp;
        }
        std::memcpy(hp.Tcr + 16 * b, ss.Tcr, sizeof ss.Tcr);
    }
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (frame_stride == (size_t)stride * hgt)
        SE2_CUDA(cudaMemcpy2DAsync(t->d_frames, w, frames, stride, w, (size_t)hgt * B, kind, t->s));
    else
        for (int b = 0; b < B; b++)
            SE2_CUDA(cudaMemcpy2DAsync(t->d_frames + (size_t)b * w * hgt, w, frames + b * frame_stride, stride, w, hgt, kind, t->s));
    if (t->eager) {
        if (int rc = orb_prepare_shape(t->orb, w, hgt, t->s)) return rc;
        if (int rc = fundam_prepare()) return rc;
        if (int rc = enqueue_step(t, B, w, hgt)) return rc;
    } else {
        if (int rc = ensure_graph(t, B, w, hgt)) return rc;
        SE2_CUDA(cudaGraphLaunch(t->exec, t->s));
        ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    SE2_CUDA(cudaStreamSynchronize(t->s));
    const int S = t->S;
    for (int b = 0; b < B; b++) {
        StreamState& ss = t->st[b];
        se2gpu_track_result& r = out[b];
        std::memset(&r, 0, sizeof r);
        r.frame_id = fid[b];
        ss.frame_id = fid[b];
        ss.next_id = fid[b] + 1;
        r.n_keypoints = t->h_rec[4 * S + b];
        if (!ss.has_ref) {                       // mCreateFrame (Track.cpp:105-120)
            r.first = 1;
            r.new_kf = r.n_keypoints > 100;
            if (!r.new_kf) ss.next_id = 0;       // Frame::nextId = 0
        } else {
            r.n_matched = t->h_rec[b];
            r.n_inlier = t->h_rec[S + b];
            r.triangulated = hp.gate[b];
            if (hp.gate[b]) {
                r.n_tracked_old = t->h_rec[2 * S + 2 * b];
                ss.n_good_prl = t->h_rec[2 * S + 2 * b + 1];
            }
            r.n_good_prl = ss.n_good_prl;
            host_decide(t->p, fid[b] - ss.kf_id, r.n_tracked_old, kf[b].n_obs_mp, ss.n_good_prl, r.n_inlier, odo3(odom + 3 * b),
                        odo3(kf[b].odom), kf[b].accept_new_kf != 0, &r.new_kf, &r.abort_ba);
        }
        ss.last_odom = odo3(odom + 3 * b);       // lastOdom = odo
    }
    return SE2GPU_OK;
}

}  // namespace

extern "C" {

se2gpu_tracker* se2gpu_tracker_create(int max_streams, int max_w, int max_h, const se2gpu_tracker_params* params, int device) {
    if (max_streams <= 0 || max_w <= 0 || max_h <= 0 || !params_ok(params)) { fail(SE2GPU_ERR_INVALID, "bad arguments"); return nullptr; }
    if (max_streams > 65535) { fail(SE2GPU_ERR_CAPACITY, "%d streams: at most 65535", max_streams); return nullptr; }
    if (select_device(device) != SE2GPU_OK) return nullptr;
    if (!matcher_window_capturable(device, params->nfeatures, params->nfeatures)) {
        fail(SE2GPU_ERR_CAPACITY, "%d features per frame are too many for the matcher's shared-memory resolve", params->nfeatures);
        return nullptr;
    }
    se2gpu_tracker* t = new se2gpu_tracker;
    t->device = device; t->S = max_streams; t->cap = params->nfeatures; t->max_w = max_w; t->max_h = max_h; t->p = *params;
    t->st.resize(max_streams);
    auto bad = [&](const char* what) { fail(SE2GPU_ERR_CUDA, "tracker: %s", what); delete t; return (se2gpu_tracker*)nullptr; };
    t->orb = se2gpu_orb_create(params->nfeatures, params->scale_factor, params->nlevels, params->fast_th, max_w, max_h, max_streams, device);
    if (!t->orb) { delete t; return nullptr; }
    if (se2gpu_orb_set_undistort(t->orb, params->ndist ? params->K : nullptr, params->dist, params->ndist) != SE2GPU_OK) { delete t; return nullptr; }
    t->matcher = se2gpu_matcher_create_batch(params->nfeatures, params->nfeatures, max_streams, device);
    if (!t->matcher) { delete t; return nullptr; }
    const size_t S = max_streams, C = t->cap;
    bool ok = true;
    auto A = [&](auto** p, size_t count) { ok = ok && t->bufs.alloc(p, count) == cudaSuccess; };
    A(&t->d_frames, S * max_w * max_h);
    A(&t->d_ref_kp, S * C); A(&t->d_cur_kp, S * C); A(&t->d_ref_desc, S * C * 32); A(&t->d_cur_desc, S * C * 32);
    A(&t->d_ref_n, S); A(&t->d_rec, kRecFields * S); A(&t->d_matches, S * C); A(&t->d_prev, 2 * S * C);
    A(&t->d_local, 3 * S * C); A(&t->d_good, S * C); A(&t->d_K, 9);
    uint8_t* par = nullptr;
    A(&par, step_par_bytes(max_streams)); t->d_par = par;
    A(&t->d_reset_list, S);
    uint8_t* rv = nullptr;
    A(&rv, S * sizeof(void*)); t->d_reset_vmp = (const float**)rv;
    if (!ok) return bad("device allocation failed");
    ok = t->pin.reserve(step_par_bytes(max_streams) + S * (kRecFields * sizeof(int) + sizeof(int) + sizeof(void*)) + 4 * 64);
    if (ok) {
        t->h_par = t->pin.alloc<uint8_t>(step_par_bytes(max_streams));
        t->h_rec = t->pin.alloc<int>(kRecFields * S);
        t->h_reset_list = t->pin.alloc<int>(S);
        t->h_reset_vmp = (const float**)t->pin.alloc<void*>(S);
        ok = t->h_par && t->h_rec && t->h_reset_list && t->h_reset_vmp;
    }
    if (!ok) return bad("page-locked allocation failed");
    std::memset(t->h_par, 0, step_par_bytes(max_streams));
    if (cudaStreamCreateWithFlags(&t->s, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&t->ev_reset, cudaEventDisableTiming) != cudaSuccess)
        return bad("stream creation failed");
    // no reference frame anywhere: MatchByWindow and removeOutliers see empty reference frames. Every array a stream's
    // state exposes is defined from here on, whatever the allocation held before.
    k_fill<<<(unsigned)std::min<size_t>((3 * S * C + kBlock - 1) / kBlock, 4096), kBlock, 0, t->s>>>(t->d_local, 3 * S * C, -1.f);
    ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    ok = cudaGetLastError() == cudaSuccess &&
         cudaMemsetAsync(t->d_ref_n, 0, sizeof(int) * S, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_ref_kp, 0, sizeof(se2gpu_keypoint) * S * C, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_ref_desc, 0, 32 * S * C, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_prev, 0, sizeof(float) * 2 * S * C, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_rec, 0, sizeof(int) * kRecFields * S, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_matches, 0xff, sizeof(int) * S * C, t->s) == cudaSuccess &&
         cudaMemsetAsync(t->d_good, 0, S * C, t->s) == cudaSuccess &&
         cudaMemcpyAsync(t->d_K, params->K, sizeof(float) * 9, cudaMemcpyHostToDevice, t->s) == cudaSuccess &&
         cudaEventRecord(t->ev_reset, t->s) == cudaSuccess && cudaStreamSynchronize(t->s) == cudaSuccess;
    if (!ok) return bad("initialisation failed");
    return t;
}

void se2gpu_tracker_destroy(se2gpu_tracker* t) { delete t; }

int se2gpu_tracker_step(se2gpu_tracker* t, int B, const uint8_t* frames, int frames_on_device, int w, int hgt, int stride,
                        size_t frame_stride, const float* odom, const se2gpu_track_kf* kf, se2gpu_track_result* out) {
    return run_step(t, B, frames, frames_on_device, w, hgt, stride, frame_stride, odom, kf, out, false);
}

int se2gpu_tracker_first(se2gpu_tracker* t, int B, const uint8_t* frames, int frames_on_device, int w, int hgt, int stride,
                         size_t frame_stride, const float* odom, se2gpu_track_result* out) {
    return run_step(t, B, frames, frames_on_device, w, hgt, stride, frame_stride, odom, nullptr, out, true);
}

int se2gpu_tracker_reset(se2gpu_tracker* t, int n, const int* streams, const float* const* d_view_mp) {
    if (!t) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (n < 0 || (n && (!streams || !d_view_mp))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n > t->S) return fail(SE2GPU_ERR_CAPACITY, "%d streams exceed the tracker's %d", n, t->S);
    std::vector<uint8_t> seen(t->S, 0);
    for (int j = 0; j < n; j++) {
        const int b = streams[j];
        if (b < 0 || b >= t->S) return fail(SE2GPU_ERR_INVALID, "stream %d out of range", b);
        if (seen[b]++) return fail(SE2GPU_ERR_INVALID, "stream %d listed twice", b);
        if (t->st[b].frame_id < 0) return fail(SE2GPU_ERR_INVALID, "stream %d has no frame to make its reference", b);
        if (!d_view_mp[j]) return fail(SE2GPU_ERR_INVALID, "null mViewMPs for stream %d", b);
    }
    if (n == 0) return SE2GPU_OK;
    SE2_CUDA(cudaSetDevice(t->device));
    SE2_CUDA(cudaEventSynchronize(t->ev_reset));           // the staging of the previous reset has been read
    std::memcpy(t->h_reset_list, streams, sizeof(int) * n);
    std::memcpy((void*)t->h_reset_vmp, d_view_mp, sizeof(void*) * n);
    SE2_CUDA(cudaMemcpyAsync(t->d_reset_list, t->h_reset_list, sizeof(int) * n, cudaMemcpyHostToDevice, t->s));
    SE2_CUDA(cudaMemcpyAsync((void*)t->d_reset_vmp, (const void*)t->h_reset_vmp, sizeof(void*) * n, cudaMemcpyHostToDevice, t->s));
    SE2_LAUNCH(k_track_reset, dim3((t->cap + kBlock - 1) / kBlock, n), kBlock, 0, t->s, t->d_reset_list, t->d_reset_vmp, t->cap,
               t->d_cur_kp, reinterpret_cast<const uint4*>(t->d_cur_desc), t->d_rec + 4 * t->S, t->d_ref_kp,
               reinterpret_cast<uint4*>(t->d_ref_desc), t->d_ref_n, t->d_prev, t->d_local, t->d_matches);
    SE2_CUDA(cudaGetLastError());
    SE2_CUDA(cudaEventRecord(t->ev_reset, t->s));
    for (int j = 0; j < n; j++) {
        StreamState& ss = t->st[streams[j]];
        ss.has_ref = true;
        ss.kf_id = ss.frame_id;
        static const float eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
        std::memcpy(ss.Tcr, eye, sizeof eye);
        std::fill(ss.meas, ss.meas + 3, 0.0);
        std::fill(ss.cov, ss.cov + 9, 0.0);
        ss.n_good_prl = 0;
    }
    return SE2GPU_OK;
}

int se2gpu_tracker_state(se2gpu_tracker* t, int b, se2gpu_track_state* out) {
    if (!t || !out) return fail(SE2GPU_ERR_INVALID, "null argument");
    if (b < 0 || b >= t->S) return fail(SE2GPU_ERR_INVALID, "stream %d out of range", b);
    SE2_CUDA(cudaSetDevice(t->device));
    SE2_CUDA(cudaStreamSynchronize(t->s));
    const size_t C = t->cap, k = (size_t)b * C;
    out->d_ref_kp = t->d_ref_kp + k; out->d_ref_desc = t->d_ref_desc + 32 * k; out->d_ref_n = t->d_ref_n + b;
    out->d_cur_kp = t->d_cur_kp + k; out->d_cur_desc = t->d_cur_desc + 32 * k; out->d_cur_n = t->d_rec + 4 * t->S + b;
    out->d_prev = t->d_prev + 2 * k; out->d_matches = t->d_matches + k; out->d_local_mps = t->d_local + 3 * k; out->d_good_prl = t->d_good + k;
    const StreamState& ss = t->st[b];
    std::memcpy(out->Tcr, ss.Tcr, sizeof ss.Tcr);
    std::memcpy(out->pre_meas, ss.meas, sizeof ss.meas);
    std::memcpy(out->pre_cov, ss.cov, sizeof ss.cov);
    out->frame_id = ss.frame_id; out->kf_id = ss.kf_id; out->has_ref = ss.has_ref; out->n_good_prl = ss.n_good_prl;
    return SE2GPU_OK;
}

int se2gpu_tracker_graph_nodes(se2gpu_tracker* t, int* kernels, int* nodes) {
    if (!t) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (kernels) *kernels = t->g_kernels;
    if (nodes) *nodes = t->g_nodes;
    return SE2GPU_OK;
}

int se2gpu_tracker_debug_eager(se2gpu_tracker* t, int eager) {
    if (!t) return fail(SE2GPU_ERR_INVALID, "null handle");
    t->eager = eager != 0;
    return SE2GPU_OK;
}

int se2gpu_track_host_pose(const se2gpu_tracker_params* p, const float* odom, const float* kf_odom, const float* last_odom,
                           float* Tcr, double* meas, double* cov) {
    if (!p || !odom || !kf_odom || !last_odom || !Tcr || !meas || !cov) return fail(SE2GPU_ERR_INVALID, "null argument");
    host_pose(*p, odo3(odom), odo3(kf_odom), odo3(last_odom), Tcr, meas, cov);
    return SE2GPU_OK;
}

int se2gpu_track_host_decide(const se2gpu_tracker_params* p, int dframes, int n_tracked_old, int n_obs_mp, int n_good_prl,
                             int n_inlier, const float* odom, const float* kf_odom, int accept_new_kf, int* new_kf, int* abort_ba) {
    if (!p || !odom || !kf_odom || !new_kf || !abort_ba) return fail(SE2GPU_ERR_INVALID, "null argument");
    host_decide(*p, dframes, n_tracked_old, n_obs_mp, n_good_prl, n_inlier, odo3(odom), odo3(kf_odom), accept_new_kf != 0, new_kf, abort_ba);
    return SE2GPU_OK;
}

}  // extern "C"
