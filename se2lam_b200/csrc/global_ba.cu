// Global pose graph: GlobalMapper::GlobalBA (reference src/GlobalMapper.cpp:328-535). One g2o VertexSE3 per keyframe with
// the plane-motion EdgeSE3Prior of addVertexSE3PlaneMotion, one EdgeSE3 per odometry and per feature constraint, and
// optimize(GLOBAL_ITER) under OptimizationAlgorithmLevenberg with a sparse direct solve over the free vertices
// (DESIGN.md section 11).
//
// The symbolic phase (global_ba_plan.h) runs on the host once per call: reverse Cuthill-McKee order, 6 x 6 block envelope,
// fixed-order gather lists. The numeric phase, the whole optimize(), is one persistent kernel on one CTA:
//  * per iteration: every edge is linearised by one thread into its own blocks (H_ii, H_jj, H_ij, b_i, b_j), every free
//    vertex's prior likewise; then H and b are gathered block entry by block entry, each entry one thread summing its
//    contributions in ascending edge order (no atomics: the bytes do not depend on scheduling);
//  * per trial: damping, a block-envelope Cholesky (LL^T, 6 x 6 pivots) in RCM order, forward and back substitution,
//    oplus, chi2 at the trial state, accept or keep; phases are separated by __syncthreads.
// All arithmetic is double precision; every reduction is a fixed tree over the CTA's threads.
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstring>

#include "common.h"
#include "envelope.h"
#include "global_ba_plan.h"
#include "lm.h"
#include "se3iso.h"

using namespace se2gpu;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct KArgs {
    int N, E, nf, S, iterations;
    float Tbc[16];
    float xrot, yrot, zinfo;
    const float* Tcw;       // [N*16]
    const float* measure;   // [E*16]
    const float* info;      // [E*36]
    const int* from;        // [E]
    const int* to;          // [E]
    const int* edge_status; // [E] or NULL: SE2GPU_FEAT_EDGE_TOO_FEW leaves the edge out
    // plan
    const int* pos; const int* vert; const int* first; const long long* rowoff;
    const int* col_ptr; const int* col_rows; const int* diag_ptr; const int* diag_code;
    const long long* off_blk; const int* off_ptr; const int* off_code;
    // work
    Iso* X[2];              // [N] current and trial estimates (which is which: s_buf)
    Prior* prior;           // [N]
    Iso* Zinv;              // [E]
    double* Om;             // [E*36]
    double* lin;            // [E*kEdgeRec]
    double* pH;             // [nf*36] prior blocks, by position
    double* pb;             // [nf*6]
    double* Hs;             // [env*36] the gathered H (blocks outside the gather lists stay zero)
    double* L;              // [env*36] damped H, factorised in place
    double* b;              // [nf*6]
    double* x;              // [nf*6]
    // outputs
    float* Tcw_out; int* status; int* iters; se2gpu_ba_iter_stats* stats; double* poses;
    unsigned long long* prof;  // [kPhases] ns per phase, accumulated by thread 0 (NULL: not profiled)
};

// the phases se2gpu_global_ba_profile_read reports
enum Phase { kSetup, kLinearise, kGather, kDamp, kFactor, kSubstitute, kTrial, kPhases };

__device__ inline unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ inline bool edge_active(const KArgs& a, int e) {
    return !a.edge_status || a.edge_status[e] != SE2GPU_FEAT_EDGE_TOO_FEW;
}

// cvu::inv of a float 4 x 4 rigid transform: R^T, and -R^T t accumulated in double (OpenCV's float gemm) and rounded once;
// the products of two floats are exact in double, so the rounding does not depend on contraction
__device__ inline void rigid_inv_f32(const float* T, float* out) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) out[i * 4 + j] = T[j * 4 + i];
        const double s = ((double)T[i] * T[3] + (double)T[4 + i] * T[7]) + (double)T[8 + i] * T[11];
        out[i * 4 + 3] = (float)(-s);
    }
    out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = 1.f;
}

// converter.cpp toIsometry3D(cv::Mat): the rotation through an un-normalised Quaterniond, the translation as it is
__device__ inline Iso iso_from_f32(const float* T) {
    Iso X;
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    quat_to_R(quat_from_R(R), X.R);
    X.t[0] = T[3]; X.t[1] = T[7]; X.t[2] = T[11];
    return X;
}

// EdgeSE3::computeError: e = toVectorMQT(Z^-1 Xi^-1 Xj); returns e^T Omega e. With J, the Jacobians through oplus on both
// vertices, E = A D(di)^-1 B with A = Z^-1, B = Xi^-1 Xj and (v, w) the quaternion of E (w >= 0):
//   Ji = [[-R_A, 2 R_A skew(t_B)], [0, -(w I - skew(v)) R_A]],  Jj = [[R_E, 0], [0, w I + skew(v)]]
__device__ __noinline__ double edge_error(const Iso& Zinv, const double* Om, const Iso& Xi, const Iso& Xj, double* e, double* Ji,
                                          double* Jj) {
    const Iso B = iso_mul(iso_inv(Xi), Xj);
    const Iso E = iso_mul(Zinv, B);
    Quat q = quat_from_R(E.R);
    normalize_rotation(q);
    e[0] = E.t[0]; e[1] = E.t[1]; e[2] = E.t[2]; e[3] = q.x; e[4] = q.y; e[5] = q.z;
    double chi = 0;
    for (int r = 0; r < 6; ++r) {
        double we = 0;
        for (int c = 0; c < 6; ++c) we += Om[r * 6 + c] * e[c];
        chi += e[r] * we;
    }
    if (!Ji) return chi;
    for (int k = 0; k < 36; ++k) { Ji[k] = 0; Jj[k] = 0; }
    const double* RA = Zinv.R;
    double S[9], RS[9], W[9];
    skew(B.t, S);
    mul3(RA, S, RS);
    // w I - skew(v)
    W[0] = q.w;  W[1] = q.z;  W[2] = -q.y;
    W[3] = -q.z; W[4] = q.w;  W[5] = q.x;
    W[6] = q.y;  W[7] = -q.x; W[8] = q.w;
    double WR[9];
    mul3(W, RA, WR);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            Ji[r * 6 + c] = -RA[r * 3 + c];
            Ji[r * 6 + 3 + c] = 2 * RS[r * 3 + c];
            Ji[(r + 3) * 6 + 3 + c] = -WR[r * 3 + c];
            Jj[r * 6 + c] = E.R[r * 3 + c];
        }
    Jj[21] = q.w;  Jj[22] = -q.z; Jj[23] = q.y;
    Jj[27] = q.z;  Jj[28] = q.w;  Jj[29] = -q.x;
    Jj[33] = -q.y; Jj[34] = q.x;  Jj[35] = q.w;
    return chi;
}

// one edge's record (envelope.h): H_ii, H_jj, H_ij = Ji^T Om Jj, b_i = -Ji^T Om e, b_j
__device__ __noinline__ void edge_linearise(const Iso& Zinv, const double* Om, const Iso& Xi, const Iso& Xj, double* out) {
    double e[6], J[2][36];
    edge_error(Zinv, Om, Xi, Xj, e, J[0], J[1]);
    edge_record(Om, e, J, out);
}

// activeChi2 at the estimates X: every active edge and every vertex's prior (the fixed ones are constant, but g2o counts them);
// valid in thread 0
__device__ double total_chi2(const KArgs& a, const Iso* X, double (&s_red)[kWarps][1]) {
    double acc = 0;
    for (int e = threadIdx.x; e < a.E; e += kThreads) {
        if (!edge_active(a, e)) continue;
        double err[6];
        acc += edge_error(a.Zinv[e], a.Om + 36 * (size_t)e, X[a.from[e]], X[a.to[e]], err, nullptr, nullptr);
    }
    for (int v = threadIdx.x; v < a.N; v += kThreads) acc += prior_terms(a.prior[v], X[v], nullptr, nullptr);
    double tot = 0;
    cta_sum<1>(&acc, s_red, &tot);
    return tot;
}

__global__ void __launch_bounds__(kThreads, 1) k_global_ba(KArgs a) {
    __shared__ double s_red[kWarps][1], s_D[36];
    __shared__ double s_cur, s_lambda, s_ni;
    __shared__ int s_flag, s_more, s_stop, s_buf;
    const int tid = threadIdx.x;
    const size_t env36 = 36 * (size_t)(a.nf ? a.rowoff[a.nf] : 0);
    // phase timing: thread 0 stamps right after the barrier that ends a phase
    unsigned long long t_last = (a.prof && tid == 0) ? global_ns() : 0;
    auto stamp = [&](int phase) {
        if (a.prof && tid == 0) {
            const unsigned long long t = global_ns();
            a.prof[phase] += t - t_last;
            t_last = t;
        }
    };

    for (int v = tid; v < a.N; v += kThreads) {  // vertices: toIsometry3D(cvu::inv(Tcw)) and their priors
        float Twc[16];
        rigid_inv_f32(a.Tcw + 16 * (size_t)v, Twc);
        const Iso X = iso_from_f32(Twc);
        a.X[0][v] = X;
        a.X[1][v] = X;
        plane_motion_prior(X, a.Tbc, a.xrot, a.yrot, a.zinfo, &a.prior[v]);
    }
    for (int e = tid; e < a.E; e += kThreads) {  // edges: toIsometry3D(measure).inverse(), toMatrix6d(info)
        a.Zinv[e] = iso_inv(iso_from_f32(a.measure + 16 * (size_t)e));
        for (int k = 0; k < 36; ++k) a.Om[36 * (size_t)e + k] = (double)a.info[36 * (size_t)e + k];
    }
    for (size_t i = tid; i < env36; i += kThreads) a.Hs[i] = 0;
    if (tid == 0) { s_stop = 0; s_buf = 0; }
    __syncthreads();
    {
        const double c = total_chi2(a, a.X[0], s_red);
        if (tid == 0) s_cur = c;
    }
    stamp(kSetup);

    // g2o's optimize() returns before its first iteration when no vertex is free
    const int iterations = a.nf ? a.iterations : 0;
    int it = 0, last_failed = 0;
    for (; it < iterations; ++it) {
        const Iso* X = a.X[s_buf];
        Iso* Xt = a.X[s_buf ^ 1];
        // linearise
        for (int e = tid; e < a.E; e += kThreads)
            if (edge_active(a, e)) edge_linearise(a.Zinv[e], a.Om + 36 * (size_t)e, X[a.from[e]], X[a.to[e]], a.lin + kEdgeRec * (size_t)e);
        for (int p = tid; p < a.nf; p += kThreads) {
            const int v = a.vert[p];
            prior_terms(a.prior[v], X[v], a.pH + 36 * (size_t)p, a.pb + 6 * (size_t)p);
        }
        __syncthreads();
        stamp(kLinearise);
        // gather H and b in ascending edge order
        const auto active = [&](int e) { return edge_active(a, e); };
        gather_diag(a, a.lin, a.b, tid, kThreads, active, [](int, int, double s) { return s; });
        gather_off(a, a.lin, tid, kThreads, active);
        __syncthreads();
        stamp(kGather);
        if (it == 0) {  // computeLambdaInit over the free vertices
            double m = 0;
            for (int idx = tid; idx < a.nf * 6; idx += kThreads)
                m = fmax(m, fabs(blkp(a.Hs, a, idx / 6, idx / 6)[(idx % 6) * 7]));
            m = cta_max(m, s_red);
            if (tid == 0) lm_lambda_init(m, s_lambda, s_ni);
        }
        const double chi_before = s_cur;
        int qmax = 0, failed = 0, accepted = 0;
        double rho = 0;
        for (;;) {
            __syncthreads();
            const double lambda = s_lambda;
            for (size_t i = tid; i < env36; i += kThreads) a.L[i] = a.Hs[i];
            __syncthreads();
            damp(a, a.L, lambda, tid, kThreads);
            __syncthreads();
            stamp(kDamp);
            const bool ok = env_factor<kThreads>(a, s_D, &s_flag);
            stamp(kFactor);
            double temp = DBL_MAX, scale = 0;
            if (ok) {
                env_substitute(a);
                __syncthreads();
                stamp(kSubstitute);
                double sc = 0;
                for (int p = tid; p < a.nf; p += kThreads) {
                    const double* d = a.x + 6 * (size_t)p;
                    const int v = a.vert[p];
                    Xt[v] = oplus(X[v], d);
                    for (int r = 0; r < 6; ++r) sc += d[r] * (lambda * d[r] + a.b[6 * (size_t)p + r]);
                }
                cta_sum<1>(&sc, s_red, &scale);
                temp = total_chi2(a, Xt, s_red);
            }
            if (tid == 0) {
                if (!ok) ++failed;
                if (lm_gain_step(temp, scale, ok, s_cur, s_lambda, s_ni, rho)) { s_buf ^= 1; accepted = 1; }
                ++qmax;
                s_more = lm_retry(rho, qmax);
            }
            __syncthreads();
            stamp(kTrial);
            if (!s_more) break;
        }
        if (tid == 0) {
            const se2gpu_ba_iter_stats st = lm_iter_stats(chi_before, s_cur, s_lambda, rho, qmax, accepted);
            last_failed = lm_not_pd(st, failed);
            if (a.stats) a.stats[it] = st;
            s_stop = st.terminate;
        }
        __syncthreads();
        // the fixed vertices are the same in both buffers; a free vertex's trial is rewritten before it is read
        if (s_stop) { ++it; break; }
    }

    // write-back: cvu::inv(toCvMat(toSE3Quat(estimate)))
    const Iso* X = a.X[s_buf];
    for (int v = tid; v < a.N; v += kThreads) {
        const SE3 T = se3_from_iso(X[v]);
        float Twc[16];
        se3_to_f32(T, Twc);
        rigid_inv_f32(Twc, a.Tcw_out + 16 * (size_t)v);
        if (a.poses) store_pose(T, a.poses + 7 * (size_t)v);
    }
    if (tid == 0) {
        if (a.iters) *a.iters = it;
        if (a.status) *a.status = last_failed ? SE2GPU_GLOBAL_BA_NOT_PD : SE2GPU_GLOBAL_BA_OK;
    }
}

// GlobalBA's map-point write-back (:506-531): pos = Rwc * view + twc of the main keyframe, Twc its rigid inverse
__global__ void k_update_points(int M, const int* __restrict__ kf, const float* __restrict__ view, const float* __restrict__ Tcw,
                                float* __restrict__ pos) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float Twc[16];
    rigid_inv_f32(Tcw + 16 * (size_t)kf[m], Twc);
    const float* v = view + 3 * (size_t)m;
    for (int r = 0; r < 3; ++r) {
        const double s = ((double)Twc[r * 4] * v[0] + (double)Twc[r * 4 + 1] * v[1]) + (double)Twc[r * 4 + 2] * v[2];
        pos[3 * (size_t)m + r] = (float)(s + (double)Twc[r * 4 + 3]);
    }
}

int check_params(const se2gpu_global_ba_params* p) {
    if (!p) return fail(SE2GPU_ERR_INVALID, "null parameters");
    if (p->iterations < 0) return fail(SE2GPU_ERR_INVALID, "iterations = %d", p->iterations);
    return SE2GPU_OK;
}

// the graph; with measure / info (host entries) also the edges' values
int check_graph(int N, const uint8_t* fixed, int E, const int* from, const int* to, const float* measure, const float* info) {
    if (N <= 0) return fail(SE2GPU_ERR_INVALID, "N = %d", N);
    if (E < 0) return fail(SE2GPU_ERR_INVALID, "E = %d", E);
    if (!fixed || (E && (!from || !to))) return fail(SE2GPU_ERR_INVALID, "null topology arrays");
    return check_se3_links(N, E, from, to, measure, info, "edge", "vertex");
}

}  // namespace

struct se2gpu_global_ba_ctx : se2gpu::PlanContext {
    unsigned long long* d_prof = nullptr;  // [kPhases] while profiling is on
    unsigned long long* d_prof_buf = nullptr;
};

namespace {

// plans the call, uploads the plan on `stream` and launches the kernel there; every value array is device memory
int run(se2gpu_global_ba_ctx* h, int N, const uint8_t* fixed, int E, const int* from, const int* to, const float* d_Tcw,
        const float* d_measure, const float* d_info, const int* d_from, const int* d_to, const int* d_edge_status,
        const se2gpu_global_ba_params* prm, float* d_Tcw_out, int* d_status, int* d_iters, se2gpu_ba_iter_stats* d_stats,
        double* d_poses, cudaStream_t stream) {
    const gba::Plan P = gba::make_plan(N, fixed, E, from, to);
    const int nf = P.n_free, S = (int)P.off_blk.size();
    const size_t env = (size_t)P.env_blocks();
    // the plan (from / to only when they are not given on the device), then the work
    Packed<int> ints;
    Packed<long long> lls;
    Layout dbl;
    struct {
        size_t from, to, pos, vert, first, col_ptr, col_rows, diag_ptr, diag_code, off_ptr, off_code;  // ints
        size_t rowoff, off_blk;                                                                      // long longs
        size_t X[2], prior, Zinv, Om, lin, pH, pb, b, x, Hs, L;                                      // doubles
    } o;
    o.from = ints.put(from, d_from ? 0 : (size_t)E); o.to = ints.put(to, d_to ? 0 : (size_t)E);
    o.pos = ints.put(P.pos); o.vert = ints.put(P.vert); o.first = ints.put(P.first); o.col_ptr = ints.put(P.col_ptr);
    o.col_rows = ints.put(P.col_rows); o.diag_ptr = ints.put(P.diag_ptr); o.diag_code = ints.put(P.diag_code);
    o.off_ptr = ints.put(P.off_ptr); o.off_code = ints.put(P.off_code);
    o.rowoff = lls.put(P.rowoff); o.off_blk = lls.put(P.off_blk);
    o.X[0] = dbl.take(12 * (size_t)N); o.X[1] = dbl.take(12 * (size_t)N); o.prior = dbl.take(sizeof(Prior) / 8 * (size_t)N);
    o.Zinv = dbl.take(12 * (size_t)E); o.Om = dbl.take(36 * (size_t)E); o.lin = dbl.take(kEdgeRec * (size_t)E);
    o.pH = dbl.take(36 * (size_t)nf); o.pb = dbl.take(6 * (size_t)nf); o.b = dbl.take(6 * (size_t)nf); o.x = dbl.take(6 * (size_t)nf);
    o.Hs = dbl.take(36 * env); o.L = dbl.take(36 * env);
    { const int rc = h->grow(&h->d_dbl, &h->cap_dbl, dbl.size); if (rc) return rc; }
    { const int rc = h->upload_plan(ints.data, lls.data, stream); if (rc) return rc; }

    KArgs a{};
    a.N = N; a.E = E; a.nf = nf; a.S = S; a.iterations = prm->iterations;
    std::memcpy(a.Tbc, prm->Tbc, sizeof a.Tbc);
    a.xrot = prm->xrot_info; a.yrot = prm->yrot_info; a.zinfo = prm->z_info;
    a.Tcw = d_Tcw; a.measure = d_measure; a.info = d_info;
    const int* I = h->d_int;
    a.from = d_from ? d_from : I + o.from;
    a.to = d_to ? d_to : I + o.to;
    a.edge_status = d_edge_status;
    a.pos = I + o.pos; a.vert = I + o.vert; a.first = I + o.first; a.col_ptr = I + o.col_ptr; a.col_rows = I + o.col_rows;
    a.diag_ptr = I + o.diag_ptr; a.diag_code = I + o.diag_code; a.off_ptr = I + o.off_ptr; a.off_code = I + o.off_code;
    a.rowoff = h->d_ll + o.rowoff; a.off_blk = h->d_ll + o.off_blk;
    double* D = h->d_dbl;
    a.X[0] = (Iso*)(D + o.X[0]); a.X[1] = (Iso*)(D + o.X[1]); a.prior = (Prior*)(D + o.prior); a.Zinv = (Iso*)(D + o.Zinv);
    a.Om = D + o.Om; a.lin = D + o.lin; a.pH = D + o.pH; a.pb = D + o.pb; a.b = D + o.b; a.x = D + o.x; a.Hs = D + o.Hs; a.L = D + o.L;
    a.Tcw_out = d_Tcw_out; a.status = d_status; a.iters = d_iters; a.stats = d_stats; a.poses = d_poses;
    a.prof = h->d_prof;
    if (d_stats && prm->iterations)
        SE2_CUDA(cudaMemsetAsync(d_stats, 0, sizeof(se2gpu_ba_iter_stats) * (size_t)prm->iterations, stream));
    SE2_NVTX("se2gpu_global_ba");
    SE2_LAUNCH(k_global_ba, 1, kThreads, 0, stream, a);
    SE2_CUDA(cudaGetLastError());
    SE2_CUDA(cudaEventRecord(h->done, stream));
    return SE2GPU_OK;
}

}  // namespace

se2gpu_global_ba_ctx* se2gpu_global_ba_create(int device) { return create_plan_context<se2gpu_global_ba_ctx>(device); }

void se2gpu_global_ba_destroy(se2gpu_global_ba_ctx* h) { delete h; }

int se2gpu_global_ba(se2gpu_global_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, int E, const int* edge_from,
                     const int* edge_to, const float* measure, const float* info, const se2gpu_global_ba_params* params,
                     float* Tcw_out, int* status, int* iterations, se2gpu_ba_iter_stats* stats, double* poses) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null context");
    { const int rc = check_params(params); if (rc) return rc; }
    if (!Tcw || !Tcw_out || (E && (!measure || !info))) return fail(SE2GPU_ERR_INVALID, "null arrays");
    { const int rc = check_graph(N, fixed, E, edge_from, edge_to, measure, info); if (rc) return rc; }
    HostStage st(h->device);
    if (const int rc = st.status()) return rc;
    const float* dT = st.upload(Tcw, 16 * (size_t)N);
    const float* dm = st.upload(measure, 16 * (size_t)E);
    const float* di = st.upload(info, 36 * (size_t)E);
    const int* df = st.upload(edge_from, (size_t)E);
    const int* dt = st.upload(edge_to, (size_t)E);
    float* dout = st.output(Tcw_out, 16 * (size_t)N);
    int* dst = status ? st.output(status, 1) : nullptr;
    int* dit = iterations ? st.output(iterations, 1) : nullptr;
    se2gpu_ba_iter_stats* dstats = stats && params->iterations ? st.output(stats, (size_t)params->iterations) : nullptr;
    double* dposes = poses ? st.output(poses, 7 * (size_t)N) : nullptr;
    if (const int rc = st.status()) return rc;
    // h->stream is a blocking stream: the staged copies on the legacy stream order themselves around the kernel
    { const int rc = run(h, N, fixed, E, edge_from, edge_to, dT, dm, di, df, dt, nullptr, params, dout, dst, dit, dstats, dposes, h->stream); if (rc) return rc; }
    return st.finish();
}

int se2gpu_global_ba_device(se2gpu_global_ba_ctx* h, int N, const float* d_Tcw, const uint8_t* fixed, int E, const int* edge_from,
                            const int* edge_to, const float* d_measure, const float* d_info, const int* d_edge_status,
                            const se2gpu_global_ba_params* params, float* d_Tcw_out, int* d_status, int* d_iterations,
                            se2gpu_ba_iter_stats* d_stats, double* d_poses, void* stream) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null context");
    { const int rc = check_params(params); if (rc) return rc; }
    if (!d_Tcw || !d_Tcw_out || (E && (!d_measure || !d_info))) return fail(SE2GPU_ERR_INVALID, "null arrays");
    { const int rc = check_graph(N, fixed, E, edge_from, edge_to, nullptr, nullptr); if (rc) return rc; }
    { const int rc = select_device(h->device); if (rc) return rc; }
    return run(h, N, fixed, E, edge_from, edge_to, d_Tcw, d_measure, d_info, nullptr, nullptr, d_edge_status, params, d_Tcw_out,
               d_status, d_iterations, d_stats, d_poses, (cudaStream_t)stream);
}

int se2gpu_global_ba_update_points(int M, const int* kf_index, const float* view_mp, int N, const float* Tcw, float* pos_out,
                                   int device) {
    if (M < 0 || N <= 0 || !Tcw || (M && (!kf_index || !view_mp || !pos_out))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    for (int m = 0; m < M; ++m)
        if (kf_index[m] < 0 || kf_index[m] >= N) return fail(SE2GPU_ERR_INVALID, "kf_index[%d] = %d out of range", m, kf_index[m]);
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (M == 0) return SE2GPU_OK;
    const int* dk = st.upload(kf_index, (size_t)M);
    const float* dv = st.upload(view_mp, 3 * (size_t)M);
    const float* dT = st.upload(Tcw, 16 * (size_t)N);
    float* dp = st.output(pos_out, 3 * (size_t)M);
    if (const int rc = st.status()) return rc;
    { const int rc = se2gpu_global_ba_update_points_device(M, dk, dv, dT, dp, nullptr); if (rc) return rc; }
    return st.finish();
}

int se2gpu_global_ba_update_points_device(int M, const int* d_kf_index, const float* d_view_mp, const float* d_Tcw, float* d_pos_out,
                                          void* stream) {
    if (M < 0 || (M && (!d_kf_index || !d_view_mp || !d_Tcw || !d_pos_out))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    if (M == 0) return SE2GPU_OK;
    SE2_NVTX("se2gpu_global_ba_update_points");
    SE2_LAUNCH(k_update_points, (M + 255) / 256, 256, 0, (cudaStream_t)stream, M, d_kf_index, d_view_mp, d_Tcw, d_pos_out);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_global_ba_profile(se2gpu_global_ba_ctx* h, int on) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null context");
    { const int rc = select_device(h->device); if (rc) return rc; }
    SE2_CUDA(cudaEventSynchronize(h->done));
    if (!on) { h->d_prof = nullptr; return SE2GPU_OK; }
    if (!h->d_prof_buf) SE2_CUDA(h->bufs.alloc(&h->d_prof_buf, (size_t)kPhases));
    SE2_CUDA(cudaMemset(h->d_prof_buf, 0, sizeof(unsigned long long) * kPhases));
    h->d_prof = h->d_prof_buf;
    return SE2GPU_OK;
}

int se2gpu_global_ba_profile_read(se2gpu_global_ba_ctx* h, double* ms) {
    if (!h || !ms) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (!h->d_prof) return fail(SE2GPU_ERR_INVALID, "profiling is off");
    { const int rc = select_device(h->device); if (rc) return rc; }
    SE2_CUDA(cudaEventSynchronize(h->done));
    unsigned long long ns[kPhases];
    SE2_CUDA(cudaMemcpy(ns, h->d_prof, sizeof ns, cudaMemcpyDeviceToHost));
    for (int i = 0; i < kPhases; ++i) ms[i] = ns[i] * 1e-6;
    return SE2GPU_OK;
}
