// Pose-only SE(3) bundle adjustment: Localizer::DoLocalBA (reference src/Localizer.cpp:233-302) for B independent problems,
// one CTA each, all LM iterations inside the kernel.
//
// What a problem is (DESIGN.md section 9): one g2o VertexSE3Expmap (estimate toSE3Quat(Tcw)), one EdgeSE3ExpmapPrior from
// addPlaneMotionSE3Expmap (src/optimizer.cpp:236-314) and one EdgeProjectXYZ2UV with a Huber kernel per observed map point
// (fixed points, information w_e I), optimised by g2o's OptimizationAlgorithmLevenberg. Everything is double precision.
//
// Per CTA: thread 0 builds the prior and holds the LM scalars in shared memory; the edges are staged in shared memory when
// they fit (kStageMax), otherwise read from global memory. Each linearisation has every thread accumulate the 21 upper
// entries of H, the 6 of b and the robust chi2 of the edges e = tid, tid + 256, ... in registers; a warp xor-shuffle tree
// and then the 8 warp sums in index order combine them (no atomics: bit-reproducible, independent of the CTA's position in
// the batch). Thread 0 adds the prior, damps, factorises the 6 x 6 system (LL^T), applies SE3Quat::exp and the compose,
// and a second reduction gives the trial chi2.
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstring>

#include "common.h"
#include "lm.h"
#include "se3expmap.h"

using namespace se2gpu;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kStageMax = 1536;  // edges staged in shared memory: 24 B each, 36 KB
constexpr int kAcc = 28;         // 21 upper entries of H, 6 of b, chi2

struct Params {
    double fx, cx, cy, delta;
    float Tbc[16];
    float xrot, yrot, zinfo;
    int iterations;
};

__global__ void __launch_bounds__(kThreads) k_pose_ba(float* __restrict__ Tcw, const int* __restrict__ edge_ptr, int edge_slot,
                                                      const int* __restrict__ skip, const float* __restrict__ xyz,
                                                      const float* __restrict__ uv, const float* __restrict__ info, Params p,
                                                      int min_edges, se2gpu_ba_iter_stats* __restrict__ stats,
                                                      int* __restrict__ iters, int* __restrict__ status,
                                                      double* __restrict__ pose_out, double* __restrict__ trace) {
    extern __shared__ float s_stage[];  // [kStageMax*3] xyz, [kStageMax*2] uv, [kStageMax] info
    __shared__ double s_red[kWarps][kAcc];
    __shared__ double s_H[36], s_b[6], s_info[36], s_sum[kAcc];
    __shared__ SE3 s_est, s_trial, s_meas;
    __shared__ double s_cur, s_lambda, s_ni;
    __shared__ int s_ok2, s_more, s_stop;

    const int pb = blockIdx.x, tid = threadIdx.x;
    // edge_slot 0: problem pb's edges are edge_ptr[pb] .. edge_ptr[pb+1]-1; otherwise the first edge_ptr[pb] of its slot
    const int e0 = edge_slot ? pb * edge_slot : edge_ptr[pb], E = edge_slot ? edge_ptr[pb] : edge_ptr[pb + 1] - e0;
    const int sk = skip ? skip[pb] : 0;  // 1: gated by the caller, 2: not run
    float* T16 = Tcw + 16 * (size_t)pb;
    if (E <= 0 || E <= min_edges || sk) {  // nothing to refine against: the pose is left as it is
        if (tid == 0) {
            if (iters) iters[pb] = 0;
            if (status) status[pb] = (sk == 1 || (E > 0 && sk == 0)) ? SE2GPU_POSE_BA_GATED : SE2GPU_POSE_BA_NO_EDGES;
            if (pose_out) store_pose(se3_from_f32(T16), pose_out + 7 * (size_t)pb);
        }
        return;
    }
    if (tid == 0) {
        s_est = se3_from_f32(T16);
        plane_motion_prior(s_est, p, &s_meas, s_info);
        s_stop = 0;
    }
    const float* gx = xyz + 3 * (size_t)e0;
    const float* gu = uv + 2 * (size_t)e0;
    const float* gw = info + e0;
    const bool staged = E <= kStageMax;
    const float* px = gx;
    const float* pu = gu;
    const float* pw = gw;
    if (staged) {
        for (int k = tid; k < 3 * E; k += kThreads) s_stage[k] = gx[k];
        for (int k = tid; k < 2 * E; k += kThreads) s_stage[3 * kStageMax + k] = gu[k];
        for (int k = tid; k < E; k += kThreads) s_stage[5 * kStageMax + k] = gw[k];
        px = s_stage; pu = s_stage + 3 * kStageMax; pw = s_stage + 5 * kStageMax;
    }
    __syncthreads();

    int it = 0, last_failed = 0;
    for (; it < p.iterations; ++it) {
        // linearise at the current estimate: chi2, H, b
        {
            double acc[kAcc];
#pragma unroll
            for (int k = 0; k < kAcc; ++k) acc[k] = 0;
            const SE3 T = s_est;
            for (int e = tid; e < E; e += kThreads) edge_terms<true>(T, px + 3 * e, pu + 2 * e, pw[e], p, acc[27], acc);
            cta_sum<kAcc>(acc, s_red, s_sum);
        }
        double chi_before = 0;
        if (tid == 0) {
            double ep[6];
            const double pchi = prior_error(s_meas, s_info, s_est, ep);
            int k = 0;
            for (int r = 0; r < 6; ++r)
                for (int c = r; c < 6; ++c, ++k) s_H[r * 6 + c] = s_H[c * 6 + r] = s_sum[k] + s_info[r * 6 + c];
            for (int r = 0; r < 6; ++r) {  // EdgeSE3ExpmapPrior, J = -I: b += Omega e
                double we = 0;
                for (int c = 0; c < 6; ++c) we += s_info[r * 6 + c] * ep[c];
                s_b[r] = s_sum[21 + r] + we;
            }
            s_cur = s_sum[27] + pchi;
            if (it == 0) {
                double m = 0;
                for (int r = 0; r < 6; ++r) m = fmax(m, fabs(s_H[r * 7]));
                lm_lambda_init(m, s_lambda, s_ni);
            }
            chi_before = s_cur;
        }
        int qmax = 0, failed = 0, accepted = 0;
        double rho = 0;
        for (;;) {
            double x[6], scale = 0;
            if (tid == 0) {
                double L[36];  // LL^T of H + lambda I
                for (int r = 0; r < 6; ++r)
                    for (int c = 0; c <= r; ++c) L[r * 6 + c] = s_H[r * 6 + c] + (r == c ? s_lambda : 0.0);
                const bool ok2 = chol_factor(6, 6, L);
                s_ok2 = ok2;
                if (ok2) {
                    chol_solve(6, 6, L, s_b, x);
                    s_trial = se3_mul(se3_exp(x), s_est);
                    for (int r = 0; r < 6; ++r) scale += x[r] * (s_lambda * x[r] + s_b[r]);
                }
            }
            __syncthreads();
            double temp = DBL_MAX;
            if (s_ok2) {
                double a[1] = {0};
                const SE3 T = s_trial;
                for (int e = tid; e < E; e += kThreads) edge_terms<false>(T, px + 3 * e, pu + 2 * e, pw[e], p, a[0], nullptr);
                double tot[1];
                cta_sum<1>(a, s_red, tot);
                if (tid == 0) {
                    double ep[6];
                    temp = tot[0] + prior_error(s_meas, s_info, s_trial, ep);
                }
            }
            if (tid == 0) {
                if (!s_ok2) ++failed;
                if (lm_gain_step(temp, scale, s_ok2, s_cur, s_lambda, s_ni, rho)) { s_est = s_trial; accepted = 1; }
                ++qmax;
                s_more = lm_retry(rho, qmax);
            }
            __syncthreads();
            if (!s_more) break;
        }
        if (tid == 0) {
            const se2gpu_ba_iter_stats st = lm_iter_stats(chi_before, s_cur, s_lambda, rho, qmax, accepted);
            last_failed = lm_not_pd(st, failed);
            if (stats) stats[(size_t)pb * p.iterations + it] = st;
            if (trace) store_pose(s_est, trace + ((size_t)pb * p.iterations + it) * 7);
            s_stop = st.terminate;
        }
        __syncthreads();
        if (s_stop) { ++it; break; }
    }
    if (tid == 0) {
        if (iters) iters[pb] = it;
        if (status) status[pb] = last_failed ? SE2GPU_POSE_BA_NOT_PD : SE2GPU_POSE_BA_OK;
        if (pose_out) store_pose(s_est, pose_out + 7 * (size_t)pb);
        se3_to_f32(s_est, T16);
    }
}

// Localizer::DoLocalBA's edge lists for B streams (one CTA each), in ascending map-point index: map point j is an edge of
// stream b when some keypoint i < n[b] of b matched it (the highest such i, as repeated KeyFrame::addObservation leaves it)
// and use[j]; every edge's information is inv_sigma2[kp[0].octave] (MapPoint::getOctave on a keyframe it never observed).
// Stream b reads kp / matches + b * cap_kf and writes best + b * n_mp, xyz / uv / w at b * edge_slot (edge_slot 0: one
// stream, edge_ptr = {0, count}; otherwise edge_ptr[b] = count). The count of distinct matched map points, used or not,
// is getSizeObsMP(): with run (may be NULL) and min_obs >= 0, skip[b] is 2 when !run[b] (no edges) and 1 when that count
// is min_obs or less (DoLocalBA's gate); n_obs (may be NULL) receives it.
__global__ void __launch_bounds__(1024) k_localizer_edges(const se2gpu_keypoint* __restrict__ kp, int cap_kf, const int* __restrict__ d_n_kf,
                                                          const int* __restrict__ matches, int n_mp, const float* __restrict__ mp_xyz,
                                                          const uint8_t* __restrict__ mp_use, const float* __restrict__ inv_sigma2,
                                                          int nlevels, const int* __restrict__ run, int min_obs, int edge_slot,
                                                          int* __restrict__ best_all, float* __restrict__ xyz_all,
                                                          float* __restrict__ uv_all, float* __restrict__ w_all,
                                                          int* __restrict__ edge_ptr, int* __restrict__ n_edges,
                                                          int* __restrict__ skip, int* __restrict__ n_obs) {
    __shared__ int s_wcount[32], s_wobs[32];
    __shared__ int s_base, s_obs;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool go = !run || run[b];
    kp += (size_t)b * cap_kf; matches += (size_t)b * cap_kf;
    int* best = best_all + (size_t)b * n_mp;
    const size_t eo = (size_t)b * edge_slot;
    float* xyz = xyz_all + 3 * eo;
    float* uv = uv_all + 2 * eo;
    float* w = w_all + eo;
    const int n = go ? count_of(d_n_kf ? d_n_kf + b : nullptr, cap_kf) : 0;
    for (int j = tid; j < n_mp; j += blockDim.x) best[j] = -1;
    if (tid == 0) { s_base = 0; s_obs = 0; }
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
        const int m = matches[i];
        if (m >= 0 && m < n_mp) atomicMax(&best[m], i);
    }
    __syncthreads();
    const float w0 = n > 0 ? inv_sigma2[min(max(kp[0].octave, 0), nlevels - 1)] : 0.f;
    for (int j0 = 0; j0 < n_mp; j0 += blockDim.x) {
        const int j = j0 + tid;
        const int k = j < n_mp ? best[j] : -1;
        const bool take = k >= 0 && mp_use[j];
        const unsigned bal = __ballot_sync(0xffffffffu, take);
        const unsigned bobs = __ballot_sync(0xffffffffu, k >= 0);
        if (lane == 0) { s_wcount[warp] = __popc(bal); s_wobs[warp] = __popc(bobs); }
        __syncthreads();
        int off = s_base;
        for (int v = 0; v < warp; ++v) off += s_wcount[v];
        off += __popc(bal & ((1u << lane) - 1));
        if (take) {
            xyz[3 * off] = mp_xyz[3 * (size_t)j]; xyz[3 * off + 1] = mp_xyz[3 * (size_t)j + 1]; xyz[3 * off + 2] = mp_xyz[3 * (size_t)j + 2];
            uv[2 * off] = kp[k].x; uv[2 * off + 1] = kp[k].y;
            w[off] = w0;
        }
        __syncthreads();
        if (tid == 0) {
            int tot = 0, obs = 0;
            for (int v = 0; v < (int)(blockDim.x >> 5); ++v) { tot += s_wcount[v]; obs += s_wobs[v]; }
            s_base += tot;
            s_obs += obs;
        }
        __syncthreads();
    }
    if (tid == 0) {
        if (edge_slot) {
            edge_ptr[b] = s_base;
        } else {
            edge_ptr[0] = 0;
            edge_ptr[1] = s_base;
        }
        if (n_edges) n_edges[b] = s_base;
        if (skip) skip[b] = !go ? 2 : (min_obs >= 0 && s_obs <= min_obs ? 1 : 0);
        if (n_obs) n_obs[b] = s_obs;
    }
}

int check_params(const se2gpu_pose_ba_params* prm, Params* p) {
    if (!prm) return fail(SE2GPU_ERR_INVALID, "null parameters");
    if (prm->iterations < 0) return fail(SE2GPU_ERR_INVALID, "iterations = %d", prm->iterations);
    p->fx = prm->fx; p->cx = prm->cx; p->cy = prm->cy; p->delta = prm->huber_delta;
    std::memcpy(p->Tbc, prm->Tbc, sizeof p->Tbc);
    p->xrot = prm->xrot_info; p->yrot = prm->yrot_info; p->zinfo = prm->z_info;
    p->iterations = prm->iterations;
    return SE2GPU_OK;
}

constexpr size_t kStageBytes = sizeof(float) * 6 * kStageMax;

int launch(int B, float* d_Tcw, const int* d_edge_ptr, int edge_slot, const int* d_skip, const float* d_xyz, const float* d_uv,
           const float* d_info, const Params& p, int min_edges, se2gpu_ba_iter_stats* d_stats, int* d_iters, int* d_status,
           double* d_pose, double* d_trace, cudaStream_t stream) {
    SE2_NVTX("se2gpu_pose_ba");
    SE2_LAUNCH(k_pose_ba, B, kThreads, kStageBytes, stream, d_Tcw, d_edge_ptr, edge_slot, d_skip, d_xyz, d_uv, d_info, p, min_edges,
               d_stats, d_iters, d_status, d_pose, d_trace);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int host_run(int B, float* Tcw, const int* edge_ptr, const float* xyz, const float* uv, const float* info,
             const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* stats, int* iterations, int* status, double* pose,
             double* trace, int device) {
    Params p;
    { const int rc = check_params(params, &p); if (rc) return rc; }
    if (B < 0 || (B && (!Tcw || !edge_ptr))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (B && edge_ptr[0] != 0) return fail(SE2GPU_ERR_INVALID, "edge_ptr[0] must be 0");
    for (int b = 0; b < B; ++b)
        if (edge_ptr[b + 1] < edge_ptr[b]) return fail(SE2GPU_ERR_INVALID, "edge_ptr not ascending at %d", b);
    const size_t E = B ? (size_t)edge_ptr[B] : 0;
    if (E && (!xyz || !uv || !info)) return fail(SE2GPU_ERR_INVALID, "null edge arrays");
    HostStage st(device);
    if (const int rc = st.status()) return rc;
    if (B == 0) return SE2GPU_OK;
    const size_t it = (size_t)p.iterations;
    float* dT = st.inout(Tcw, 16 * (size_t)B);
    const int* dptr = st.upload(edge_ptr, (size_t)B + 1);
    const float* dx = st.upload(xyz, 3 * E);
    const float* du = st.upload(uv, 2 * E);
    const float* dw = st.upload(info, E);
    se2gpu_ba_iter_stats* dst = stats ? st.output(stats, B * it) : nullptr;
    int* dit = iterations ? st.output(iterations, B) : st.scratch<int>(B);
    int* dsts = status ? st.output(status, B) : st.scratch<int>(B);
    double* dpose = pose ? st.output(pose, 7 * (size_t)B) : nullptr;
    double* dtr = trace ? st.output(trace, 7 * B * it) : nullptr;
    if (dst) st.check(cudaMemset(dst, 0, sizeof(se2gpu_ba_iter_stats) * B * it), "cudaMemset");
    if (dtr) st.check(cudaMemset(dtr, 0, sizeof(double) * 7 * B * it), "cudaMemset");
    if (const int rc = st.status()) return rc;
    { const int rc = launch(B, dT, dptr, 0, nullptr, dx, du, dw, p, 0, dst, dit, dsts, dpose, dtr, nullptr); if (rc) return rc; }
    return st.finish();
}

}  // namespace

struct se2gpu_localizer {
    int device = 0, max_mp = 0;
    int* best = nullptr;
    float* xyz = nullptr;
    float* uv = nullptr;
    float* w = nullptr;
    int* edge_ptr = nullptr;
    se2gpu::DeviceBuffers bufs;
};

se2gpu_localizer* se2gpu_localizer_create(int max_map_points, int device) {
    if (max_map_points < 0) { fail(SE2GPU_ERR_INVALID, "max_map_points = %d", max_map_points); return nullptr; }
    if (select_device(device)) return nullptr;
    auto* h = new se2gpu_localizer;
    h->device = device; h->max_mp = max_map_points;
    const size_t m = (size_t)(max_map_points ? max_map_points : 1);
    if (h->bufs.alloc(&h->best, m) != cudaSuccess || h->bufs.alloc(&h->xyz, 3 * m) != cudaSuccess || h->bufs.alloc(&h->uv, 2 * m) != cudaSuccess ||
        h->bufs.alloc(&h->w, m) != cudaSuccess || h->bufs.alloc(&h->edge_ptr, 2) != cudaSuccess) {
        fail(SE2GPU_ERR_CUDA, "device allocation failed");
        se2gpu_localizer_destroy(h);
        return nullptr;
    }
    return h;
}

void se2gpu_localizer_destroy(se2gpu_localizer* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    delete h;
}

int se2gpu_pose_ba(int B, float* Tcw, const int* edge_ptr, const float* xyz, const float* uv, const float* info,
                   const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* stats, int* iterations, int* status, double* pose,
                   int device) {
    return host_run(B, Tcw, edge_ptr, xyz, uv, info, params, stats, iterations, status, pose, nullptr, device);
}

int se2gpu_pose_ba_debug_trace(int B, float* Tcw, const int* edge_ptr, const float* xyz, const float* uv, const float* info,
                               const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* stats, int* iterations, int* status,
                               double* pose, double* trace, int device) {
    return host_run(B, Tcw, edge_ptr, xyz, uv, info, params, stats, iterations, status, pose, trace, device);
}

int se2gpu_pose_ba_device(int B, float* d_Tcw, const int* d_edge_ptr, const float* d_xyz, const float* d_uv, const float* d_info,
                          const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* d_stats, int* d_iterations, int* d_status,
                          double* d_pose, void* stream) {
    Params p;
    { const int rc = check_params(params, &p); if (rc) return rc; }
    if (B < 0 || (B && (!d_Tcw || !d_edge_ptr))) return fail(SE2GPU_ERR_INVALID, "bad arguments");
    { const int rc = require_device(); if (rc) return rc; }
    if (B == 0) return SE2GPU_OK;
    return launch(B, d_Tcw, d_edge_ptr, 0, nullptr, d_xyz, d_uv, d_info, p, 0, d_stats, d_iterations, d_status, d_pose, nullptr, (cudaStream_t)stream);
}

int se2gpu_localizer_ba_device(se2gpu_localizer* h, const se2gpu_keypoint* d_kf_kp, int n_kf, const int* d_n_kf,
                               const int* d_matches_idx_mp, int n_mp, const float* d_mp_xyz, const uint8_t* d_mp_use,
                               const float* d_inv_sigma2, int nlevels, float* d_Tcw, const se2gpu_pose_ba_params* params,
                               int min_edges, int* d_n_edges, se2gpu_ba_iter_stats* d_stats, int* d_iterations, int* d_status,
                               double* d_pose, void* stream) {
    Params p;
    { const int rc = check_params(params, &p); if (rc) return rc; }
    if (!h || n_kf < 0 || n_mp < 0 || nlevels <= 0 || !d_Tcw || !d_inv_sigma2 || (n_kf && (!d_kf_kp || !d_matches_idx_mp)) ||
        (n_mp && (!d_mp_xyz || !d_mp_use)))
        return fail(SE2GPU_ERR_INVALID, "bad arguments");
    if (n_mp > h->max_mp) return fail(SE2GPU_ERR_CAPACITY, "n_mp = %d exceeds the context's %d map points", n_mp, h->max_mp);
    SE2_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = (cudaStream_t)stream;
    // the B = 1 call of the batched edge kernel se2gpu_loc_step runs
    SE2_LAUNCH(k_localizer_edges, 1, 1024, 0, s, d_kf_kp, n_kf, d_n_kf, d_matches_idx_mp, n_mp, d_mp_xyz, d_mp_use, d_inv_sigma2,
               nlevels, nullptr, -1, 0, h->best, h->xyz, h->uv, h->w, h->edge_ptr, d_n_edges, nullptr, nullptr);
    SE2_CUDA(cudaGetLastError());
    return launch(1, d_Tcw, h->edge_ptr, 0, nullptr, h->xyz, h->uv, h->w, p, min_edges, d_stats, d_iterations, d_status, d_pose,
                  nullptr, s);
}

// DoLocalBA for B streams of the localization handle (loc.cu): edges at stream b's slot of edge_slot entries, run / gate as
// k_localizer_edges above, then the batched solve with min_edges 0 (a stream without edges keeps its pose).
int se2gpu::loc_local_ba(int B, const se2gpu_keypoint* d_kp, int cap_kf, const int* d_n, const int* d_obs_mp, int n_mp,
                         const float* d_mp_xyz, const uint8_t* d_mp_use, const float* d_inv_sigma2, int nlevels, const int* d_run,
                         int min_obs, int* d_best, float* d_xyz, float* d_uv, float* d_w, int* d_edges, int* d_skip, int* d_n_obs,
                         float* d_Tcw, const se2gpu_pose_ba_params* params, int* d_iterations, int* d_status, cudaStream_t s) {
    Params p;
    { const int rc = check_params(params, &p); if (rc) return rc; }
    SE2_LAUNCH(k_localizer_edges, B, 1024, 0, s, d_kp, cap_kf, d_n, d_obs_mp, n_mp, d_mp_xyz, d_mp_use, d_inv_sigma2, nlevels, d_run,
               min_obs, cap_kf, d_best, d_xyz, d_uv, d_w, d_edges, nullptr, d_skip, d_n_obs);
    SE2_CUDA(cudaGetLastError());
    return launch(B, d_Tcw, d_edges, cap_kf, d_skip, d_xyz, d_uv, d_w, p, 0, nullptr, d_iterations, d_status, nullptr, nullptr, s);
}
