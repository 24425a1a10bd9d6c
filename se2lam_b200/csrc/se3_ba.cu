// SE(3)-XYZ window bundle adjustment: the graph of Map::loadLocalGraph (reference src/Map.cpp:414-566) and of
// Map::loadLocalGraphOnlyBa (:568-698), optimised by g2o's OptimizationAlgorithmLevenberg (DESIGN.md section 12).
// One VertexSE3Expmap per keyframe (estimate toSE3Quat(Tcw)), optionally with the plane-motion EdgeSE3ExpmapPrior, one
// EdgeSE3Expmap per odometry link, one marginalised VertexSBAPointXYZ per map point and one Huber EdgeProjectXYZ2UV per
// observation.
//
// The host plans the call (se3_ba_plan.h: the reduced system's RCM order and 6 x 6 block envelope, and fixed-order gather
// lists); the whole optimize() is then ONE cooperative kernel over as many CTAs as are co-resident, its phases
// separated by grid-wide barriers. Landmark work (linearisation, Hll, (Hll + lambda I)^-1, the Schur complement, the back
// substitution, the trial chi2) is spread over every CTA; the reduced system is factorised and solved by CTA 0 with
// envelope.h. Every sum is a gather in a fixed order, and every reduction over items runs over fixed chunks of 256 items
// whose sums are added in chunk order, so the bytes depend neither on scheduling nor on the grid size. The LM decisions
// are taken on the device by CTA 0's thread 0; the host reads nothing until the call's outputs.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.h"
#include "envelope.h"
#include "lm.h"
#include "se3_ba_plan.h"
#include "se3expmap.h"
#include "sym3.h"

using namespace se2gpu;
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = kThreads;  // items per partial sum
constexpr int kLin = 72;          // per projection edge: Hpp (36), bp (6), Hpl (18, pose-major), Hll (6 upper), bl (3), pad

struct Ctl {  // the LM state, written by CTA 0's thread 0 between barriers
    double cur, lambda, ni, rho, chi_before;
    int buf, ok, more, stop, qmax, failed, accepted, last_failed;
};

struct KArgs {
    int N, O, L, E, nf, iterations, n_chunks;
    double fx, cx, cy, delta, cut;
    float Tbc[16];
    float xrot, yrot, zinfo;
    // inputs (device)
    const float* Tcw; const float* measure; const float* info; const float* xyz; const float* uv; const float* w;
    // plan
    const int* kf_flags;   // [N] bit 0 fixed, bit 1 prior
    const int* pos;        // [N] RCM position of a free keyframe, -1 otherwise
    const int* vert; const int* first; const long long* rowoff; const int* col_ptr; const int* col_rows;
    const int* odo_from; const int* odo_to;
    const int* diag_ptr; const int* diag_code; const long long* off_blk; const int* off_ptr; const int* off_code; int S;
    const int* kf_ptr; const int* kf_edges;    // [nf + 1], projection edges of the keyframe at each position
    const int* pt_ptr; const int* pt_edges;    // [L + 1], each point's edges, ascending
    const int* e_pt; const int* e_kf;          // [E]
    const long long* pair_ptr; const int* pair_a; const int* pair_b;  // [env + 1], Schur pairs of every envelope block
    // work
    SE3* X[2];        // [N] poses, current / trial
    double* P[2];     // [3 L] points
    SE3* pmeas; double* pinfo;   // [N], [36 N] priors
    SE3* Z; double* Om; double* olin;  // odometry: measurements, informations, records [O * kEdgeRec]
    double* lin;      // [E * kLin]
    double* Y;        // [E * 18] Hpl_e (Hll + lambda I)^-1, pose-major
    double* Hl;       // [L * 9] Hll upper, bl
    double* D;        // [L * 6] (Hll + lambda I)^-1 upper
    double* pH; double* pb;   // [36 nf], [6 nf] prior blocks by position
    double* Hs;       // [env * 36] pose blocks of H (prior, odometry, projection)
    double* bf;       // [6 nf] pose part of b
    double* L_;       // [env * 36] the damped Schur complement, factorised in place
    double* b;        // [6 nf] reduced right-hand side
    double* x;        // [6 nf]
    double* part;     // [n_chunks]
    double* part_max; // [grid]
    Ctl* ctl;
    // outputs
    float* Tcw_out; float* xyz_out; double* poses; double* points; double* chi2; uint8_t* outlier;
    int* status; int* iters; se2gpu_ba_iter_stats* stats; double* trace;
};

// the view envelope.h reads
struct Env {
    int nf;
    const int* first; const long long* rowoff; const int* col_ptr; const int* col_rows;
    double* L; double* b; double* x;
};

// one EdgeProjectXYZ2UV at the poses X and points P: robust chi2 (raw into *raw when given)
__device__ inline double proj_chi2(const KArgs& a, const SE3* X, const double* P, int e, double* raw) {
    double err[2];
    const double c2 = xyz2uv_terms(X[a.e_kf[e]], P + 3 * (size_t)a.e_pt[e], a.uv + 2 * (size_t)e, (double)a.w[e], a, err, nullptr, nullptr);
    if (raw) *raw = c2;
    return huber(c2, a.delta, nullptr);
}

// item i of the chi2 sum: projection edges, then priors, then odometry
__device__ inline double chi2_item(const KArgs& a, const SE3* X, const double* P, int i) {
    if (i < a.E) return proj_chi2(a, X, P, i, nullptr);
    i -= a.E;
    if (i < a.N) {
        if (!(a.kf_flags[i] & 2)) return 0.0;
        double e[6];
        return prior_error(a.pmeas[i], a.pinfo + 36 * (size_t)i, X[i], e);
    }
    i -= a.N;
    double e[6];
    return expmap_edge(a.Z[i], a.Om + 36 * (size_t)i, X[a.odo_from[i]], X[a.odo_to[i]], e, nullptr, nullptr);
}

// fixed-order sum of f(i) over n items: chunk sums by the CTAs, then (after a grid barrier) the chunk sums in order by
// CTA 0's thread 0, returned there
template <class F>
__device__ double grid_sum(const KArgs& a, int n, F f, double (&s_red)[kWarps][1], cg::grid_group& grid) {
    const int chunks = (n + kChunk - 1) / kChunk;
    for (int c = blockIdx.x; c < chunks; c += gridDim.x) {
        const int i = c * kChunk + threadIdx.x;
        double v = i < n ? f(i) : 0.0;
        double t;
        cta_sum<1>(&v, s_red, &t);
        if (threadIdx.x == 0) a.part[c] = t;
    }
    grid.sync();
    double s = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0)
        for (int c = 0; c < chunks; ++c) s += a.part[c];
    return s;
}

__global__ void __launch_bounds__(kThreads, 1) k_se3_ba(KArgs a) {
    cg::grid_group grid = cg::this_grid();
    __shared__ double s_red[kWarps][1], s_D[36];
    __shared__ int s_flag;
    const int tid = threadIdx.x;
    const int gt = blockIdx.x * kThreads + tid, gs = gridDim.x * kThreads;
    const bool lead = blockIdx.x == 0 && tid == 0;
    const size_t env = a.nf ? (size_t)a.rowoff[a.nf] : 0;
    volatile Ctl* ctl = a.ctl;

    // setup: toSE3Quat(Tcw), the priors, the odometry measurements and informations ([trans rot] -> [rot trans])
    for (int v = gt; v < a.N; v += gs) {
        const SE3 T = se3_from_f32(a.Tcw + 16 * (size_t)v);
        a.X[0][v] = T; a.X[1][v] = T;
        if (a.kf_flags[v] & 2) plane_motion_prior(T, a, &a.pmeas[v], a.pinfo + 36 * (size_t)v);
    }
    for (int j = gt; j < 3 * a.L; j += gs) a.P[0][j] = a.P[1][j] = (double)a.xyz[j];
    for (int o = gt; o < a.O; o += gs) {
        a.Z[o] = se3_from_f32(a.measure + 16 * (size_t)o);
        const float* I = a.info + 36 * (size_t)o;
        double* M = a.Om + 36 * (size_t)o;
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {  // addEdgeSE3Expmap (src/optimizer.cpp:489-494)
                const int sr = r < 3 ? r + 3 : r - 3, sc = c < 3 ? c + 3 : c - 3;
                M[r * 6 + c] = (double)I[sr * 6 + sc];
            }
    }
    for (size_t i = gt; i < env * 36; i += gs) a.Hs[i] = 0;
    grid.sync();
    {
        const double c = grid_sum(a, a.E + a.N + a.O, [&](int i) { return chi2_item(a, a.X[0], a.P[0], i); }, s_red, grid);
        if (lead) { ctl->cur = c; ctl->buf = 0; ctl->stop = 0; ctl->last_failed = 0; }
    }
    // g2o's optimize() returns before its first iteration when no vertex is free (a point is free when it has an edge)
    const int iterations = a.nf > 0 || a.E > 0 ? a.iterations : 0;
    int it = 0;
    for (; it < iterations; ++it) {
        grid.sync();
        const int buf = ctl->buf;
        const SE3* X = a.X[buf];
        const double* P = a.P[buf];
        SE3* Xt = a.X[buf ^ 1];
        double* Pt = a.P[buf ^ 1];
        // linearise: projection edges, odometry, priors of the free keyframes
        for (int e = gt; e < a.E; e += gs) {
            double err[2], Jp[12], Jl[6];
            const double w = a.w[e];
            const double c2 = xyz2uv_terms(X[a.e_kf[e]], P + 3 * (size_t)a.e_pt[e], a.uv + 2 * (size_t)e, w, a, err, Jp, Jl);
            double rho1;
            huber(c2, a.delta, &rho1);
            const double W = rho1 * w, r0 = -(w * err[0]) * rho1, r1 = -(w * err[1]) * rho1;
            double* o = a.lin + kLin * (size_t)e;
            if (a.pos[a.e_kf[e]] >= 0) {
                for (int r = 0; r < 6; ++r) {
                    for (int c = 0; c < 6; ++c) o[r * 6 + c] = (Jp[r] * W) * Jp[c] + (Jp[6 + r] * W) * Jp[6 + c];
                    o[36 + r] = Jp[r] * r0 + Jp[6 + r] * r1;
                    for (int c = 0; c < 3; ++c) o[42 + r * 3 + c] = (Jp[r] * W) * Jl[c] + (Jp[6 + r] * W) * Jl[3 + c];
                }
            }
            int k = 0;
            for (int r = 0; r < 3; ++r) {
                for (int c = r; c < 3; ++c) o[60 + k++] = (Jl[r] * W) * Jl[c] + (Jl[3 + r] * W) * Jl[3 + c];
                o[66 + r] = Jl[r] * r0 + Jl[3 + r] * r1;
            }
        }
        for (int o = gt; o < a.O; o += gs) {
            double e[6], J[2][36];
            const double* Om = a.Om + 36 * (size_t)o;
            expmap_edge(a.Z[o], Om, X[a.odo_from[o]], X[a.odo_to[o]], e, J[0], J[1]);
            edge_record(Om, e, J, a.olin + kEdgeRec * (size_t)o);
        }
        for (int p = gt; p < a.nf; p += gs) {  // EdgeSE3ExpmapPrior, J = -I: H += Omega, b += Omega e
            const int v = a.vert[p];
            double* H = a.pH + 36 * (size_t)p;
            double* bb = a.pb + 6 * (size_t)p;
            if (!(a.kf_flags[v] & 2)) {
                for (int k = 0; k < 36; ++k) H[k] = 0;
                for (int k = 0; k < 6; ++k) bb[k] = 0;
                continue;
            }
            double e[6];
            const double* I = a.pinfo + 36 * (size_t)v;
            prior_error(a.pmeas[v], I, X[v], e);
            for (int r = 0; r < 6; ++r) {
                double we = 0;
                for (int c = 0; c < 6; ++c) { H[r * 6 + c] = I[r * 6 + c]; we += I[r * 6 + c] * e[c]; }
                bb[r] = we;
            }
        }
        grid.sync();
        // gather: the points' Hll and bl, the pose blocks of H and b, and max |diag H| for lambda_0
        double m = 0;
        for (int j = gt; j < a.L; j += gs) {
            double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int q = a.pt_ptr[j]; q < a.pt_ptr[j + 1]; ++q) {
                const double* o = a.lin + kLin * (size_t)a.pt_edges[q] + 60;
                for (int k = 0; k < 9; ++k) h[k] += o[k];
            }
            for (int k = 0; k < 9; ++k) a.Hl[9 * (size_t)j + k] = h[k];
            m = fmax(m, fmax(fabs(h[0]), fmax(fabs(h[3]), fabs(h[5]))));
        }
        const auto all = [](int) { return true; };
        gather_diag(a, a.olin, a.bf, gt, gs, all, [&](int p, int rc, double s) {  // the projection edges after the odometry
            for (int q = a.kf_ptr[p]; q < a.kf_ptr[p + 1]; ++q) s += a.lin[kLin * (size_t)a.kf_edges[q] + rc];
            if (rc < 36 && rc % 7 == 0) m = fmax(m, fabs(s));
            return s;
        });
        gather_off(a, a.olin, gt, gs, all);
        if (it == 0) {
            m = cta_max(m, s_red);
            if (tid == 0) a.part_max[blockIdx.x] = m;
        }
        grid.sync();
        if (lead) {
            if (it == 0) {  // computeLambdaInit over every free vertex, landmarks included
                double mm = 0;
                for (int g = 0; g < (int)gridDim.x; ++g) mm = fmax(mm, a.part_max[g]);
                double lam, ni;
                lm_lambda_init(mm, lam, ni);
                ctl->lambda = lam; ctl->ni = ni;
            }
            ctl->chi_before = ctl->cur; ctl->qmax = 0; ctl->failed = 0; ctl->accepted = 0; ctl->rho = 0;
        }
        for (;;) {
            grid.sync();
            const double lambda = ctl->lambda;
            // (Hll + lambda I)^-1 and Y_e = Hpl_e (Hll + lambda I)^-1 for every edge to a free keyframe
            for (int j = gt; j < a.L; j += gs) {
                const double* h = a.Hl + 9 * (size_t)j;
                const Sym3Inv inv = sym3_inverse(h[0] + lambda, h[1], h[2], h[3] + lambda, h[4], h[5] + lambda);
                const double Dm[9] = {inv.i00, inv.i01, inv.i02, inv.i01, inv.i11, inv.i12, inv.i02, inv.i12, inv.i22};
                double* d = a.D + 6 * (size_t)j;
                d[0] = inv.i00; d[1] = inv.i01; d[2] = inv.i02; d[3] = inv.i11; d[4] = inv.i12; d[5] = inv.i22;
                for (int q = a.pt_ptr[j]; q < a.pt_ptr[j + 1]; ++q) {
                    const int e = a.pt_edges[q];
                    if (a.pos[a.e_kf[e]] < 0) continue;
                    const double* W = a.lin + kLin * (size_t)e + 42;
                    double* y = a.Y + 18 * (size_t)e;
                    for (int r = 0; r < 6; ++r)
                        for (int c = 0; c < 3; ++c) y[r * 3 + c] = W[r * 3] * Dm[c] + W[r * 3 + 1] * Dm[3 + c] + W[r * 3 + 2] * Dm[6 + c];
                }
            }
            grid.sync();
            // the damped Schur complement S = H_pp + lambda I - sum Y_a Hpl_b^T and the reduced b
            for (size_t idx = gt; idx < env * 36; idx += gs) {
                const size_t k = idx / 36;
                const int rc = (int)(idx % 36), r = rc / 6, c = rc % 6;
                double s = a.Hs[idx];
                for (long long q = a.pair_ptr[k]; q < a.pair_ptr[k + 1]; ++q) {
                    const double* y = a.Y + 18 * (size_t)a.pair_a[q] + r * 3;
                    const double* W = a.lin + kLin * (size_t)a.pair_b[q] + 42 + c * 3;
                    s -= y[0] * W[0] + y[1] * W[1] + y[2] * W[2];
                }
                a.L_[idx] = s;
            }
            for (int idx = gt; idx < a.nf * 6; idx += gs) {
                const int p = idx / 6, r = idx % 6;
                double s = a.bf[idx];
                for (int q = a.kf_ptr[p]; q < a.kf_ptr[p + 1]; ++q) {
                    const int e = a.kf_edges[q];
                    const double* y = a.Y + 18 * (size_t)e + r * 3;
                    const double* bl = a.Hl + 9 * (size_t)a.e_pt[e] + 6;
                    s -= y[0] * bl[0] + y[1] * bl[1] + y[2] * bl[2];
                }
                a.b[idx] = s;
            }
            grid.sync();
            damp(a, a.L_, lambda, gt, gs);
            grid.sync();
            // the reduced solve on CTA 0
            if (blockIdx.x == 0) {
                Env en{a.nf, a.first, a.rowoff, a.col_ptr, a.col_rows, a.L_, a.b, a.x};
                const bool ok = env_factor<kThreads>(en, s_D, &s_flag);
                if (ok) env_substitute(en);
                if (tid == 0) ctl->ok = ok;
            }
            grid.sync();
            const bool ok = ctl->ok;
            double temp = DBL_MAX, scale = 0;
            if (ok) {
                // back substitution dl = D (bl - sum Hpl_e^T dp), oplus, and computeScale's terms: poses, then points
                scale = grid_sum(a, a.nf + a.L, [&](int i) {
                    double sc = 0;
                    if (i < a.nf) {
                        const double* d = a.x + 6 * (size_t)i;
                        const int v = a.vert[i];
                        Xt[v] = se3_mul(se3_exp(d), X[v]);
                        for (int r = 0; r < 6; ++r) sc += d[r] * (lambda * d[r] + a.bf[6 * (size_t)i + r]);
                        return sc;
                    }
                    const int j = i - a.nf;
                    if (a.pt_ptr[j + 1] == a.pt_ptr[j]) return 0.0;
                    const double* bl = a.Hl + 9 * (size_t)j + 6;
                    double rr[3] = {bl[0], bl[1], bl[2]};
                    for (int q = a.pt_ptr[j]; q < a.pt_ptr[j + 1]; ++q) {
                        const int e = a.pt_edges[q], p = a.pos[a.e_kf[e]];
                        if (p < 0) continue;
                        const double* W = a.lin + kLin * (size_t)e + 42;
                        const double* dp = a.x + 6 * (size_t)p;
                        for (int c = 0; c < 3; ++c) {
                            double t = 0;
                            for (int r = 0; r < 6; ++r) t += W[r * 3 + c] * dp[r];
                            rr[c] -= t;
                        }
                    }
                    const double* d = a.D + 6 * (size_t)j;
                    const double dl[3] = {d[0] * rr[0] + d[1] * rr[1] + d[2] * rr[2], d[1] * rr[0] + d[3] * rr[1] + d[4] * rr[2],
                                          d[2] * rr[0] + d[4] * rr[1] + d[5] * rr[2]};
                    for (int c = 0; c < 3; ++c) {
                        Pt[3 * (size_t)j + c] = P[3 * (size_t)j + c] + dl[c];
                        sc += dl[c] * (lambda * dl[c] + bl[c]);
                    }
                    return sc;
                }, s_red, grid);
                grid.sync();
                temp = grid_sum(a, a.E + a.N + a.O, [&](int i) { return chi2_item(a, Xt, Pt, i); }, s_red, grid);
            }
            if (lead) {
                double cur = ctl->cur, lam = ctl->lambda, ni = ctl->ni, rho;
                if (!ok) ctl->failed = ctl->failed + 1;
                if (lm_gain_step(temp, scale, ok, cur, lam, ni, rho)) { ctl->buf = ctl->buf ^ 1; ctl->accepted = 1; }
                ctl->cur = cur; ctl->lambda = lam; ctl->ni = ni; ctl->rho = rho;
                ctl->qmax = ctl->qmax + 1;
                ctl->more = lm_retry(rho, ctl->qmax);
            }
            grid.sync();
            if (!ctl->more) break;
        }
        if (lead) {
            const se2gpu_ba_iter_stats st = lm_iter_stats(ctl->chi_before, ctl->cur, ctl->lambda, ctl->rho, ctl->qmax, ctl->accepted);
            ctl->last_failed = lm_not_pd(st, ctl->failed);
            if (a.stats) a.stats[it] = st;
            ctl->stop = st.terminate;
        }
        grid.sync();
        if (a.trace) {  // the estimate after the iteration: N poses (7 doubles), then L points
            const SE3* Xc = a.X[ctl->buf];
            const double* Pc = a.P[ctl->buf];
            double* tr = a.trace + (size_t)it * (7 * (size_t)a.N + 3 * (size_t)a.L);
            for (int v = gt; v < a.N; v += gs) store_pose(Xc[v], tr + 7 * (size_t)v);
            for (int j = gt; j < 3 * a.L; j += gs) tr[7 * (size_t)a.N + j] = Pc[j];
        }
        if (ctl->stop) { ++it; break; }
    }
    grid.sync();
    // outputs: the estimates, and every edge's raw chi2 at them with removeOutlierChi2's cut
    const SE3* X = a.X[ctl->buf];
    const double* P = a.P[ctl->buf];
    for (int v = gt; v < a.N; v += gs) {
        if (a.Tcw_out) {  // a keyframe that is not optimised keeps its input matrix bit for bit
            float* o = a.Tcw_out + 16 * (size_t)v;
            if (a.pos[v] >= 0) se3_to_f32(X[v], o);
            else for (int k = 0; k < 16; ++k) o[k] = a.Tcw[16 * (size_t)v + k];
        }
        if (a.poses) store_pose(X[v], a.poses + 7 * (size_t)v);
    }
    for (int j = gt; j < 3 * a.L; j += gs) {
        if (a.points) a.points[j] = P[j];
        if (a.xyz_out) a.xyz_out[j] = (float)P[j];
    }
    for (int e = gt; e < a.E; e += gs) {
        double c2;
        proj_chi2(a, X, P, e, &c2);
        if (a.chi2) a.chi2[e] = c2;
        if (a.outlier) a.outlier[e] = c2 > a.cut ? 1 : 0;
    }
    if (lead) {
        if (a.iters) *a.iters = it;
        if (a.status) *a.status = ctl->last_failed ? SE2GPU_SE3_BA_NOT_PD : SE2GPU_SE3_BA_OK;
    }
}

bool finite_all(const float* p, size_t n) {
    for (size_t i = 0; i < n; ++i)
        if (!std::isfinite(p[i])) return false;
    return true;
}

int check_params(const se2gpu_se3_ba_params* p) {
    if (!p) return fail(SE2GPU_ERR_INVALID, "null parameters");
    if (p->iterations < 0) return fail(SE2GPU_ERR_INVALID, "iterations = %d", p->iterations);
    if (!(p->fx != 0.f) || !std::isfinite(p->fx) || !std::isfinite(p->cx) || !std::isfinite(p->cy) || !(p->huber_delta > 0.f) ||
        !std::isfinite(p->huber_delta) || !finite_all(p->Tbc, 16) || !std::isfinite(p->xrot_info) || !std::isfinite(p->yrot_info) ||
        !std::isfinite(p->z_info) || std::isnan(p->chi2_cut))
        return fail(SE2GPU_ERR_INVALID, "camera, Huber delta, Tbc, prior informations or chi2 cut not valid");
    return SE2GPU_OK;
}

int check_topology(int N, const uint8_t* fixed, const uint8_t* prior, int O, const int* from, const int* to, int L, int E,
                   const int* e_pt, const int* e_kf) {
    if (N <= 0 || O < 0 || L < 0 || E < 0) return fail(SE2GPU_ERR_INVALID, "N = %d, O = %d, L = %d, E = %d", N, O, L, E);
    if (!fixed || !prior || (O && (!from || !to)) || (E && (!e_pt || !e_kf))) return fail(SE2GPU_ERR_INVALID, "null topology arrays");
    { const int rc = check_se3_links(N, O, from, to, nullptr, nullptr, "odometry", "keyframe"); if (rc) return rc; }
    std::vector<std::vector<int>> seen(L);
    for (int e = 0; e < E; ++e) {
        if (e_pt[e] < 0 || e_pt[e] >= L || e_kf[e] < 0 || e_kf[e] >= N) return fail(SE2GPU_ERR_INVALID, "edge %d: index out of range", e);
        seen[e_pt[e]].push_back(e_kf[e]);
    }
    for (int j = 0; j < L; ++j) {
        std::sort(seen[j].begin(), seen[j].end());
        if (std::adjacent_find(seen[j].begin(), seen[j].end()) != seen[j].end())
            return fail(SE2GPU_ERR_INVALID, "point %d: two edges to one keyframe", j);
    }
    return SE2GPU_OK;
}

int check_values(int N, const float* Tcw, int O, const int* from, const int* to, const float* measure, const float* info, int L,
                 const float* xyz, int E, const float* uv, const float* w) {
    if (!Tcw || (O && (!measure || !info)) || (L && !xyz) || (E && (!uv || !w))) return fail(SE2GPU_ERR_INVALID, "null arrays");
    if (!finite_all(Tcw, 16 * (size_t)N)) return fail(SE2GPU_ERR_INVALID, "Tcw not finite");
    { const int rc = check_se3_links(N, O, from, to, measure, info, "odometry", "keyframe"); if (rc) return rc; }
    if (!finite_all(xyz, 3 * (size_t)L) || !finite_all(uv, 2 * (size_t)E) || !finite_all(w, (size_t)E))
        return fail(SE2GPU_ERR_INVALID, "points or observations not finite");
    for (int e = 0; e < E; ++e)
        if (!(w[e] > 0.f)) return fail(SE2GPU_ERR_INVALID, "edge %d: invSigma2 not positive", e);
    return SE2GPU_OK;
}

}  // namespace

struct se2gpu_se3_ba_ctx : se2gpu::PlanContext {
    int grid_limit = 0;  // SE2GPU_SE3_BA_GRID: cap on the cooperative grid (several contexts on one GPU); 0 = none
};

namespace {

struct Outs {
    float* Tcw; float* xyz; double* poses; double* points; double* chi2; uint8_t* outlier; int* status; int* iters;
    se2gpu_ba_iter_stats* stats; double* trace;
};

int run(se2gpu_se3_ba_ctx* h, int N, const uint8_t* fixed, const uint8_t* prior, int O, const int* from, const int* to, int L,
        int E, const int* e_pt, const int* e_kf, const float* d_Tcw, const float* d_measure, const float* d_info,
        const float* d_xyz, const float* d_uv, const float* d_w, const se2gpu_se3_ba_params* prm, const Outs& out,
        cudaStream_t stream) {
    const se3ba::Plan P = se3ba::make_plan(N, fixed, prior, O, from, to, L, E, e_pt, e_kf);
    const int nf = P.G.n_free;
    const size_t env = (size_t)P.G.env_blocks();
    const int n_items = std::max(E + N + O, nf + L);
    const int n_chunks = std::max(1, (n_items + kChunk - 1) / kChunk);
    int dev_sms = 0, per_sm = 0;
    SE2_CUDA(cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device));
    SE2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_se3_ba, kThreads, 0));
    if (per_sm < 1) return fail(SE2GPU_ERR_CUDA, "k_se3_ba cannot be resident");
    const size_t work = std::max<size_t>({(size_t)E, (size_t)L * 3, env * 36, (size_t)N, (size_t)O});
    int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)dev_sms * per_sm, (work + kThreads - 1) / kThreads));
    if (h->grid_limit >= 1) grid = std::min(grid, h->grid_limit);
    // the plan, the window's topology, then the work
    Packed<int> ints;
    Packed<long long> lls;
    Layout dbl;
    struct {
        size_t flags, pos, vert, first, col_ptr, col_rows, diag_ptr, diag_code, off_ptr, off_code, kf_ptr, kf_edges, pt_ptr,
            pt_edges, pair_a, pair_b, e_pt, e_kf, odo_from, odo_to;                                               // ints
        size_t rowoff, off_blk, pair_ptr;                                                                       // long longs
        size_t X[2], P[2], pmeas, pinfo, Z, Om, olin, lin, Y, Hl, D, pH, pb, bf, b, x, Hs, L, part, part_max, ctl;  // doubles
    } o;
    o.flags = ints.put(P.flags); o.pos = ints.put(P.G.pos); o.vert = ints.put(P.G.vert); o.first = ints.put(P.G.first);
    o.col_ptr = ints.put(P.G.col_ptr); o.col_rows = ints.put(P.G.col_rows); o.diag_ptr = ints.put(P.diag_ptr);
    o.diag_code = ints.put(P.diag_code); o.off_ptr = ints.put(P.off_ptr); o.off_code = ints.put(P.off_code);
    o.kf_ptr = ints.put(P.kf_ptr); o.kf_edges = ints.put(P.kf_edges); o.pt_ptr = ints.put(P.pt_ptr); o.pt_edges = ints.put(P.pt_edges);
    o.pair_a = ints.put(P.pair_a); o.pair_b = ints.put(P.pair_b); o.e_pt = ints.put(e_pt, (size_t)E); o.e_kf = ints.put(e_kf, (size_t)E);
    o.odo_from = ints.put(from, (size_t)O); o.odo_to = ints.put(to, (size_t)O);
    o.rowoff = lls.put(P.G.rowoff); o.off_blk = lls.put(P.off_blk); o.pair_ptr = lls.put(P.pair_ptr);
    o.X[0] = dbl.take(7 * (size_t)N); o.X[1] = dbl.take(7 * (size_t)N); o.P[0] = dbl.take(3 * (size_t)L); o.P[1] = dbl.take(3 * (size_t)L);
    o.pmeas = dbl.take(7 * (size_t)N); o.pinfo = dbl.take(36 * (size_t)N); o.Z = dbl.take(7 * (size_t)O); o.Om = dbl.take(36 * (size_t)O);
    o.olin = dbl.take(kEdgeRec * (size_t)O); o.lin = dbl.take(kLin * (size_t)E); o.Y = dbl.take(18 * (size_t)E);
    o.Hl = dbl.take(9 * (size_t)L); o.D = dbl.take(6 * (size_t)L); o.pH = dbl.take(36 * (size_t)nf); o.pb = dbl.take(6 * (size_t)nf);
    o.bf = dbl.take(6 * (size_t)nf); o.b = dbl.take(6 * (size_t)nf); o.x = dbl.take(6 * (size_t)nf); o.Hs = dbl.take(36 * env);
    o.L = dbl.take(36 * env); o.part = dbl.take((size_t)n_chunks); o.part_max = dbl.take((size_t)grid); o.ctl = dbl.take(sizeof(Ctl) / 8 + 1);
    { const int rc = h->grow(&h->d_dbl, &h->cap_dbl, dbl.size); if (rc) return rc; }
    { const int rc = h->upload_plan(ints.data, lls.data, stream); if (rc) return rc; }

    KArgs a{};
    a.N = N; a.O = O; a.L = L; a.E = E; a.nf = nf; a.iterations = prm->iterations; a.n_chunks = n_chunks;
    a.fx = prm->fx; a.cx = prm->cx; a.cy = prm->cy; a.delta = prm->huber_delta; a.cut = prm->chi2_cut;
    std::memcpy(a.Tbc, prm->Tbc, sizeof a.Tbc);
    a.xrot = prm->xrot_info; a.yrot = prm->yrot_info; a.zinfo = prm->z_info;
    a.Tcw = d_Tcw; a.measure = d_measure; a.info = d_info; a.xyz = d_xyz; a.uv = d_uv; a.w = d_w;
    const int* I = h->d_int;
    a.kf_flags = I + o.flags; a.pos = I + o.pos; a.vert = I + o.vert; a.first = I + o.first; a.col_ptr = I + o.col_ptr;
    a.col_rows = I + o.col_rows; a.diag_ptr = I + o.diag_ptr; a.diag_code = I + o.diag_code; a.off_ptr = I + o.off_ptr;
    a.off_code = I + o.off_code; a.kf_ptr = I + o.kf_ptr; a.kf_edges = I + o.kf_edges; a.pt_ptr = I + o.pt_ptr;
    a.pt_edges = I + o.pt_edges; a.pair_a = I + o.pair_a; a.pair_b = I + o.pair_b; a.e_pt = I + o.e_pt; a.e_kf = I + o.e_kf;
    a.odo_from = I + o.odo_from; a.odo_to = I + o.odo_to;
    a.rowoff = h->d_ll + o.rowoff; a.off_blk = h->d_ll + o.off_blk; a.pair_ptr = h->d_ll + o.pair_ptr; a.S = (int)P.off_blk.size();
    double* D = h->d_dbl;
    a.X[0] = (SE3*)(D + o.X[0]); a.X[1] = (SE3*)(D + o.X[1]); a.P[0] = D + o.P[0]; a.P[1] = D + o.P[1];
    a.pmeas = (SE3*)(D + o.pmeas); a.pinfo = D + o.pinfo; a.Z = (SE3*)(D + o.Z); a.Om = D + o.Om; a.olin = D + o.olin;
    a.lin = D + o.lin; a.Y = D + o.Y; a.Hl = D + o.Hl; a.D = D + o.D; a.pH = D + o.pH; a.pb = D + o.pb; a.bf = D + o.bf;
    a.b = D + o.b; a.x = D + o.x; a.Hs = D + o.Hs; a.L_ = D + o.L; a.part = D + o.part; a.part_max = D + o.part_max;
    a.ctl = (Ctl*)(D + o.ctl);
    a.Tcw_out = out.Tcw; a.xyz_out = out.xyz; a.poses = out.poses; a.points = out.points; a.chi2 = out.chi2; a.outlier = out.outlier;
    a.status = out.status; a.iters = out.iters; a.stats = out.stats; a.trace = out.trace;
    const size_t it = (size_t)prm->iterations;
    if (out.stats && it) SE2_CUDA(cudaMemsetAsync(out.stats, 0, sizeof(se2gpu_ba_iter_stats) * it, stream));
    if (out.trace && it) SE2_CUDA(cudaMemsetAsync(out.trace, 0, sizeof(double) * it * (7 * (size_t)N + 3 * (size_t)L), stream));
    SE2_NVTX("se2gpu_se3_ba");
    void* args[] = {&a};
    SE2_CUDA(cudaLaunchCooperativeKernel((const void*)k_se3_ba, grid, kThreads, args, 0, stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);  // the one launch of the call (SE2_LAUNCH cannot launch cooperatively)
    SE2_CUDA(cudaGetLastError());
    SE2_CUDA(cudaEventRecord(h->done, stream));
    return SE2GPU_OK;
}

int host_run(se2gpu_se3_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O, const int* odo_from,
             const int* odo_to, const float* odo_measure, const float* odo_info, int L, const float* xyz, int E, const int* edge_point,
             const int* edge_kf, const float* uv, const float* inv_sigma2, const se2gpu_se3_ba_params* params, double* chi2,
             uint8_t* outlier, int* status, int* iterations, se2gpu_ba_iter_stats* stats, double* poses, double* points,
             float* Tcw_out, float* xyz_out, double* trace) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null context");
    { const int rc = check_params(params); if (rc) return rc; }
    { const int rc = check_topology(N, fixed, prior, O, odo_from, odo_to, L, E, edge_point, edge_kf); if (rc) return rc; }
    { const int rc = check_values(N, Tcw, O, odo_from, odo_to, odo_measure, odo_info, L, xyz, E, uv, inv_sigma2); if (rc) return rc; }
    if (E && (!chi2 || !outlier)) return fail(SE2GPU_ERR_INVALID, "null chi2 / outlier outputs");
    HostStage st(h->device);
    if (const int rc = st.status()) return rc;
    const size_t it = (size_t)params->iterations;
    Outs o{};
    const float* dT = st.upload(Tcw, 16 * (size_t)N);
    const float* dm = st.upload(odo_measure, 16 * (size_t)O);
    const float* di = st.upload(odo_info, 36 * (size_t)O);
    const float* dx = st.upload(xyz, 3 * (size_t)L);
    const float* du = st.upload(uv, 2 * (size_t)E);
    const float* dw = st.upload(inv_sigma2, (size_t)E);
    o.chi2 = E ? st.output(chi2, (size_t)E) : nullptr;
    o.outlier = E ? st.output(outlier, (size_t)E) : nullptr;
    o.status = status ? st.output(status, 1) : nullptr;
    o.iters = iterations ? st.output(iterations, 1) : nullptr;
    o.stats = stats && it ? st.output(stats, it) : nullptr;
    o.poses = poses ? st.output(poses, 7 * (size_t)N) : nullptr;
    o.points = points && L ? st.output(points, 3 * (size_t)L) : nullptr;
    o.Tcw = Tcw_out ? st.output(Tcw_out, 16 * (size_t)N) : nullptr;
    o.xyz = xyz_out && L ? st.output(xyz_out, 3 * (size_t)L) : nullptr;
    o.trace = trace && it ? st.output(trace, it * (7 * (size_t)N + 3 * (size_t)L)) : nullptr;
    if (const int rc = st.status()) return rc;
    // h->stream is a blocking stream: the staged copies on the legacy stream order themselves around the kernel
    { const int rc = run(h, N, fixed, prior, O, odo_from, odo_to, L, E, edge_point, edge_kf, dT, dm, di, dx, du, dw, params, o, h->stream); if (rc) return rc; }
    return st.finish();
}

}  // namespace

se2gpu_se3_ba_ctx* se2gpu_se3_ba_create(int device) {
    se2gpu_se3_ba_ctx* h = create_plan_context<se2gpu_se3_ba_ctx>(device);
    if (h)
        if (const char* g = getenv("SE2GPU_SE3_BA_GRID")) h->grid_limit = atoi(g);  // the only place this BA reads the environment
    return h;
}

void se2gpu_se3_ba_destroy(se2gpu_se3_ba_ctx* h) { delete h; }

int se2gpu_se3_ba(se2gpu_se3_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O, const int* odo_from,
                  const int* odo_to, const float* odo_measure, const float* odo_info, int L, const float* xyz, int E,
                  const int* edge_point, const int* edge_kf, const float* uv, const float* inv_sigma2,
                  const se2gpu_se3_ba_params* params, double* chi2, uint8_t* outlier, int* status, int* iterations,
                  se2gpu_ba_iter_stats* stats, double* poses, double* points, float* Tcw_out, float* xyz_out) {
    return host_run(h, N, Tcw, fixed, prior, O, odo_from, odo_to, odo_measure, odo_info, L, xyz, E, edge_point, edge_kf, uv, inv_sigma2,
                    params, chi2, outlier, status, iterations, stats, poses, points, Tcw_out, xyz_out, nullptr);
}

int se2gpu_se3_ba_debug_trace(se2gpu_se3_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O,
                              const int* odo_from, const int* odo_to, const float* odo_measure, const float* odo_info, int L,
                              const float* xyz, int E, const int* edge_point, const int* edge_kf, const float* uv,
                              const float* inv_sigma2, const se2gpu_se3_ba_params* params, double* chi2, uint8_t* outlier,
                              int* status, int* iterations, se2gpu_ba_iter_stats* stats, double* poses, double* points,
                              double* trace) {
    return host_run(h, N, Tcw, fixed, prior, O, odo_from, odo_to, odo_measure, odo_info, L, xyz, E, edge_point, edge_kf, uv, inv_sigma2,
                    params, chi2, outlier, status, iterations, stats, poses, points, nullptr, nullptr, trace);
}

int se2gpu_se3_ba_device(se2gpu_se3_ba_ctx* h, int N, const float* d_Tcw, const uint8_t* fixed, const uint8_t* prior, int O,
                         const int* odo_from, const int* odo_to, const float* d_odo_measure, const float* d_odo_info, int L,
                         const float* d_xyz, int E, const int* edge_point, const int* edge_kf, const float* d_uv,
                         const float* d_inv_sigma2, const se2gpu_se3_ba_params* params, double* d_chi2, uint8_t* d_outlier,
                         int* d_status, int* d_iterations, se2gpu_ba_iter_stats* d_stats, double* d_poses, double* d_points,
                         float* d_Tcw_out, float* d_xyz_out, void* stream) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null context");
    { const int rc = check_params(params); if (rc) return rc; }
    { const int rc = check_topology(N, fixed, prior, O, odo_from, odo_to, L, E, edge_point, edge_kf); if (rc) return rc; }
    if (!d_Tcw || (O && (!d_odo_measure || !d_odo_info)) || (L && !d_xyz) || (E && (!d_uv || !d_inv_sigma2)))
        return fail(SE2GPU_ERR_INVALID, "null arrays");
    { const int rc = select_device(h->device); if (rc) return rc; }
    Outs o{d_Tcw_out, d_xyz_out, d_poses, d_points, d_chi2, d_outlier, d_status, d_iterations, d_stats, nullptr};
    return run(h, N, fixed, prior, O, odo_from, odo_to, L, E, edge_point, edge_kf, d_Tcw, d_odo_measure, d_odo_info, d_xyz, d_uv,
               d_inv_sigma2, params, o, (cudaStream_t)stream);
}
