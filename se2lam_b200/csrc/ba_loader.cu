// Loader side of the local BA (SURVEY.md section 8f N1).
//
// se2gpu_ba_build_information: what Map::loadLocalGraph computes per EdgeSE2XYZ right before handing the graph to the
// optimiser (reference src/Map.cpp:1024-1049) - the 2x2 information matrix
//   Omega = (sigma_rot * J_rotxy J_rotxy^T + sigma_z * J_z J_z^T + sigma_l^2 I)^-1
// evaluated ONCE at load time from the keyframe's float Tcw / Twb, the float camera-frame measurement mViewMPs[ftrIdx],
// the float landmark position and mvLevelSigma2[octave]; all arithmetic in double on the widened floats, like the
// reference's toVector3d / toMatrix3d conversions. One thread per edge, coalesced SoA reads, three doubles out.
//
// se2gpu_ba_set_problem: the window of one localBA call -> the device arrays of the context, in four steps, each written once:
//   same_topology                   the graph structure is the loaded one: only the values are gathered and uploaded
//   gather_values                   measurements and information in landmark-sorted edge order, the odometry as SoA
//   plan_window                     host only: everything initializeOptimization / buildStructure derive from the structure
//   upload_window / upload_values   one copy per array
#include <chrono>

#include "ba_context.h"

using namespace se2ba;

namespace {

using se2gpu::fail;
using se2gpu::PinnedArena;

struct InfoArgs {
    int P, L, E;
    const float* lc;          // [E*3] pKF->mViewMPs[ftrIdx]
    const int* edge_pose;     // [E] keyframe slot
    const int* edge_point;    // [E] landmark slot
    const int* octave;        // [E]
    const float* Rcw;         // [P*9] rows of pKF->Tcw(0:3,0:3)
    const float* twb;         // [P*2] pKF->Twb.x, .y
    const float* lw;          // [L*3] pMP->getPos()
    const float* level_sigma2;  // [nlevels] mvLevelSigma2
    int nlevels;
    float fx, sigma_rotxy, sigma_z;
    double* info;             // [E*3] xx, xy, yy
};

__global__ void __launch_bounds__(256) k_edge_information(InfoArgs a) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.E) return;
    const int p = a.edge_pose[e], j = a.edge_point[e];
    if (p < 0 || p >= a.P || j < 0 || j >= a.L) {   // only the device entry can get here (the host one checks first)
        for (int q = 0; q < 3; ++q) a.info[3 * (size_t)e + q] = __longlong_as_double(0x7ff8000000000000LL);
        return;
    }
    int oc = a.octave[e];
    oc = oc < 0 ? 0 : (oc >= a.nlevels ? a.nlevels - 1 : oc);
    const double sigma2 = (double)a.level_sigma2[oc];
    const double lc0 = a.lc[3 * e], lc1 = a.lc[3 * e + 1], lc2 = a.lc[3 * e + 2];
    const double zc_inv = 1. / lc2, zc_inv2 = zc_inv * zc_inv;
    const double fx = (double)a.fx;
    const double Jpi[6] = {fx * zc_inv, 0, -fx * lc0 * zc_inv2, 0, fx * zc_inv, -fx * lc1 * zc_inv2};
    double R[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = (double)a.Rcw[9 * (size_t)p + k];
    double M[6];    // J_pi * Rcw (2x3)
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) M[r * 3 + c] = Jpi[r * 3] * R[c] + Jpi[r * 3 + 1] * R[3 + c] + Jpi[r * 3 + 2] * R[6 + c];
    const double d0 = (double)a.lw[3 * (size_t)j] - (double)a.twb[2 * (size_t)p], d1 = (double)a.lw[3 * (size_t)j + 1] - (double)a.twb[2 * (size_t)p + 1];
    const double d2 = (double)a.lw[3 * (size_t)j + 2];
    // (M * skew(d))[:, 0:2] with skew(d) = [[0,-d2,d1],[d2,0,-d0],[-d1,d0,0]];  J_z = -M[:, 2]
    double Jr[4], Jz[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        Jr[r * 2 + 0] = M[r * 3 + 1] * d2 - M[r * 3 + 2] * d1;
        Jr[r * 2 + 1] = -M[r * 3 + 0] * d2 + M[r * 3 + 2] * d0;
        Jz[r] = -M[r * 3 + 2];
    }
    const double sr = (double)a.sigma_rotxy, sz = (double)a.sigma_z;
    // Sigma_all = sr * Jr Jr^T + sz * Jz Jz^T + sigma2 I   (Eigen evaluates (sr*Jr)*Jr^T; the difference is below 1 ulp of the sum)
    const double s00 = (sr * Jr[0]) * Jr[0] + (sr * Jr[1]) * Jr[1] + (sz * Jz[0]) * Jz[0] + sigma2;
    const double s01 = (sr * Jr[0]) * Jr[2] + (sr * Jr[1]) * Jr[3] + (sz * Jz[0]) * Jz[1];
    const double s10 = (sr * Jr[2]) * Jr[0] + (sr * Jr[3]) * Jr[1] + (sz * Jz[1]) * Jz[0];
    const double s11 = (sr * Jr[2]) * Jr[2] + (sr * Jr[3]) * Jr[3] + (sz * Jz[1]) * Jz[1] + sigma2;
    // Matrix2d::inverse(): adjugate / determinant
    const double invdet = 1. / (s00 * s11 - s10 * s01);
    const double i00 = s11 * invdet, i01 = -s01 * invdet, i10 = -s10 * invdet, i11 = s00 * invdet;
    a.info[3 * (size_t)e] = i00;
    a.info[3 * (size_t)e + 1] = 0.5 * (i01 + i10);     // se2gpu_ba_set_problem stores the symmetric part (xx, xy, yy)
    a.info[3 * (size_t)e + 2] = i11;
}

// ================================================================================================= se2gpu_ba_set_problem

// an array set_problem builds on the host: in the page-locked arena (uploaded in place, no staging copy), or in `pageable`
// when the arena is exhausted or unavailable
template <class T>
T* host_array(PinnedArena& built, size_t count, std::vector<T>& pageable) {
    T* q = built.alloc<T>(count);
    if (!q) { pageable.resize(count); q = pageable.data(); }
    return q;
}

// page-locked bytes of the arrays gather_values builds (5 doubles per edge, 9 per odometry edge, alignment slack)
size_t values_bytes(int El, int Ol) { return (size_t)El * 40 + (size_t)Ol * 72 + 64 * 16; }

// --- same graph structure as the loaded window (same vertices, fixed flags, edge endpoints, shard): everything
// initializeOptimization / buildStructure derives is still valid on the device
bool same_topology(const se2gpu_ba* h, int P, int L, int E, int O, const uint8_t* fixed, const int* edge_pose, const int* edge_point,
                   const int* odo_i, const int* odo_j) {
    return h->loaded && P == h->P && L == h->L && E == h->E && O == h->O && h->t_rank == h->rank && h->t_world == h->world &&
           (int)h->t_edge_pose.size() == E && (int)h->t_odo_i.size() == O && (int)h->t_fixed.size() == P &&
           memcmp(h->t_fixed.data(), fixed, P) == 0 &&
           (E == 0 || (memcmp(h->t_edge_pose.data(), edge_pose, sizeof(int) * E) == 0 && memcmp(h->t_edge_point.data(), edge_point, sizeof(int) * E) == 0)) &&
           (O == 0 || (memcmp(h->t_odo_i.data(), odo_i, sizeof(int) * O) == 0 && memcmp(h->t_odo_j.data(), odo_j, sizeof(int) * O) == 0));
}

struct WindowValues {   // what a window with the loaded structure may change
    int El = 0, Ol = 0;
    double *e_u, *e_v, *w00, *w01, *w11;   // [El] measurement and information (xx, xy, yy) per landmark-sorted edge
    double *o_m, *o_w;                     // [3][Ol], [6][Ol] odometry measurement and information, component-major
    std::vector<double> pageable[7];
};

// perm: sorted edge position -> original edge; this rank's El edges and Ol odometry edges
WindowValues gather_values(se2gpu_ba* h, const std::vector<int>& perm, int El, int Ol, const double* uv, const double* info,
                           const double* odo_meas, const double* odo_info) {
    WindowValues v;
    v.El = El; v.Ol = Ol;
    PinnedArena& built = h->arena2;
    v.e_u = host_array(built, El, v.pageable[0]); v.e_v = host_array(built, El, v.pageable[1]);
    v.w00 = host_array(built, El, v.pageable[2]); v.w01 = host_array(built, El, v.pageable[3]); v.w11 = host_array(built, El, v.pageable[4]);
    for (int k = 0; k < El; ++k) {
        const int e = perm[k];
        v.e_u[k] = uv[2 * e]; v.e_v[k] = uv[2 * e + 1];
        v.w00[k] = info[3 * e]; v.w01[k] = info[3 * e + 1]; v.w11[k] = info[3 * e + 2];
    }
    v.o_m = host_array(built, 3 * (size_t)Ol, v.pageable[5]); v.o_w = host_array(built, 6 * (size_t)Ol, v.pageable[6]);
    for (int o = 0; o < Ol; ++o) {
        for (int q = 0; q < 3; ++q) v.o_m[q * (size_t)Ol + o] = odo_meas[3 * o + q];
        for (int q = 0; q < 6; ++q) v.o_w[q * (size_t)Ol + o] = odo_info[6 * o + q];
    }
    return v;
}

struct Decisions {   // what the host decides from the envelope and the per-block work alone (both load paths)
    int tw_m0 = 0, tw_w = 0;         // two-sided reduced solve (Dev::tw_m0)
    int workers = 0, maxlen = 0, uncached = 0;   // persistent kernel: worker CTAs, longest worker list, workers running the uncached Schur sweep
    std::vector<int> colmax, env_idx, tw_cmax1, blk_order;
};

struct WindowPlan : Decisions {   // everything derived from the graph structure alone
    int nf = 0, n = 0, El = 0, Ol = 0, nblk = 0;
    size_t npairs = 0;
    bool sorted_structure = false;   // block and pair lists by comparison sort (nf^2 beyond the dense table)
    std::vector<int> hidx, lm_ptr, perm, pose_ptr, pose_edges, pose_odo_ptr, pose_odo;
    std::vector<int> blk_a, blk_b, blk_pair_ptr, blk_odo_ptr, blk_odo, bmax;
    std::vector<int> plan_in;        // decide()'s inputs: bmax | np | ne
    int *e_pose, *e_hidx, *pair_e1, *pair_e2;   // [El], [El], [npairs], [npairs]
    std::vector<int> pageable[4];
};

// fn(a, b, k1, k2) for every pair of edges (k1, k2) of one landmark whose free poses satisfy a >= b: landmarks in order,
// k1 ascending, k2 ascending - the order of the pairs inside a block of S, i.e. of its gather's summation
template <class F>
void for_each_pair(const std::vector<int>& lm_ptr, const int* e_hidx, F fn) {
    for (size_t j = 0; j + 1 < lm_ptr.size(); ++j)
        for (int k1 = lm_ptr[j]; k1 < lm_ptr[j + 1]; ++k1) {
            const int a = e_hidx[k1];
            if (a < 0) continue;
            for (int k2 = lm_ptr[j]; k2 < lm_ptr[j + 1]; ++k2) {
                const int b = e_hidx[k2];
                if (b >= 0 && b <= a) fn(a, b, k1, k2);
            }
        }
}

// The host's decisions from the monotone envelope bmax [nf] and, per block of S in key order, its pair count np and the
// pose-side edge count ne of a diagonal block (0 off the diagonal): the envelope lists, the two-sided split, the persistent
// kernel's serving order and its uncached workers. O(nf + nblk) apart from the sharded envelope list.
void decide(Decisions& w, int nf, const int* bmax, const int* np, const int* ne, int nblk, int world, int pk_grid, const Switches& sw) {
    const int n = 3 * nf;
    w.colmax.resize(n);
    for (int a = 0; a < nf; ++a) for (int r = 0; r < 3; ++r) w.colmax[3 * a + r] = 3 * bmax[a] + 2;
    // sharded persistent kernel: the entries of [S | bs] the ranks exchange = lower triangle inside the envelope + right-hand side
    if (world > 1 && n <= SMEM_CHOL_MAX_N) {
        for (int c = 0; c < n; ++c) for (int r = c; r <= w.colmax[c]; ++r) w.env_idx.push_back(r * n + c);
        for (int r = 0; r < n; ++r) w.env_idx.push_back(n * n + r);
    }
    // two-sided solve plan: split point m0 with separator w = bmax[m0-1] - m0 + 1 blocks (bmax is monotone), chain max(m0, m1) + w
    int tw_m0 = 0, tw_w = 0;
    if (n <= SMEM_CHOL_MAX_N && nf >= 16 && pk_grid >= 4 && !sw.no_twist) {
        int best = nf;
        for (int m0 = 1; m0 < nf; ++m0) {
            const int sep = bmax[m0 - 1] - m0 + 1, m1 = nf - m0 - sep;
            if (sep < 1 || sep > TW_MAX_W || m1 < 1) continue;
            const int chain = std::max(m0, m1 + 4) + sep;          // + 4: the bottom part is staged element-wise, not by one bulk copy (~4 pivot steps)
            if (chain < best) { best = chain; tw_m0 = m0; tw_w = sep; }
        }
        if (best * 4 > nf * 3) tw_m0 = tw_w = 0;                  // not worth two hand-overs
        if (tw_m0 > 0) {
            // envelope of the index-reversed bottom part: block column b' <-> global block row R = nf-1-b', reaching up to the
            // first block column whose envelope contains R
            const int nb1 = nf - tw_m0;
            std::vector<int> rminb(nf);
            for (int R = 0, C = 0; R < nf; ++R) { while (bmax[C] < R) ++C; rminb[R] = C; }
            w.tw_cmax1.resize(3 * (size_t)nb1);
            for (int b = 0; b < nb1; ++b) {
                int cb = std::min(nf - 1 - rminb[nf - 1 - b], nb1 - 1);
                if (b >= nb1 - tw_w) cb = nb1 - 1;
                for (int r = 0; r < 3; ++r) w.tw_cmax1[3 * b + r] = 3 * cb + 2;
            }
        }
    }
    w.tw_m0 = tw_m0; w.tw_w = tw_w;
    // Serving order of the blocks for the persistent kernel, by longest-processing-time assignment: blocks by decreasing
    // work (pairs + pose-side edges of a diagonal block, which also carries the pose-side gather) to the least loaded worker,
    // at most 12 blocks per worker (the concurrent Schur phase gives every owned block its own warp group).
    // Worker q serves positions q, q + W, q + 2W, ...; unused trailing positions are holes (-1).
    const int W = w.workers = pk_grid > 1 ? pk_grid - (tw_m0 > 0 ? 2 : 1) : 1;
    std::vector<std::pair<long long, int>> byw(nblk);
    for (int b = 0; b < nblk; ++b) byw[b] = {-(long long)(np[b] + 8 + ne[b]), b};
    std::sort(byw.begin(), byw.end());
    std::vector<std::vector<int>> lists(W);
    std::vector<long long> load(W, 0);
    const size_t cap = std::max<size_t>(12, (nblk + W - 1) / W);
    for (auto& it : byw) {
        int best = -1;
        for (int w2 = 0; w2 < W; ++w2) if (lists[w2].size() < cap && (best < 0 || load[w2] < load[best])) best = w2;
        lists[best].push_back(it.second); load[best] += -it.first;
    }
    size_t maxlen = 0;
    for (auto& l : lists) maxlen = std::max(maxlen, l.size());
    w.maxlen = (int)maxlen;
    w.blk_order.assign((size_t)W * maxlen, -1);
    for (int w2 = 0; w2 < W; ++w2) for (size_t i = 0; i < lists[w2].size(); ++i) w.blk_order[i * W + w2] = lists[w2][i];
    // workers whose blocks do not all fit the shared-memory cache (the rule of ba_persistent's prologue): they run the
    // sequential Schur sweep over pair lists in global memory
    const int arena_ints = (int)(pk_dyn_smem_bytes(n) - PK_RED_SCRATCH_BYTES) / 4;
    for (auto& l : lists) {
        int off = 0, no = 0;
        for (int b : l) {
            if (no >= PK_MAXOWN || off + 2 * np[b] + ne[b] > arena_ints) break;
            off += 2 * np[b] + ne[b]; ++no;
        }
        if (no < (int)l.size()) ++w.uncached;
    }
}

// Host code only; `built` receives the per-edge and per-pair index arrays (and is sized here for gather_values' arrays too).
WindowPlan plan_window(PinnedArena& built, int P, int L, int E, int O, const uint8_t* fixed, const int* edge_pose,
                       const int* edge_point, const int* odo_i, const int* odo_j, int rank, int world, int pk_grid, const Switches& sw) {
    WindowPlan w;
    // --- index mapping (SparseOptimizer::buildIndexMapping): free poses in id order
    std::vector<int>& hidx = w.hidx;
    hidx.assign(P, -1);
    int nf = 0;
    for (int i = 0; i < P; ++i) if (!fixed[i]) hidx[i] = nf++;
    const int n = 3 * nf;
    w.nf = nf; w.n = n;
    // --- shard: this rank keeps the edges of landmarks j % world == rank; odometry lives on rank 0
    std::vector<int>& lm_ptr = w.lm_ptr;
    lm_ptr.assign(L + 1, 0);
    for (int e = 0; e < E; ++e) if (edge_point[e] % world == rank) lm_ptr[edge_point[e] + 1]++;
    for (int j = 0; j < L; ++j) lm_ptr[j + 1] += lm_ptr[j];
    const int El = lm_ptr[L];
    w.perm.resize(El);
    { std::vector<int> cursor(lm_ptr.begin(), lm_ptr.end() - 1);
      for (int e = 0; e < E; ++e) if (edge_point[e] % world == rank) w.perm[cursor[edge_point[e]]++] = e; }
    const int Ol = (rank == 0) ? O : 0;
    w.El = El; w.Ol = Ol;
    // the per-edge and per-pair arrays are built directly in page-locked memory (no staging copy before the upload)
    size_t pair_bound = 0;
    for (int j = 0; j < L; ++j) { const size_t k = (size_t)(lm_ptr[j + 1] - lm_ptr[j]); pair_bound += k * (k + 1) / 2; }
    built.reserve((size_t)El * 8 + pair_bound * 8 + values_bytes(El, Ol));
    int *e_pose = w.e_pose = host_array(built, El, w.pageable[0]), *e_hidx = w.e_hidx = host_array(built, El, w.pageable[1]);
    for (int k = 0; k < El; ++k) { const int e = w.perm[k]; e_pose[k] = edge_pose[e]; e_hidx[k] = hidx[edge_pose[e]]; }
    // --- pose CSR over sorted edges, and over odometry edges (code = 2*o + role)
    std::vector<int>& pose_ptr = w.pose_ptr;
    pose_ptr.assign(nf + 1, 0);
    for (int k = 0; k < El; ++k) if (e_hidx[k] >= 0) pose_ptr[e_hidx[k] + 1]++;
    for (int a = 0; a < nf; ++a) pose_ptr[a + 1] += pose_ptr[a];
    w.pose_edges.resize(pose_ptr[nf]);
    { std::vector<int> cur(pose_ptr.begin(), pose_ptr.end() - 1); for (int k = 0; k < El; ++k) if (e_hidx[k] >= 0) w.pose_edges[cur[e_hidx[k]]++] = k; }
    std::vector<int>& pose_odo_ptr = w.pose_odo_ptr;
    pose_odo_ptr.assign(nf + 1, 0);
    for (int o = 0; o < Ol; ++o) { if (hidx[odo_i[o]] >= 0) pose_odo_ptr[hidx[odo_i[o]] + 1]++; if (hidx[odo_j[o]] >= 0) pose_odo_ptr[hidx[odo_j[o]] + 1]++; }
    for (int a = 0; a < nf; ++a) pose_odo_ptr[a + 1] += pose_odo_ptr[a];
    w.pose_odo.resize(pose_odo_ptr[nf]);
    { std::vector<int> cur(pose_odo_ptr.begin(), pose_odo_ptr.end() - 1);
      for (int o = 0; o < Ol; ++o) { int a = hidx[odo_i[o]], b = hidx[odo_j[o]]; if (a >= 0) w.pose_odo[cur[a]++] = 2 * o; if (b >= 0) w.pose_odo[cur[b]++] = 2 * o + 1; } }
    // --- structure of the reduced system (BlockSolver::buildStructure): blocks (a>=b) touched by co-observation or odometry
    // The (edge, edge) pair list of every block, blocks in key order (a*nf + b), pairs inside a block in landmark
    // order: a stable counting sort over a dense nf x nf table when that is small, a comparison sort otherwise.
    struct OdoB { long long key; int code; };
    std::vector<OdoB> odob;
    for (int o = 0; o < Ol; ++o) {
        const int a = hidx[odo_i[o]], b = hidx[odo_j[o]];
        if (a < 0 || b < 0 || a == b) continue;
        // oAij has rows = vertex i, cols = vertex j; the stored block has rows = max index
        if (a > b) odob.push_back({(long long)a * nf + b, 2 * o});
        else odob.push_back({(long long)b * nf + a, 2 * o + 1});
    }
    std::stable_sort(odob.begin(), odob.end(), [](const OdoB& x, const OdoB& y) { return x.key < y.key; });
    std::vector<long long> keys;
    int *pe1 = nullptr, *pe2 = nullptr;
    std::vector<int>& blk_pair_ptr = w.blk_pair_ptr;
    size_t npairs = 0;
    w.sorted_structure = (size_t)nf * nf > ((size_t)1 << 22);
    if (!w.sorted_structure) {
        std::vector<int> cnt((size_t)nf * nf, 0);
        std::vector<uint8_t> used((size_t)nf * nf, 0);
        for_each_pair(lm_ptr, e_hidx, [&](int a, int b, int, int) { cnt[(size_t)a * nf + b]++; ++npairs; });
        for (int a = 0; a < nf; ++a) used[(size_t)a * nf + a] = 1;
        for (auto& p : odob) used[(size_t)p.key] = 1;
        size_t run = 0;
        for (size_t k = 0; k < cnt.size(); ++k) {
            const int c = cnt[k];
            if (c || used[k]) { keys.push_back((long long)k); blk_pair_ptr.push_back((int)run); }
            cnt[k] = (int)run;     // becomes the fill cursor of block k
            run += c;
        }
        blk_pair_ptr.push_back((int)run);
        pe1 = host_array(built, npairs, w.pageable[2]); pe2 = host_array(built, npairs, w.pageable[3]);
        for_each_pair(lm_ptr, e_hidx, [&](int a, int b, int k1, int k2) { const int at = cnt[(size_t)a * nf + b]++; pe1[at] = k1; pe2[at] = k2; });
    } else {
        struct Pair { long long key; int e1, e2; };
        std::vector<Pair> pairs;
        pairs.reserve((size_t)El * 4);
        for_each_pair(lm_ptr, e_hidx, [&](int a, int b, int k1, int k2) { pairs.push_back({(long long)a * nf + b, k1, k2}); });
        std::stable_sort(pairs.begin(), pairs.end(), [](const Pair& x, const Pair& y) { return x.key < y.key; });
        npairs = pairs.size();
        for (int a = 0; a < nf; ++a) keys.push_back((long long)a * nf + a);
        for (auto& p : pairs) keys.push_back(p.key);
        for (auto& p : odob) keys.push_back(p.key);
        std::sort(keys.begin(), keys.end());
        keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
        pe1 = host_array(built, npairs, w.pageable[2]); pe2 = host_array(built, npairs, w.pageable[3]);
        blk_pair_ptr.assign(keys.size() + 1, 0);
        size_t ip = 0;
        for (size_t b = 0; b < keys.size(); ++b) {
            blk_pair_ptr[b] = (int)ip;
            while (ip < npairs && pairs[ip].key == keys[b]) { pe1[ip] = pairs[ip].e1; pe2[ip] = pairs[ip].e2; ++ip; }
        }
        blk_pair_ptr[keys.size()] = (int)ip;
    }
    w.pair_e1 = pe1; w.pair_e2 = pe2; w.npairs = npairs;
    const int nblk = w.nblk = (int)keys.size();
    std::vector<int>&blk_a = w.blk_a, &blk_b = w.blk_b;
    blk_a.resize(nblk); blk_b.resize(nblk); w.blk_odo_ptr.assign(nblk + 1, 0); w.blk_odo.resize(odob.size());
    { size_t io = 0;
      for (int b = 0; b < nblk; ++b) {
          blk_a[b] = (int)(keys[b] / nf); blk_b[b] = (int)(keys[b] % nf);
          w.blk_odo_ptr[b] = (int)io;
          while (io < odob.size() && odob[io].key == keys[b]) { w.blk_odo[io] = odob[io].code; ++io; }
      }
      w.blk_odo_ptr[nblk] = (int)io; }
    // envelope of the reduced system: last block row touching each block column, made monotone so that the
    // fill-in of an LDL^T without pivoting stays inside it; in sharded mode every rank needs the envelope of the
    // SUMMED system, i.e. of all landmarks, so it is rebuilt here from the unsharded edge list
    std::vector<int>& bmax = w.bmax;
    bmax.resize(nf);
    for (int a = 0; a < nf; ++a) bmax[a] = a;
    {
        std::vector<int> lo(L, nf), hi(L, -1);
        for (int e = 0; e < E; ++e) { const int a = hidx[edge_pose[e]]; if (a < 0) continue; const int j = edge_point[e]; lo[j] = std::min(lo[j], a); hi[j] = std::max(hi[j], a); }
        for (int j = 0; j < L; ++j) if (hi[j] >= 0) bmax[lo[j]] = std::max(bmax[lo[j]], hi[j]);
        for (int o = 0; o < O; ++o) { const int a = hidx[odo_i[o]], b = hidx[odo_j[o]]; if (a < 0 || b < 0) continue; bmax[std::min(a, b)] = std::max(bmax[std::min(a, b)], std::max(a, b)); }
        for (int a = 1; a < nf; ++a) bmax[a] = std::max(bmax[a], bmax[a - 1]);
    }
    std::vector<int> np(nblk), ne(nblk);
    for (int b = 0; b < nblk; ++b) {
        np[b] = blk_pair_ptr[b + 1] - blk_pair_ptr[b];
        ne[b] = blk_a[b] == blk_b[b] ? pose_ptr[blk_a[b] + 1] - pose_ptr[blk_a[b]] : 0;
    }
    decide(w, nf, bmax.data(), np.data(), ne.data(), nblk, world, pk_grid, sw);
    w.plan_in = bmax;
    w.plan_in.insert(w.plan_in.end(), np.begin(), np.end());
    w.plan_in.insert(w.plan_in.end(), ne.begin(), ne.end());
    return w;
}

// Grows the lists whose length depends on the window's structure; an outgrown list is released. No kernel can still be
// reading one: this runs inside set_problem only, and optimize and debug_system, the calls that launch kernels on these
// lists, synchronise the stream before they return.
int ensure_cap(se2gpu_ba* h, size_t npairs, size_t nblk, size_t nenv) {
    Dev& d = h->d;
    if (npairs > h->cap_pairs) {
        const size_t cap = npairs + npairs / 4 + 1024;
        h->cap_pairs = 0;
        if (h->bufs.regrow(&d.pair_e1, cap) != cudaSuccess || h->bufs.regrow(&d.pair_e2, cap) != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "pair list alloc failed");
        h->cap_pairs = cap;
    }
    if (nblk + 1 > h->cap_blk) {
        const size_t cap = nblk + nblk / 4 + 1024;
        h->cap_blk = 0;
        for (const int** p : {&d.blk_a, &d.blk_b, &d.blk_pair_ptr, &d.blk_odo_ptr, &d.blk_odo, &d.blk_order})
            if (h->bufs.regrow(p, cap + 1) != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "block list alloc failed");
        h->cap_blk = cap;
    }
    if (nenv > h->env_cap) {
        const size_t cap = nenv + nenv / 4 + 64;
        h->env_cap = 0;
        if (h->bufs.regrow(&h->env_idx, cap) != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "envelope list alloc failed");
        h->env_cap = cap;
    }
    return SE2GPU_OK;
}

// one host array -> device: in place when it was built in the page-locked arena, staged through h->arena otherwise
template <class T>
int up(se2gpu_ba* h, const T* dst, const T* src, size_t count) {
    if (!h->arena2.owns(src)) return h->arena.up(const_cast<T*>(dst), src, count, h->stream);
    if (count) SE2_CUDA(cudaMemcpyAsync(const_cast<T*>(dst), src, sizeof(T) * count, cudaMemcpyHostToDevice, h->stream));
    return SE2GPU_OK;
}

// both estimate buffers and the copy se2gpu_ba_reset restores start from the loaded estimates; LM scalars as at creation
int reset_estimates(se2gpu_ba* h, int P, int L) {
    const Dev& d = h->d;
    cudaStream_t s = h->stream;
    SE2_CUDA(cudaMemcpyAsync(d.xp[1], d.xp[0], sizeof(double) * 3 * P, cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(d.xl[1], d.xl[0], sizeof(double) * 3 * L, cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->xp0, d.xp[0], sizeof(double) * 3 * P, cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->xl0, d.xl[0], sizeof(double) * 3 * L, cudaMemcpyDeviceToDevice, s));
    return reset_lm_state(h);
}

// bytes upload_values stages through h->arena: the estimates, and the values that could not be built page-locked
size_t values_stage_bytes(const WindowValues& v, int P, int L) {
    size_t bytes = sizeof(double) * (3 * (size_t)P + 3 * (size_t)L) + 64 * 16;
    for (const auto& f : v.pageable) bytes += sizeof(double) * f.size();
    return bytes;
}

// estimates and values -> device (enqueued; h->arena is reserved by the caller)
int upload_values(se2gpu_ba* h, const WindowValues& v, int P, int L, const double* poses, const double* points) {
    const Dev& d = h->d;
    int rc = up(h, d.xp[0], poses, 3 * (size_t)P);
    if (rc == SE2GPU_OK) rc = up(h, d.xl[0], points, 3 * (size_t)L);
    if (rc == SE2GPU_OK) rc = reset_estimates(h, P, L);
    const struct { const double* dst; const double* src; size_t count; } arrays[] = {
        {d.e_u, v.e_u, (size_t)v.El}, {d.e_v, v.e_v, (size_t)v.El}, {d.e_w00, v.w00, (size_t)v.El}, {d.e_w01, v.w01, (size_t)v.El},
        {d.e_w11, v.w11, (size_t)v.El}, {d.o_m, v.o_m, 3 * (size_t)v.Ol}, {d.o_w, v.o_w, 6 * (size_t)v.Ol}};
    for (const auto& a : arrays) if (rc == SE2GPU_OK) rc = up(h, a.dst, a.src, a.count);
    return rc;
}

// a freshly planned window -> device (enqueued, the caller synchronises once)
int upload_window(se2gpu_ba* h, const WindowPlan& w, const WindowValues& v, int P, int L, const int* odo_i, const int* odo_j,
                  const double* poses, const double* points) {
    const Dev& d = h->d;
    const struct { const int* dst; const int* src; size_t count; } arrays[] = {
        {d.e_pose, w.e_pose, (size_t)w.El}, {d.e_hidx, w.e_hidx, (size_t)w.El}, {d.lm_ptr, w.lm_ptr.data(), w.lm_ptr.size()},
        {d.hidx, w.hidx.data(), w.hidx.size()}, {d.o_i, odo_i, (size_t)w.Ol}, {d.o_j, odo_j, (size_t)w.Ol},
        {d.pose_ptr, w.pose_ptr.data(), w.pose_ptr.size()}, {d.pose_edges, w.pose_edges.data(), w.pose_edges.size()},
        {d.pose_odo_ptr, w.pose_odo_ptr.data(), w.pose_odo_ptr.size()}, {d.pose_odo, w.pose_odo.data(), w.pose_odo.size()},
        {d.blk_a, w.blk_a.data(), w.blk_a.size()}, {d.blk_b, w.blk_b.data(), w.blk_b.size()},
        {d.blk_pair_ptr, w.blk_pair_ptr.data(), w.blk_pair_ptr.size()}, {d.pair_e1, w.pair_e1, w.npairs}, {d.pair_e2, w.pair_e2, w.npairs},
        {d.blk_odo_ptr, w.blk_odo_ptr.data(), w.blk_odo_ptr.size()}, {d.blk_odo, w.blk_odo.data(), w.blk_odo.size()},
        {d.colmax, w.colmax.data(), w.colmax.size()}, {d.tw_cmax1, w.tw_cmax1.data(), w.tw_cmax1.size()},
        {d.blk_order, w.blk_order.data(), w.blk_order.size()}, {h->env_idx, w.env_idx.data(), w.env_idx.size()}};
    size_t bytes = values_stage_bytes(v, P, L) + 64 * 40;
    for (const auto& a : arrays) if (!h->arena2.owns(a.src)) bytes += sizeof(int) * a.count;
    h->arena.reserve(bytes);   // on failure the uploads fall back to pageable copies
    int rc = SE2GPU_OK;
    for (const auto& a : arrays) if (rc == SE2GPU_OK) rc = up(h, a.dst, a.src, a.count);
    if (rc != SE2GPU_OK) return rc;
    const size_t S_elems = h->band.active ? h->band.band_elems : (size_t)w.n * w.n;
    SE2_CUDA(cudaMemsetAsync(h->red, 0, sizeof(double) * (S_elems + w.n + 8), h->stream));
    return upload_values(h, v, P, L, poses, points);
}

// element counts of the arrays se2gpu_ba_debug_structure copies (the rest follow from the loaded sizes in h->d)
void set_struct_len(se2gpu_ba* h, int n_pose_edges, int n_pose_odo, size_t npairs, int n_blk_odo, size_t n_tw, size_t n_order) {
    const Dev& d = h->d;
    long long* s = h->struct_len;
    s[SE2GPU_BA_STRUCT_HIDX] = d.P; s[SE2GPU_BA_STRUCT_LM_PTR] = d.L + 1;
    s[SE2GPU_BA_STRUCT_PERM] = s[SE2GPU_BA_STRUCT_E_POSE] = s[SE2GPU_BA_STRUCT_E_HIDX] = d.E;
    s[SE2GPU_BA_STRUCT_POSE_PTR] = s[SE2GPU_BA_STRUCT_POSE_ODO_PTR] = d.nf + 1;
    s[SE2GPU_BA_STRUCT_POSE_EDGES] = n_pose_edges; s[SE2GPU_BA_STRUCT_POSE_ODO] = n_pose_odo;
    s[SE2GPU_BA_STRUCT_BLK_A] = s[SE2GPU_BA_STRUCT_BLK_B] = d.nblk;
    s[SE2GPU_BA_STRUCT_BLK_PAIR_PTR] = s[SE2GPU_BA_STRUCT_BLK_ODO_PTR] = d.nblk + 1;
    s[SE2GPU_BA_STRUCT_PAIR_E1] = s[SE2GPU_BA_STRUCT_PAIR_E2] = (long long)npairs;
    s[SE2GPU_BA_STRUCT_BLK_ODO] = n_blk_odo; s[SE2GPU_BA_STRUCT_COLMAX] = d.n;
    s[SE2GPU_BA_STRUCT_TW_CMAX1] = (long long)n_tw; s[SE2GPU_BA_STRUCT_BLK_ORDER] = (long long)n_order;
    s[SE2GPU_BA_STRUCT_ENV_IDX] = h->nenv; s[SE2GPU_BA_STRUCT_ODO_I] = s[SE2GPU_BA_STRUCT_ODO_J] = d.O;
    for (int k = SE2GPU_BA_STRUCT_E_U; k <= SE2GPU_BA_STRUCT_E_W11; ++k) s[k] = 2LL * d.E;
    s[SE2GPU_BA_STRUCT_ODO_M] = 6LL * d.O; s[SE2GPU_BA_STRUCT_ODO_W] = 12LL * d.O;
}

void set_camera(se2gpu_ba* h, double fx, double cx, double cy, const double* Tcb, double huber_delta) {
    h->cam.fx = fx; h->cam.cx = cx; h->cam.cy = cy; h->cam.delta = huber_delta;
    memcpy(h->cam.Rcb, Tcb, sizeof(double) * 9); memcpy(h->cam.tcb, Tcb + 9, sizeof(double) * 3);
}

}  // namespace

extern "C" {

int se2gpu_ba_build_information(int P, int L, int E, const float* view_mp, const int* edge_pose, const int* edge_point,
                                const int* octave, const float* kf_Rcw, const float* kf_twb_xy, const float* mp_pos,
                                const float* level_sigma2, int nlevels, float fx, float xrot_info, float z_info, double* info,
                                int device) {
    if (P <= 0 || L < 0 || E < 0 || nlevels <= 0) return fail(SE2GPU_ERR_INVALID, "bad sizes");
    if (E == 0) return SE2GPU_OK;
    if (!view_mp || !edge_pose || !edge_point || !octave || !kf_Rcw || !kf_twb_xy || !mp_pos || !level_sigma2 || !info)
        return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int e = 0; e < E; ++e)
        if (edge_pose[e] < 0 || edge_pose[e] >= P || edge_point[e] < 0 || edge_point[e] >= L) return fail(SE2GPU_ERR_INVALID, "edge %d references a missing vertex", e);
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    InfoArgs a{};
    a.P = P; a.L = L; a.E = E; a.nlevels = nlevels; a.fx = fx;
    a.sigma_rotxy = 1.f / xrot_info;       // float Sigma_rotxy = 1./Config::PLANEMOTION_XROT_INFO   (Map.cpp:1043)
    a.sigma_z = 1.f / z_info;              // float Sigma_z = 1./Config::PLANEMOTION_Z_INFO          (Map.cpp:1044)
    a.info = st.output(info, 3 * (size_t)E);
    a.lc = st.upload(view_mp, 3 * (size_t)E); a.edge_pose = st.upload(edge_pose, E); a.edge_point = st.upload(edge_point, E);
    a.octave = st.upload(octave, E); a.Rcw = st.upload(kf_Rcw, 9 * (size_t)P); a.twb = st.upload(kf_twb_xy, 2 * (size_t)P);
    a.lw = st.upload(mp_pos, 3 * (size_t)L); a.level_sigma2 = st.upload(level_sigma2, nlevels);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_edge_information, (E + 255) / 256, 256, 0, 0, a);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

}  // extern "C"

namespace {

// no window loaded: optimize / get / reset / debug_* refuse to run, and the next set_problem rebuilds the structure
void unload(se2gpu_ba* h) {
    h->loaded = false;
    h->t_edge_pose.clear(); h->t_edge_point.clear(); h->t_odo_i.clear(); h->t_odo_j.clear(); h->t_fixed.clear();
    h->t_rank = h->t_world = -1;
    h->dl.valid = false;
}

int load_window(se2gpu_ba* h, int P, int L, int E, int O, const double* poses, const uint8_t* fixed, const double* points,
                const int* edge_pose, const int* edge_point, const double* uv, const double* info, const int* odo_i,
                const int* odo_j, const double* odo_meas, const double* odo_info, double fx, double cx, double cy,
                const double* Tcb, double huber_delta) {
    if (P <= 0 || L < 0 || E < 0 || O < 0) return fail(SE2GPU_ERR_INVALID, "bad sizes");
    SE2_NVTX("se2gpu.ba.set_problem");
    if (P > h->maxP || L > h->maxL || E > h->maxE || O > h->maxO) return fail(SE2GPU_ERR_CAPACITY, "problem (%d,%d,%d,%d) exceeds capacity (%d,%d,%d,%d)", P, L, E, O, h->maxP, h->maxL, h->maxE, h->maxO);
    SE2_CUDA(cudaSetDevice(h->device));
    const auto tnow = [] { return std::chrono::steady_clock::now(); };
    const auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t_begin = tnow();
    for (int e = 0; e < E; ++e)
        if (edge_pose[e] < 0 || edge_pose[e] >= P || edge_point[e] < 0 || edge_point[e] >= L) return fail(SE2GPU_ERR_INVALID, "edge %d references a missing vertex", e);
    for (int o = 0; o < O; ++o)
        if (odo_i[o] < 0 || odo_i[o] >= P || odo_j[o] < 0 || odo_j[o] >= P) return fail(SE2GPU_ERR_INVALID, "odometry edge %d references a missing vertex", o);
    Dev& d = h->d;

    if (same_topology(h, P, L, E, O, fixed, edge_pose, edge_point, odo_i, odo_j)) {   // only the values are refreshed
        h->arena2.reserve(values_bytes(d.E, d.O));
        const WindowValues v = gather_values(h, h->perm, d.E, d.O, uv, info, odo_meas, odo_info);
        h->arena.reserve(values_stage_bytes(v, P, L));   // on failure the uploads fall back to pageable copies
        if (const int rc = upload_values(h, v, P, L, poses, points)) return rc;
        SE2_CUDA(cudaStreamSynchronize(h->stream));
        set_camera(h, fx, cx, cy, Tcb, huber_delta);
        if (h->sw.debug) fprintf(stderr, "[se2gpu_ba_set_problem] same topology: values refreshed in %.3f ms\n", ms(t_begin, tnow()));
        return SE2GPU_OK;
    }
    h->loaded = false;
    h->dl.valid = false;   // the device-side topology record is the other entry's

    const WindowPlan w = plan_window(h->arena2, P, L, E, O, fixed, edge_pose, edge_point, odo_i, odo_j, h->rank, h->world, h->pk_grid, h->sw);
    if (w.blk_odo.size() + 1 > (size_t)2 * (h->maxO ? h->maxO : 1) + 1) return fail(SE2GPU_ERR_CAPACITY, "too many odometry blocks");
    const WindowValues v = gather_values(h, w.perm, w.El, w.Ol, uv, info, odo_meas, odo_info);
    h->nenv = (int)w.env_idx.size();
    if (h->ssum) SE2_CUDA(cudaMemsetAsync(h->ssum, 0, sizeof(double) * ((size_t)SMEM_CHOL_MAX_N * SMEM_CHOL_MAX_N + SMEM_CHOL_MAX_N + 8), h->stream));   // zero outside the (new) envelope
    // windows beyond one CTA's shared memory: partitioned band factorisation when the envelope is narrow (ba_band.cu),
    // otherwise the single-CTA global-memory envelope factorisation
    se2band::release(h->band);
    if (w.n > SMEM_CHOL_MAX_N && !h->sw.no_band) se2band::plan(h->band, w.nf, w.bmax, h->smem_optin);
    const bool band = h->band.active;
    int* pl = h->plan;
    pl[0] = w.nf; pl[1] = w.n; pl[2] = w.sorted_structure ? 1 : 0;
    pl[3] = 0; for (int a = 0; a < w.nf; ++a) pl[3] = std::max(pl[3], w.bmax[a] - a);
    pl[4] = w.n <= SMEM_CHOL_MAX_N ? (w.tw_m0 > 0 ? 1 : 0) : (band ? 2 : 3);
    pl[5] = w.tw_m0; pl[6] = w.tw_w; pl[7] = band ? h->band.w : 0; pl[8] = band ? h->band.p : 0;
    pl[9] = h->pk_grid; pl[10] = w.workers; pl[11] = w.nblk; pl[12] = w.maxlen; pl[13] = w.uncached;
    int rc = ensure_cap(h, w.npairs, std::max<size_t>(std::max<size_t>(w.nblk, w.blk_order.size()), w.blk_odo.size()), w.env_idx.size());
    if (rc != SE2GPU_OK) return rc;
    const auto t_host = tnow();
    if ((rc = upload_window(h, w, v, P, L, odo_i, odo_j, poses, points)) != SE2GPU_OK) return rc;
    const auto t_enq = tnow();
    SE2_CUDA(cudaStreamSynchronize(h->stream));
    if (h->sw.debug)
        fprintf(stderr, "[se2gpu_ba_set_problem] host structure %.3f ms, stage+enqueue %.3f ms, drain %.3f ms (P %d L %d E %d blocks %d pairs %zu)\n",
                ms(t_begin, t_host), ms(t_host, t_enq), ms(t_enq, tnow()), P, L, E, w.nblk, w.npairs);

    const size_t S_elems = band ? h->band.band_elems : (size_t)w.n * w.n;
    d.P = P; d.L = L; d.E = w.El; d.O = w.Ol; d.nf = w.nf; d.n = w.n; d.nblk = w.nblk; d.rank = h->rank; d.world = h->world;
    d.nord = (int)w.blk_order.size(); d.tw_m0 = w.tw_m0; d.tw_w = w.tw_w;
    d.S = h->red; d.bs = h->red + S_elems; d.scal = d.bs + w.n; d.sbw = band ? h->band.bw : 0;
    d.nb_lm = (L + LM_THREADS - 1) / LM_THREADS; d.nb_odo = (w.Ol + LM_THREADS - 1) / LM_THREADS;
    h->nb_scale = (std::max(L, P) + LM_THREADS - 1) / LM_THREADS;
    set_camera(h, fx, cx, cy, Tcb, huber_delta);
    h->perm = w.perm; h->P = P; h->L = L; h->E = E; h->O = O;
    h->t_edge_pose.assign(edge_pose, edge_pose + E); h->t_edge_point.assign(edge_point, edge_point + E); h->t_odo_i.assign(odo_i, odo_i + O);
    h->t_odo_j.assign(odo_j, odo_j + O); h->t_fixed.assign(fixed, fixed + P); h->t_rank = h->rank; h->t_world = h->world;
    set_struct_len(h, (int)w.pose_edges.size(), (int)w.pose_odo.size(), w.npairs, (int)w.blk_odo.size(), w.tw_cmax1.size(), w.blk_order.size());
    h->plan_in = w.plan_in; h->plan_grid = h->pk_grid;
    h->loaded = true;
    return SE2GPU_OK;
}

}  // namespace

extern "C" {

int se2gpu_ba_set_problem(se2gpu_ba* h, int P, int L, int E, int O, const double* poses, const uint8_t* fixed,
                          const double* points, const int* edge_pose, const int* edge_point, const double* uv,
                          const double* info, const int* odo_i, const int* odo_j, const double* odo_meas,
                          const double* odo_info, double fx, double cx, double cy, const double* Tcb, double huber_delta) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    const int rc = load_window(h, P, L, E, O, poses, fixed, points, edge_pose, edge_point, uv, info, odo_i, odo_j, odo_meas,
                               odo_info, fx, cx, cy, Tcb, huber_delta);
    if (rc != SE2GPU_OK) unload(h);   // a rejected window leaves none loaded, never the previous one
    return rc;
}

}  // extern "C"

// ================================================================================================ se2gpu_ba_set_problem_device
//
// The same window as se2gpu_ba_set_problem, from device buffers, with the structure built on the device. Every array it
// leaves equals the host build's element for element, so the two loads optimise byte-identically. Two phases, each ending
// in one small readback:
//   count    range checks, free-pose index, landmark sort (perm, lm_ptr, e_pose, e_hidx), pose lists, pairs per edge, the
//            nf x nf bitmap of the blocks of S -> scalars (nf, El, pairs, blocks, ...)
//   fill     block lists from the bitmap, pairs in for_each_pair order keyed by block, stably sorted; odometry blocks;
//            envelope -> bmax, pairs per block, pose edges per diagonal block
// The host then takes decide()'s decisions and uploads their O(nf + nblk) results; no per-edge or per-pair array crosses
// PCIe. Orders are made stable by an LSD radix sort (8-bit digits, block-local stable ranks) over (key, index) pairs.
namespace {

constexpr int DL_THREADS = 256;
constexpr int SCAN_TILE = 1024;   // elements per CTA of the tile scan (256 threads x 4)
// device scalars of the build (DevLoad::sc)
enum { DL_ERR, DL_NF, DL_NPE, DL_NPO, DL_NODOB, DL_DIFF, DL_EL, DL_NPAIRS, DL_NBLK, DL_SCALARS = 16 };

inline int nblocks(long long n, int per) { return (int)std::max<long long>(1, (n + per - 1) / per); }

__device__ __forceinline__ bool in_range(int v, int n) { return v >= 0 && v < n; }

// exclusive scan of one CTA of 256 threads with `v` per thread; returns the exclusive prefix, *total gets the sum
__device__ int cta_excl_scan(int v, int* total) {
    __shared__ int warp_sum[DL_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int w = lane < DL_THREADS / 32 ? warp_sum[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
        if (lane < DL_THREADS / 32) warp_sum[lane] = w;
    }
    __syncthreads();
    const int excl = x - v + (wid > 0 ? warp_sum[wid - 1] : 0);
    *total = warp_sum[DL_THREADS / 32 - 1];
    __syncthreads();
    return excl;
}

// in-place exclusive scan, step 1: each CTA scans SCAN_TILE elements and leaves their sum in aux[blockIdx.x]
__global__ void __launch_bounds__(DL_THREADS) k_scan_tiles(int* a, int n, int* aux) {
    const long long base = (long long)blockIdx.x * SCAN_TILE + 4 * threadIdx.x;
    int v[4], s = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) { v[q] = base + q < n ? a[base + q] : 0; s += v[q]; }
    int total;
    int run = cta_excl_scan(s, &total);
#pragma unroll
    for (int q = 0; q < 4; ++q) { if (base + q < n) a[base + q] = run; run += v[q]; }
    if (threadIdx.x == 0) aux[blockIdx.x] = total;
}

// step 2 (one CTA): exclusive scan of the tile sums; the grand total goes to a[n]
__global__ void __launch_bounds__(DL_THREADS) k_scan_aux(int* aux, int m, int* a, int n) {
    int carry = 0;
    for (int base = 0; base < m; base += DL_THREADS) {
        const int i = base + threadIdx.x;
        const int v = i < m ? aux[i] : 0;
        int total;
        const int e = cta_excl_scan(v, &total);
        if (i < m) aux[i] = carry + e;
        carry += total;
    }
    if (threadIdx.x == 0) a[n] = carry;
}

// step 3: add each tile's offset
__global__ void __launch_bounds__(DL_THREADS) k_scan_add(int* a, int n, const int* aux) {
    const long long base = (long long)blockIdx.x * SCAN_TILE + 4 * threadIdx.x;
    const int off = aux[blockIdx.x];
#pragma unroll
    for (int q = 0; q < 4; ++q) if (base + q < n) a[base + q] += off;
}

// radix sort pass, step 1: digit histogram of each tile of DL_THREADS elements, digit-major: hist[d * ntiles + tile]
__global__ void __launch_bounds__(DL_THREADS) k_radix_hist(const int* key, int n, int shift, int* hist, int ntiles) {
    __shared__ int cnt[256];
    cnt[threadIdx.x] = 0;
    __syncthreads();
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&cnt[(key[i] >> shift) & 255], 1);
    __syncthreads();
    hist[(size_t)threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

// step 2 (after the scan of hist): stable scatter; the rank inside the tile counts the earlier elements with the same digit
// in this warp (match_any) and in the warps before it
__global__ void __launch_bounds__(DL_THREADS) k_radix_scatter(const int* key, const int* val, int n, int shift, const int* hist,
                                                              int ntiles, int* key_out, int* val_out) {
    __shared__ int wcnt[DL_THREADS / 32][256];
    for (int k = threadIdx.x; k < (DL_THREADS / 32) * 256; k += DL_THREADS) (&wcnt[0][0])[k] = 0;
    __syncthreads();
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int k = i < n ? key[i] : 0;
    const int d = i < n ? (k >> shift) & 255 : 256;
    const unsigned same = __match_any_sync(0xffffffffu, d);
    const int before = __popc(same & ((1u << lane) - 1));
    if (d < 256 && before == 0) wcnt[wid][d] = __popc(same);
    __syncthreads();
    if (d < 256) {
        int pos = hist[(size_t)d * ntiles + blockIdx.x] + before;
        for (int w = 0; w < wid; ++w) pos += wcnt[w][d];
        key_out[pos] = k;
        val_out[pos] = val[i];
    }
}

// --- count phase -------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(DL_THREADS) k_check(int P, int L, int E, int O, const int* edge_pose, const int* edge_point,
                                                      const int* odo_i, const int* odo_j, int* sc) {
    const int t = blockIdx.x * DL_THREADS + threadIdx.x;
    bool bad = false;
    if (t < E) bad = !in_range(edge_pose[t], P) || !in_range(edge_point[t], L);
    else if (t < E + O) bad = !in_range(odo_i[t - E], P) || !in_range(odo_j[t - E], P);
    if (bad) atomicOr(&sc[DL_ERR], 1);
}

// SparseOptimizer::buildIndexMapping: free poses in id order (one CTA)
__global__ void __launch_bounds__(DL_THREADS) k_hidx(int P, const uint8_t* fixed, int* hidx, int* sc) {
    int carry = 0;
    for (int base = 0; base < P; base += DL_THREADS) {
        const int i = base + threadIdx.x;
        const int f = i < P && !fixed[i];
        int total;
        const int e = cta_excl_scan(f, &total);
        if (i < P) hidx[i] = f ? carry + e : -1;
        carry += total;
    }
    if (threadIdx.x == 0) sc[DL_NF] = carry;
}

// landmark sort keys (this rank's landmarks; others and bad edges sort last as L), landmark counts, and the envelope's
// per-landmark first / last free pose over ALL landmarks (the summed system's envelope in sharded mode)
__global__ void __launch_bounds__(DL_THREADS) k_lm_keys(int P, int L, int E, int rank, int world, const int* edge_pose,
                                                        const int* edge_point, const int* hidx, int* key, int* val, int* lm_cnt,
                                                        int* lo, int* hi) {
    const int e = blockIdx.x * DL_THREADS + threadIdx.x;
    if (e >= E) return;
    const int p = edge_pose[e], j = edge_point[e];
    int k = L;
    if (in_range(p, P) && in_range(j, L)) {
        if (j % world == rank) { k = j; atomicAdd(&lm_cnt[j], 1); }
        const int a = hidx[p];
        if (a >= 0) { atomicMin(&lo[j], a); atomicMax(&hi[j], a); }
    }
    key[e] = k; val[e] = e;
}

__global__ void __launch_bounds__(DL_THREADS) k_fill(int* a, int n, int v) {
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    if (i < n) a[i] = v;
}

// landmark-sorted edges: e_pose, e_hidx, and the pose-list keys (edges of fixed poses sort last as P)
__global__ void __launch_bounds__(DL_THREADS) k_sorted_edges(int P, int E, const int* lm_ptr_end, const int* perm, const int* edge_pose,
                                                             const int* hidx, int* e_pose, int* e_hidx, int* key, int* val,
                                                             int* pose_cnt, int* sc) {
    const int k = blockIdx.x * DL_THREADS + threadIdx.x;
    if (k >= E) return;
    int pk = P;
    if (k < *lm_ptr_end) {
        const int p = edge_pose[perm[k]], a = hidx[p];
        e_pose[k] = p; e_hidx[k] = a;
        if (a >= 0) { pk = a; atomicAdd(&pose_cnt[a], 1); atomicAdd(&sc[DL_NPE], 1); }
    }
    key[k] = pk; val[k] = k;
}

// odometry pose lists: code 2o + role, keyed by the free pose of that role (rank 0 only; the others sort last as P)
__global__ void __launch_bounds__(DL_THREADS) k_odo_keys(int P, int Ol, int O, const int* odo_i, const int* odo_j, const int* hidx,
                                                         int* key, int* val, int* cnt, int* sc) {
    const int c = blockIdx.x * DL_THREADS + threadIdx.x;
    if (c >= 2 * O) return;
    int k = P;
    if ((c >> 1) < Ol) {
        const int v = (c & 1) ? odo_j[c >> 1] : odo_i[c >> 1];
        const int a = in_range(v, P) ? hidx[v] : -1;
        if (a >= 0) { k = a; atomicAdd(&cnt[a], 1); atomicAdd(&sc[DL_NPO], 1); }
    }
    key[c] = k; val[c] = c;
}

__device__ __forceinline__ void mark(unsigned* bits, long long key) {
    const unsigned b = 1u << (key & 31);
    if (!(bits[key >> 5] & b)) atomicOr(&bits[key >> 5], b);
}

// pairs (k1, k2) of each sorted edge k1 in for_each_pair's order, counted, and their blocks marked in the bitmap; also the
// diagonal blocks and the odometry blocks (rank 0), whose count goes to sc[DL_NODOB]
__global__ void __launch_bounds__(DL_THREADS) k_pair_count(int P, int E, int Ol, const int* lm_ptr, const int* El_ptr, const int* perm,
                                                           const int* edge_point, const int* e_hidx, const int* odo_i, const int* odo_j,
                                                           const int* hidx, int* sc, unsigned* bits, int* pair_cnt) {
    const int t = blockIdx.x * DL_THREADS + threadIdx.x;
    const int nf = sc[DL_NF];
    if (t < E) {
        int c = 0;
        if (t < *El_ptr) {
            const int a = e_hidx[t];
            if (a >= 0) {
                const int j = edge_point[perm[t]], k_end = lm_ptr[j + 1];
                for (int k2 = lm_ptr[j]; k2 < k_end; ++k2) {
                    const int b = e_hidx[k2];
                    if (b >= 0 && b <= a) { ++c; mark(bits, (long long)a * nf + b); }
                }
            }
        }
        pair_cnt[t] = c;
    }
    if (t < nf) mark(bits, (long long)t * nf + t);
    if (t < Ol) {
        const int i = odo_i[t], j = odo_j[t];
        const int a = in_range(i, P) ? hidx[i] : -1, b = in_range(j, P) ? hidx[j] : -1;
        if (a >= 0 && b >= 0 && a != b) { mark(bits, (long long)max(a, b) * nf + min(a, b)); atomicAdd(&sc[DL_NODOB], 1); }
    }
}

__global__ void __launch_bounds__(DL_THREADS) k_popc(const unsigned* bits, int nw, int* cnt) {
    const int w = blockIdx.x * DL_THREADS + threadIdx.x;
    if (w < nw) cnt[w] = __popc(bits[w]);
}

// --- fill phase --------------------------------------------------------------------------------------------------------

// index of block `key` among the blocks of S in key order
__device__ __forceinline__ int block_of(const unsigned* bits, const int* wprefix, long long key) {
    return wprefix[key >> 5] + __popc(bits[key >> 5] & ((1u << (key & 31)) - 1u));
}

__global__ void __launch_bounds__(DL_THREADS) k_blocks(const unsigned* bits, const int* wprefix, int nw, const int* sc, int* blk_a, int* blk_b) {
    const int w = blockIdx.x * DL_THREADS + threadIdx.x;
    if (w >= nw) return;
    const int nf = sc[DL_NF];
    unsigned m = bits[w];
    int idx = wprefix[w];
    while (m) {
        const int bit = __ffs(m) - 1;
        m &= m - 1;
        const long long key = 32LL * w + bit;
        blk_a[idx] = (int)(key / nf); blk_b[idx] = (int)(key % nf);
        ++idx;
    }
}

// pairs in for_each_pair order (landmark, k1, k2) from pair_off[k1] on, keyed by their block
__global__ void __launch_bounds__(DL_THREADS) k_pair_fill(int El, const int* lm_ptr, const int* perm, const int* edge_point, const int* e_hidx,
                                                          const int* sc, const unsigned* bits, const int* wprefix, const int* pair_off,
                                                          int* key, int* val, int* g1, int* g2, int* blk_cnt) {
    const int k1 = blockIdx.x * DL_THREADS + threadIdx.x;
    if (k1 >= El) return;
    const int a = e_hidx[k1];
    if (a < 0) return;
    const int nf = sc[DL_NF];
    const int j = edge_point[perm[k1]], k_end = lm_ptr[j + 1];
    int at = pair_off[k1];
    for (int k2 = lm_ptr[j]; k2 < k_end; ++k2) {
        const int b = e_hidx[k2];
        if (b < 0 || b > a) continue;
        const int blk = block_of(bits, wprefix, (long long)a * nf + b);
        key[at] = blk; val[at] = at; g1[at] = k1; g2[at] = k2;
        atomicAdd(&blk_cnt[blk], 1);
        ++at;
    }
}

__global__ void __launch_bounds__(DL_THREADS) k_pair_gather(int npairs, const int* order, const int* g1, const int* g2, int* pair_e1, int* pair_e2) {
    const int q = blockIdx.x * DL_THREADS + threadIdx.x;
    if (q >= npairs) return;
    const int p = order[q];
    pair_e1[q] = g1[p]; pair_e2[q] = g2[p];
}

// odometry blocks: code 2o (a > b) or 2o + 1, keyed by the block (max, min); the others sort last as nblk
__global__ void __launch_bounds__(DL_THREADS) k_odo_blocks(int Ol, int nblk, const int* odo_i, const int* odo_j, const int* hidx, const int* sc,
                                                           const unsigned* bits, const int* wprefix, int* key, int* val, int* blk_cnt) {
    const int o = blockIdx.x * DL_THREADS + threadIdx.x;
    if (o >= Ol) return;
    const int nf = sc[DL_NF];
    const int a = hidx[odo_i[o]], b = hidx[odo_j[o]];
    int k = nblk, code = 0;
    if (a >= 0 && b >= 0 && a != b) {
        k = block_of(bits, wprefix, (long long)max(a, b) * nf + min(a, b));
        code = a > b ? 2 * o : 2 * o + 1;
        atomicAdd(&blk_cnt[k], 1);
    }
    key[o] = k; val[o] = code;
}

// envelope: bmax[a] = last block row coupled to block column a (landmarks, then every odometry edge), before the prefix max
__global__ void __launch_bounds__(DL_THREADS) k_env(int P, int L, int O, const int* lo, const int* hi, const int* odo_i, const int* odo_j,
                                                    const int* hidx, int* bmax) {
    const int t = blockIdx.x * DL_THREADS + threadIdx.x;
    if (t < L && hi[t] >= 0) atomicMax(&bmax[lo[t]], hi[t]);
    if (t < O) {
        const int i = odo_i[t], j = odo_j[t];
        const int a = in_range(i, P) ? hidx[i] : -1, b = in_range(j, P) ? hidx[j] : -1;
        if (a >= 0 && b >= 0) atomicMax(&bmax[min(a, b)], max(a, b));
    }
}

__global__ void __launch_bounds__(DL_THREADS) k_iota(int* a, int n) {
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    if (i < n) a[i] = i;
}

// prefix max of bmax (one CTA), then the per-block work the host's decisions read: pairs, and pose edges of a diagonal block
__global__ void __launch_bounds__(DL_THREADS) k_env_scan_weights(int nf, int nblk, int* bmax, const int* blk_a, const int* blk_b,
                                                                 const int* blk_pair_ptr, const int* pose_ptr, int* np, int* ne) {
    __shared__ int wmax[DL_THREADS / 32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = -1;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int base = 0; base < nf; base += DL_THREADS) {
        const int i = base + threadIdx.x;
        int x = i < nf ? bmax[i] : -1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x = max(x, y); }
        if (lane == 31) wmax[threadIdx.x >> 5] = x;
        __syncthreads();
        int pre = carry;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pre = max(pre, wmax[w]);
        x = max(x, pre);
        if (i < nf) bmax[i] = x;
        __syncthreads();
        if (threadIdx.x == DL_THREADS - 1) carry = x;
        __syncthreads();
    }
    for (int b = threadIdx.x; b < nblk; b += DL_THREADS) {
        np[b] = blk_pair_ptr[b + 1] - blk_pair_ptr[b];
        const int a = blk_a[b];
        ne[b] = a == blk_b[b] ? pose_ptr[a + 1] - pose_ptr[a] : 0;
    }
}

// --- values ------------------------------------------------------------------------------------------------------------

// measurements and information in landmark-sorted edge order, odometry as SoA (gather_values on the device)
__global__ void __launch_bounds__(DL_THREADS) k_values(int El, int Ol, const int* perm, const double* uv, const double* info,
                                                       const double* odo_meas, const double* odo_info, double* e_u, double* e_v,
                                                       double* w00, double* w01, double* w11, double* o_m, double* o_w) {
    const int t = blockIdx.x * DL_THREADS + threadIdx.x;
    if (t < El) {
        const size_t e = perm[t];
        e_u[t] = uv[2 * e]; e_v[t] = uv[2 * e + 1];
        w00[t] = info[3 * e]; w01[t] = info[3 * e + 1]; w11[t] = info[3 * e + 2];
    }
    if (t < Ol) {
        for (int q = 0; q < 3; ++q) o_m[q * (size_t)Ol + t] = odo_meas[3 * (size_t)t + q];
        for (int q = 0; q < 6; ++q) o_w[q * (size_t)Ol + t] = odo_info[6 * (size_t)t + q];
    }
}

// same graph structure as the loaded window? (against the device copies of the loaded topology)
__global__ void __launch_bounds__(DL_THREADS) k_same_topology(int P, int E, int O, const uint8_t* fixed, const int* edge_pose, const int* edge_point,
                                                              const int* odo_i, const int* odo_j, const uint8_t* t_fixed, const int* t_edge_pose,
                                                              const int* t_edge_point, const int* t_odo_i, const int* t_odo_j, int* sc) {
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    bool diff = false;
    if (i < P) diff = fixed[i] != t_fixed[i];
    if (i < E) diff = diff || edge_pose[i] != t_edge_pose[i] || edge_point[i] != t_edge_point[i];
    if (i < O) diff = diff || odo_i[i] != t_odo_i[i] || odo_j[i] != t_odo_j[i];
    if (diff) atomicOr(&sc[DL_DIFF], 1);
}

// --- host side ---------------------------------------------------------------------------------------------------------

// scratch buffers of at least n elements each that share one capacity (contents not kept when they grow)
template <class T>
int grow(se2gpu_ba* h, std::initializer_list<T**> ps, size_t* cap, size_t n) {
    bool have = true;
    for (T** p : ps) have = have && *p;
    if (have && n <= *cap) return SE2GPU_OK;
    const size_t c = n + n / 4 + 1024;
    *cap = 0;
    for (T** p : ps) if (h->bufs.regrow(p, c) != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "device load scratch alloc failed");
    *cap = c;
    return SE2GPU_OK;
}

// exclusive scan of a[0..n) in place, a[n] = total
int scan(se2gpu_ba* h, int* a, int n) {
    DevLoad& g = h->dl;
    const int tiles = nblocks(n, SCAN_TILE);
    if (const int rc = grow(h, {&g.aux}, &g.cap_aux, tiles)) return rc;
    cudaStream_t s = h->stream;
    SE2_LAUNCH(k_scan_tiles, tiles, DL_THREADS, 0, s, a, n, g.aux);
    SE2_LAUNCH(k_scan_aux, 1, DL_THREADS, 0, s, g.aux, tiles, a, n);
    SE2_LAUNCH(k_scan_add, tiles, DL_THREADS, 0, s, a, n, g.aux);
    return SE2GPU_OK;
}

// stable sort of (k0, v0)[0..n) by key in [0, max_key]; *out receives the buffer that then holds the sorted values
int radix_sort(se2gpu_ba* h, int n, int max_key, const int** out) {
    DevLoad& g = h->dl;
    int *k0 = g.k0, *v0 = g.v0, *k1 = g.k1, *v1 = g.v1;
    const int tiles = nblocks(n, DL_THREADS);
    if (const int rc = grow(h, {&g.hist}, &g.cap_hist, (size_t)256 * tiles + 1)) return rc;
    int bits = 0;
    while (bits < 31 && (max_key >> bits) != 0) ++bits;
    for (int shift = 0; shift < bits && n > 0; shift += 8) {
        SE2_LAUNCH(k_radix_hist, tiles, DL_THREADS, 0, h->stream, k0, n, shift, g.hist, tiles);
        if (const int rc = scan(h, g.hist, 256 * tiles)) return rc;
        SE2_LAUNCH(k_radix_scatter, tiles, DL_THREADS, 0, h->stream, k0, v0, n, shift, g.hist, tiles, k1, v1);
        std::swap(k0, k1); std::swap(v0, v1);
    }
    *out = v0;
    return SE2GPU_OK;
}

// the four ping-pong buffers of radix_sort, n elements each
int grow_sort(se2gpu_ba* h, size_t n) {
    DevLoad& g = h->dl;
    return grow(h, {&g.k0, &g.v0, &g.k1, &g.v1}, &g.cap_sort, n);
}

// the device record of the loaded topology, and the build's fixed-size buffers
int dl_alloc(se2gpu_ba* h) {
    DevLoad& g = h->dl;
    if (g.sc_host) return SE2GPU_OK;
    const size_t P = h->maxP, E = h->maxE, O = h->maxO ? h->maxO : 1;
    if (h->bufs.alloc(&g.fixed, P) != cudaSuccess || h->bufs.alloc(&g.edge_pose, E) != cudaSuccess || h->bufs.alloc(&g.edge_point, E) != cudaSuccess ||
        h->bufs.alloc(&g.odo_i, O) != cudaSuccess || h->bufs.alloc(&g.odo_j, O) != cudaSuccess || h->bufs.alloc(&g.perm, E) != cudaSuccess ||
        h->bufs.alloc(&g.sc, DL_SCALARS) != cudaSuccess)
        return fail(SE2GPU_ERR_CUDA, "device load alloc failed");
    if (cudaMallocHost((void**)&g.sc_host, sizeof(int) * DL_SCALARS) != cudaSuccess) { g.sc_host = nullptr; return fail(SE2GPU_ERR_CUDA, "cudaMallocHost failed"); }
    return SE2GPU_OK;
}

// estimates -> both buffers and the reset copy, LM scalars, and the values in landmark-sorted order (enqueued)
int device_values(se2gpu_ba* h, int P, int L, const double* poses, const double* points, const double* uv, const double* info,
                  const double* odo_meas, const double* odo_info) {
    const Dev& d = h->d;
    cudaStream_t s = h->stream;
    SE2_CUDA(cudaMemcpyAsync(d.xp[0], poses, sizeof(double) * 3 * P, cudaMemcpyDeviceToDevice, s));
    if (L) SE2_CUDA(cudaMemcpyAsync(d.xl[0], points, sizeof(double) * 3 * L, cudaMemcpyDeviceToDevice, s));
    if (const int rc = reset_estimates(h, P, L)) return rc;
    const int n = std::max(d.E, d.O);
    if (n > 0)
        SE2_LAUNCH(k_values, nblocks(n, DL_THREADS), DL_THREADS, 0, s, d.E, d.O, h->dl.perm, uv, info, odo_meas, odo_info,
                   const_cast<double*>(d.e_u), const_cast<double*>(d.e_v), const_cast<double*>(d.e_w00), const_cast<double*>(d.e_w01),
                   const_cast<double*>(d.e_w11), const_cast<double*>(d.o_m), const_cast<double*>(d.o_w));
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

// the build's scalars -> host (one copy, then the stream is drained)
int read_scalars(se2gpu_ba* h) {
    SE2_CUDA(cudaMemcpyAsync(h->dl.sc_host, h->dl.sc, sizeof(int) * DL_SCALARS, cudaMemcpyDeviceToHost, h->stream));
    SE2_CUDA(cudaStreamSynchronize(h->stream));
    return SE2GPU_OK;
}

int load_window_device(se2gpu_ba* h, int P, int L, int E, int O, const double* poses, const uint8_t* fixed, const double* points,
                       const int* edge_pose, const int* edge_point, const double* uv, const double* info, const int* odo_i,
                       const int* odo_j, const double* odo_meas, const double* odo_info, double fx, double cx, double cy,
                       const double* Tcb, double huber_delta) {
    if (P <= 0 || L < 0 || E < 0 || O < 0) return fail(SE2GPU_ERR_INVALID, "bad sizes");
    SE2_NVTX("se2gpu.ba.set_problem_device");
    if (P > h->maxP || L > h->maxL || E > h->maxE || O > h->maxO) return fail(SE2GPU_ERR_CAPACITY, "problem (%d,%d,%d,%d) exceeds capacity (%d,%d,%d,%d)", P, L, E, O, h->maxP, h->maxL, h->maxE, h->maxO);
    if (!poses || !fixed || !Tcb || (L && !points) || (E && (!edge_pose || !edge_point || !uv || !info)) ||
        (O && (!odo_i || !odo_j || !odo_meas || !odo_info)))
        return fail(SE2GPU_ERR_INVALID, "null argument");
    SE2_CUDA(cudaSetDevice(h->device));
    if (const int rc = dl_alloc(h)) return rc;
    const auto tnow = [] { return std::chrono::steady_clock::now(); };
    const auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t_begin = tnow();
    DevLoad& g = h->dl;
    Dev& d = h->d;
    cudaStream_t s = h->stream;
    const int* sc = g.sc_host;
    SE2_CUDA(cudaMemsetAsync(g.sc, 0, sizeof(int) * DL_SCALARS, s));

    if (h->loaded && g.valid && P == h->P && L == h->L && E == h->E && O == h->O && h->t_rank == h->rank && h->t_world == h->world) {
        SE2_LAUNCH(k_same_topology, nblocks(std::max(P, std::max(E, O)), DL_THREADS), DL_THREADS, 0, s, P, E, O, fixed, edge_pose, edge_point,
                   odo_i, odo_j, g.fixed, g.edge_pose, g.edge_point, g.odo_i, g.odo_j, g.sc);
        if (const int rc = read_scalars(h)) return rc;
        if (!sc[DL_DIFF]) {   // only the values are refreshed
            if (const int rc = device_values(h, P, L, poses, points, uv, info, odo_meas, odo_info)) return rc;
            SE2_CUDA(cudaStreamSynchronize(s));
            set_camera(h, fx, cx, cy, Tcb, huber_delta);
            if (h->sw.debug) fprintf(stderr, "[se2gpu_ba_set_problem_device] same topology: values refreshed in %.3f ms\n", ms(t_begin, tnow()));
            return SE2GPU_OK;
        }
        SE2_CUDA(cudaMemsetAsync(g.sc, 0, sizeof(int) * DL_SCALARS, s));
    }
    h->loaded = false;
    g.valid = false;
    // the host-side topology record belongs to the other entry: a host load after this one rebuilds
    h->t_edge_pose.clear(); h->t_edge_point.clear(); h->t_odo_i.clear(); h->t_odo_j.clear(); h->t_fixed.clear(); h->perm.clear();
    h->t_rank = h->t_world = -1;

    // ---------------------------------------------------------------------------------------------------- count phase
    const int rank = h->rank, world = h->world, Ol = rank == 0 ? O : 0;
    const size_t nw = ((size_t)P * P + 31) / 32;   // bitmap words of the nf x nf block table (nf <= P)
    int rc = SE2GPU_OK;
    if ((rc = grow_sort(h, std::max<size_t>(E, 2 * (size_t)O))) || (rc = grow(h, {&g.lo, &g.hi}, &g.cap_lm, L)) ||
        (rc = grow(h, {&g.pair_off}, &g.cap_off, (size_t)E + 1)) || (rc = grow(h, {&g.bits}, &g.cap_bits, nw + 1)) ||
        (rc = grow(h, {&g.wprefix}, &g.cap_wprefix, nw + 1))) return rc;
    int* lm_ptr = const_cast<int*>(d.lm_ptr);
    int* hidx = const_cast<int*>(d.hidx);
    int* pose_ptr = const_cast<int*>(d.pose_ptr);
    int* pose_odo_ptr = const_cast<int*>(d.pose_odo_ptr);
    SE2_CUDA(cudaMemsetAsync(lm_ptr, 0, sizeof(int) * (L + 1), s));
    SE2_CUDA(cudaMemsetAsync(pose_ptr, 0, sizeof(int) * (P + 1), s));
    SE2_CUDA(cudaMemsetAsync(pose_odo_ptr, 0, sizeof(int) * (P + 1), s));
    SE2_CUDA(cudaMemsetAsync(g.bits, 0, sizeof(unsigned) * (nw + 1), s));
    if (E + O > 0) SE2_LAUNCH(k_check, nblocks(E + O, DL_THREADS), DL_THREADS, 0, s, P, L, E, O, edge_pose, edge_point, odo_i, odo_j, g.sc);
    SE2_LAUNCH(k_hidx, 1, DL_THREADS, 0, s, P, fixed, hidx, g.sc);
    if (L) {
        SE2_LAUNCH(k_fill, nblocks(L, DL_THREADS), DL_THREADS, 0, s, g.lo, L, P);
        SE2_LAUNCH(k_fill, nblocks(L, DL_THREADS), DL_THREADS, 0, s, g.hi, L, -1);
    }
    const int* sorted = nullptr;
    if (E) {   // landmark sort: perm, lm_ptr
        SE2_LAUNCH(k_lm_keys, nblocks(E, DL_THREADS), DL_THREADS, 0, s, P, L, E, rank, world, edge_pose, edge_point, hidx, g.k0, g.v0, lm_ptr, g.lo, g.hi);
        if ((rc = radix_sort(h, E, L, &sorted))) return rc;
        SE2_CUDA(cudaMemcpyAsync(g.perm, sorted, sizeof(int) * E, cudaMemcpyDeviceToDevice, s));
    }
    if ((rc = scan(h, lm_ptr, L))) return rc;
    const int* El_ptr = lm_ptr + L;
    if (E) {   // e_pose, e_hidx; pose lists over sorted edges
        SE2_LAUNCH(k_sorted_edges, nblocks(E, DL_THREADS), DL_THREADS, 0, s, P, E, El_ptr, g.perm, edge_pose, hidx, const_cast<int*>(d.e_pose),
                   const_cast<int*>(d.e_hidx), g.k0, g.v0, pose_ptr, g.sc);
        if ((rc = radix_sort(h, E, P, &sorted))) return rc;
        SE2_CUDA(cudaMemcpyAsync(const_cast<int*>(d.pose_edges), sorted, sizeof(int) * E, cudaMemcpyDeviceToDevice, s));
    }
    if ((rc = scan(h, pose_ptr, P))) return rc;
    if (O) {   // pose lists over odometry edges
        SE2_LAUNCH(k_odo_keys, nblocks(2 * O, DL_THREADS), DL_THREADS, 0, s, P, Ol, O, odo_i, odo_j, hidx, g.k0, g.v0, pose_odo_ptr, g.sc);
        if ((rc = radix_sort(h, 2 * O, P, &sorted))) return rc;
        SE2_CUDA(cudaMemcpyAsync(const_cast<int*>(d.pose_odo), sorted, sizeof(int) * 2 * O, cudaMemcpyDeviceToDevice, s));
    }
    if ((rc = scan(h, pose_odo_ptr, P))) return rc;
    SE2_LAUNCH(k_pair_count, nblocks(std::max(std::max(E, P), Ol), DL_THREADS), DL_THREADS, 0, s, P, E, Ol, lm_ptr, El_ptr, g.perm,
               edge_point, d.e_hidx, odo_i, odo_j, hidx, g.sc, g.bits, g.pair_off);
    if ((rc = scan(h, g.pair_off, E))) return rc;
    SE2_LAUNCH(k_popc, nblocks((long long)nw, DL_THREADS), DL_THREADS, 0, s, g.bits, (int)nw, g.wprefix);
    if ((rc = scan(h, g.wprefix, (int)nw))) return rc;
    SE2_CUDA(cudaGetLastError());
    // El, pairs and blocks are the scans' totals
    SE2_CUDA(cudaMemcpyAsync(g.sc + DL_EL, El_ptr, sizeof(int), cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(g.sc + DL_NPAIRS, g.pair_off + E, sizeof(int), cudaMemcpyDeviceToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(g.sc + DL_NBLK, g.wprefix + nw, sizeof(int), cudaMemcpyDeviceToDevice, s));
    if ((rc = read_scalars(h))) return rc;
    const auto t_count = tnow();
    if (sc[DL_ERR]) return fail(SE2GPU_ERR_INVALID, "an edge or odometry edge references a missing vertex");
    const int nf = sc[DL_NF], n = 3 * nf, El = sc[DL_EL], npairs = sc[DL_NPAIRS], nblk = sc[DL_NBLK], nodob = sc[DL_NODOB];
    if (nodob + 1 > 2 * (h->maxO ? h->maxO : 1) + 1) return fail(SE2GPU_ERR_CAPACITY, "too many odometry blocks");

    // ----------------------------------------------------------------------------------------------------- fill phase
    // the block lists are sized for the serving order too (W * maxlen <= max(12 W, nblk + W)): growing them after the
    // fill would drop their contents
    const size_t W = std::max(h->pk_grid, 1);
    if ((rc = ensure_cap(h, npairs, std::max<size_t>(std::max<size_t>(nblk + W, 12 * W), nodob), 0)) || (rc = grow_sort(h, npairs)) ||
        (rc = grow(h, {&g.g1, &g.g2}, &g.cap_pairs, npairs)) || (rc = grow(h, {&g.planin}, &g.cap_plan, (size_t)nf + 2 * (size_t)nblk))) return rc;
    int* blk_a = const_cast<int*>(d.blk_a);
    int* blk_b = const_cast<int*>(d.blk_b);
    int* blk_pair_ptr = const_cast<int*>(d.blk_pair_ptr);
    int* blk_odo_ptr = const_cast<int*>(d.blk_odo_ptr);
    SE2_CUDA(cudaMemsetAsync(blk_pair_ptr, 0, sizeof(int) * (nblk + 1), s));
    SE2_CUDA(cudaMemsetAsync(blk_odo_ptr, 0, sizeof(int) * (nblk + 1), s));
    SE2_LAUNCH(k_blocks, nblocks((long long)nw, DL_THREADS), DL_THREADS, 0, s, g.bits, g.wprefix, (int)nw, g.sc, blk_a, blk_b);
    if (El) SE2_LAUNCH(k_pair_fill, nblocks(El, DL_THREADS), DL_THREADS, 0, s, El, lm_ptr, g.perm, edge_point, d.e_hidx, g.sc, g.bits,
                       g.wprefix, g.pair_off, g.k0, g.v0, g.g1, g.g2, blk_pair_ptr);
    if (npairs) {   // pairs by block, landmark order kept inside a block
        if ((rc = radix_sort(h, npairs, nblk, &sorted))) return rc;
        SE2_LAUNCH(k_pair_gather, nblocks(npairs, DL_THREADS), DL_THREADS, 0, s, npairs, sorted, g.g1, g.g2, const_cast<int*>(d.pair_e1),
                   const_cast<int*>(d.pair_e2));
    }
    if ((rc = scan(h, blk_pair_ptr, nblk))) return rc;
    if (Ol) {   // odometry by block, odometry order kept inside a block
        SE2_LAUNCH(k_odo_blocks, nblocks(Ol, DL_THREADS), DL_THREADS, 0, s, Ol, nblk, odo_i, odo_j, hidx, g.sc, g.bits, g.wprefix, g.k0, g.v0, blk_odo_ptr);
        if ((rc = radix_sort(h, Ol, nblk, &sorted))) return rc;
        if (nodob) SE2_CUDA(cudaMemcpyAsync(const_cast<int*>(d.blk_odo), sorted, sizeof(int) * nodob, cudaMemcpyDeviceToDevice, s));
    }
    if ((rc = scan(h, blk_odo_ptr, nblk))) return rc;
    int* bmax = g.planin;
    if (nf) SE2_LAUNCH(k_iota, nblocks(nf, DL_THREADS), DL_THREADS, 0, s, bmax, nf);
    if (nf && L + O > 0) SE2_LAUNCH(k_env, nblocks(std::max(L, O), DL_THREADS), DL_THREADS, 0, s, P, L, O, g.lo, g.hi, odo_i, odo_j, hidx, bmax);
    SE2_LAUNCH(k_env_scan_weights, 1, DL_THREADS, 0, s, nf, nblk, bmax, blk_a, blk_b, blk_pair_ptr, pose_ptr, g.planin + nf, g.planin + nf + nblk);
    SE2_CUDA(cudaGetLastError());
    const size_t nplan = (size_t)nf + 2 * (size_t)nblk;
    g.planin_host.resize(std::max<size_t>(nplan, 1));
    SE2_CUDA(cudaMemcpyAsync(g.planin_host.data(), g.planin, sizeof(int) * nplan, cudaMemcpyDeviceToHost, s));
    const auto t_fill_enq = tnow();
    // the rest of the device work does not depend on the host's decisions: enqueue it before waiting for the plan input
    SE2_CUDA(cudaMemcpyAsync(g.fixed, fixed, P, cudaMemcpyDeviceToDevice, s));
    if (E) {
        SE2_CUDA(cudaMemcpyAsync(g.edge_pose, edge_pose, sizeof(int) * E, cudaMemcpyDeviceToDevice, s));
        SE2_CUDA(cudaMemcpyAsync(g.edge_point, edge_point, sizeof(int) * E, cudaMemcpyDeviceToDevice, s));
    }
    if (O) {
        SE2_CUDA(cudaMemcpyAsync(g.odo_i, odo_i, sizeof(int) * O, cudaMemcpyDeviceToDevice, s));
        SE2_CUDA(cudaMemcpyAsync(g.odo_j, odo_j, sizeof(int) * O, cudaMemcpyDeviceToDevice, s));
    }
    if (Ol) {
        SE2_CUDA(cudaMemcpyAsync(const_cast<int*>(d.o_i), odo_i, sizeof(int) * Ol, cudaMemcpyDeviceToDevice, s));
        SE2_CUDA(cudaMemcpyAsync(const_cast<int*>(d.o_j), odo_j, sizeof(int) * Ol, cudaMemcpyDeviceToDevice, s));
    }
    d.E = El; d.O = Ol;
    if ((rc = device_values(h, P, L, poses, points, uv, info, odo_meas, odo_info))) return rc;
    SE2_CUDA(cudaStreamSynchronize(s));
    const auto t_fill = tnow();

    // ---------------------------------------------------------------------------------------------- host decisions
    const std::vector<int> bmax_h(g.planin_host.begin(), g.planin_host.begin() + nf);
    Decisions w;
    decide(w, nf, bmax_h.data(), g.planin_host.data() + nf, g.planin_host.data() + nf + nblk, nblk, world, h->pk_grid, h->sw);
    if ((rc = ensure_cap(h, npairs, nblk, w.env_idx.size()))) return rc;
    h->nenv = (int)w.env_idx.size();
    if (h->ssum) SE2_CUDA(cudaMemsetAsync(h->ssum, 0, sizeof(double) * ((size_t)SMEM_CHOL_MAX_N * SMEM_CHOL_MAX_N + SMEM_CHOL_MAX_N + 8), s));
    se2band::release(h->band);
    if (n > SMEM_CHOL_MAX_N && !h->sw.no_band) se2band::plan(h->band, nf, bmax_h, h->smem_optin);
    const bool band = h->band.active;
    int* pl = h->plan;
    pl[0] = nf; pl[1] = n; pl[2] = 2;
    pl[3] = 0; for (int a = 0; a < nf; ++a) pl[3] = std::max(pl[3], bmax_h[a] - a);
    pl[4] = n <= SMEM_CHOL_MAX_N ? (w.tw_m0 > 0 ? 1 : 0) : (band ? 2 : 3);
    pl[5] = w.tw_m0; pl[6] = w.tw_w; pl[7] = band ? h->band.w : 0; pl[8] = band ? h->band.p : 0;
    pl[9] = h->pk_grid; pl[10] = w.workers; pl[11] = nblk; pl[12] = w.maxlen; pl[13] = w.uncached;
    const struct { const int* dst; const int* src; size_t count; } arrays[] = {
        {d.colmax, w.colmax.data(), w.colmax.size()}, {d.tw_cmax1, w.tw_cmax1.data(), w.tw_cmax1.size()},
        {d.blk_order, w.blk_order.data(), w.blk_order.size()}, {h->env_idx, w.env_idx.data(), w.env_idx.size()}};
    size_t bytes = 64 * 8;
    for (const auto& a : arrays) bytes += sizeof(int) * a.count;
    h->arena.reserve(bytes);   // on failure the uploads fall back to pageable copies
    for (const auto& a : arrays) if ((rc = up(h, a.dst, a.src, a.count))) return rc;
    const size_t S_elems = band ? h->band.band_elems : (size_t)n * n;
    SE2_CUDA(cudaMemsetAsync(h->red, 0, sizeof(double) * (S_elems + n + 8), s));
    const auto t_host = tnow();
    SE2_CUDA(cudaStreamSynchronize(s));
    if (h->sw.debug)
        fprintf(stderr, "[se2gpu_ba_set_problem_device] count %.3f ms, sort/fill enqueue %.3f ms, values + drain %.3f ms, host decisions %.3f ms, "
                "upload + drain %.3f ms (P %d L %d E %d blocks %d pairs %d)\n", ms(t_begin, t_count), ms(t_count, t_fill_enq),
                ms(t_fill_enq, t_fill), ms(t_fill, t_host), ms(t_host, tnow()), P, L, E, nblk, npairs);

    d.P = P; d.L = L; d.nf = nf; d.n = n; d.nblk = nblk; d.rank = rank; d.world = world;
    d.nord = (int)w.blk_order.size(); d.tw_m0 = w.tw_m0; d.tw_w = w.tw_w;
    d.S = h->red; d.bs = h->red + S_elems; d.scal = d.bs + n; d.sbw = band ? h->band.bw : 0;
    d.nb_lm = (L + LM_THREADS - 1) / LM_THREADS; d.nb_odo = (Ol + LM_THREADS - 1) / LM_THREADS;
    h->nb_scale = (std::max(L, P) + LM_THREADS - 1) / LM_THREADS;
    set_camera(h, fx, cx, cy, Tcb, huber_delta);
    h->P = P; h->L = L; h->E = E; h->O = O;
    h->t_rank = h->rank; h->t_world = h->world;
    set_struct_len(h, sc[DL_NPE], sc[DL_NPO], npairs, nodob, w.tw_cmax1.size(), w.blk_order.size());
    h->plan_in.assign(g.planin_host.begin(), g.planin_host.begin() + nplan); h->plan_grid = h->pk_grid;
    g.valid = true;
    h->loaded = true;
    return SE2GPU_OK;
}

}  // namespace

namespace se2ba {

// The decisions that depend on the number of CTAs - the two-sided split and the serving order of the Schur blocks - made again
// by the one planner from the inputs the load kept, and their O(nf + nblk) results uploaded. The envelope and the sharded
// exchange list do not depend on it. A serving order of W workers has at most max(12 W, nblk + W) positions; ensure_cap
// leaves the block lists room for nblk + 1024, so clusters of up to 8 CTAs always fit (the check below is a guard).
int plan_for_grid(se2gpu_ba* h, int grid) {
    if (h->plan_grid == grid) return SE2GPU_OK;
    Dev& d = h->d;
    const int nf = d.nf, nblk = d.nblk;
    const int* in = h->plan_in.data();
    Decisions w;
    decide(w, nf, in, in + nf, in + nf + nblk, nblk, h->world, grid, h->sw);
    if (w.blk_order.size() > h->cap_blk) return fail(SE2GPU_ERR_CAPACITY, "serving order of %zu positions exceeds the block lists", w.blk_order.size());
    h->arena.reserve(sizeof(int) * (w.tw_cmax1.size() + w.blk_order.size()) + 256);   // on failure the uploads fall back to pageable copies
    int rc = up(h, d.tw_cmax1, w.tw_cmax1.data(), w.tw_cmax1.size());
    if (rc == SE2GPU_OK) rc = up(h, d.blk_order, w.blk_order.data(), w.blk_order.size());
    if (rc != SE2GPU_OK) return rc;
    d.nord = (int)w.blk_order.size(); d.tw_m0 = w.tw_m0; d.tw_w = w.tw_w;
    h->struct_len[SE2GPU_BA_STRUCT_TW_CMAX1] = (long long)w.tw_cmax1.size();   // se2gpu_ba_debug_structure shows the plan in use
    h->struct_len[SE2GPU_BA_STRUCT_BLK_ORDER] = (long long)w.blk_order.size();
    h->plan_grid = grid;
    return SE2GPU_OK;
}

}  // namespace se2ba

extern "C" {

int se2gpu_ba_set_problem_device(se2gpu_ba* h, int P, int L, int E, int O, const double* d_poses, const uint8_t* d_fixed,
                                 const double* d_points, const int* d_edge_pose, const int* d_edge_point, const double* d_uv,
                                 const double* d_info, const int* d_odo_i, const int* d_odo_j, const double* d_odo_meas,
                                 const double* d_odo_info, double fx, double cx, double cy, const double* Tcb, double huber_delta) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    const int rc = load_window_device(h, P, L, E, O, d_poses, d_fixed, d_points, d_edge_pose, d_edge_point, d_uv, d_info, d_odo_i,
                                      d_odo_j, d_odo_meas, d_odo_info, fx, cx, cy, Tcb, huber_delta);
    if (rc != SE2GPU_OK) {
        cudaStreamSynchronize(h->stream);   // nothing of the rejected build still reads the caller's buffers
        unload(h);                          // a rejected window leaves none loaded, never the previous one
    }
    return rc;
}

int se2gpu_ba_build_information_device(int P, int L, int E, const float* d_view_mp, const int* d_edge_pose, const int* d_edge_point,
                                       const int* d_octave, const float* d_kf_Rcw, const float* d_kf_twb_xy, const float* d_mp_pos,
                                       const float* d_level_sigma2, int nlevels, float fx, float xrot_info, float z_info, double* d_info,
                                       void* stream) {
    if (P <= 0 || L < 0 || E < 0 || nlevels <= 0) return fail(SE2GPU_ERR_INVALID, "bad sizes");
    if (E == 0) return SE2GPU_OK;
    if (!d_view_mp || !d_edge_pose || !d_edge_point || !d_octave || !d_kf_Rcw || !d_kf_twb_xy || !d_mp_pos || !d_level_sigma2 || !d_info)
        return fail(SE2GPU_ERR_INVALID, "null argument");
    { const int rc = se2gpu::require_device(); if (rc) return rc; }
    InfoArgs a{};
    a.P = P; a.L = L; a.E = E; a.nlevels = nlevels; a.fx = fx;
    a.sigma_rotxy = 1.f / xrot_info;       // as se2gpu_ba_build_information
    a.sigma_z = 1.f / z_info;
    a.info = d_info; a.lc = d_view_mp; a.edge_pose = d_edge_pose; a.edge_point = d_edge_point; a.octave = d_octave;
    a.Rcw = d_kf_Rcw; a.twb = d_kf_twb_xy; a.lw = d_mp_pos; a.level_sigma2 = d_level_sigma2;
    SE2_LAUNCH(k_edge_information, (E + 255) / 256, 256, 0, (cudaStream_t)stream, a);
    SE2_CUDA(cudaGetLastError());
    return SE2GPU_OK;
}

int se2gpu_ba_debug_structure(se2gpu_ba* h, int which, int* out, int n_out) {
    if (!h || !h->loaded) return fail(SE2GPU_ERR_INVALID, "no problem loaded");
    if (which < 0 || which >= SE2GPU_BA_STRUCT_COUNT) return fail(SE2GPU_ERR_INVALID, "no structure array %d", which);
    if (n_out < 0 || (n_out > 0 && !out)) return fail(SE2GPU_ERR_INVALID, "bad output buffer");
    const Dev& d = h->d;
    const void* const src[SE2GPU_BA_STRUCT_COUNT] = {
        d.hidx, d.lm_ptr, h->dl.perm, d.e_pose, d.e_hidx, d.pose_ptr, d.pose_edges, d.pose_odo_ptr, d.pose_odo, d.blk_a, d.blk_b,
        d.blk_pair_ptr, d.pair_e1, d.pair_e2, d.blk_odo_ptr, d.blk_odo, d.colmax, d.tw_cmax1, d.blk_order, h->env_idx, d.o_i, d.o_j,
        d.e_u, d.e_v, d.e_w00, d.e_w01, d.e_w11, d.o_m, d.o_w};
    const long long len = h->struct_len[which];
    const size_t count = (size_t)std::min<long long>(n_out, len);
    if (count == 0) return (int)len;
    if (which == SE2GPU_BA_STRUCT_PERM && !h->dl.valid) {   // a host load keeps the landmark sort on the host
        memcpy(out, h->perm.data(), sizeof(int) * count);
        return (int)len;
    }
    SE2_CUDA(cudaSetDevice(h->device));
    SE2_CUDA(cudaMemcpyAsync(out, src[which], sizeof(int) * count, cudaMemcpyDeviceToHost, h->stream));
    SE2_CUDA(cudaStreamSynchronize(h->stream));
    return (int)len;
}

}  // extern "C"
