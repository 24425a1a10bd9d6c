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
    int E;
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

struct WindowPlan {   // everything derived from the graph structure alone
    int nf = 0, n = 0, El = 0, Ol = 0, nblk = 0;
    size_t npairs = 0;
    bool sorted_structure = false;   // block and pair lists by comparison sort (nf^2 beyond the dense table)
    int tw_m0 = 0, tw_w = 0;         // two-sided reduced solve (Dev::tw_m0)
    int workers = 0, maxlen = 0, uncached = 0;   // persistent kernel: worker CTAs, longest worker list, workers running the uncached Schur sweep
    std::vector<int> hidx, lm_ptr, perm, pose_ptr, pose_edges, pose_odo_ptr, pose_odo;
    std::vector<int> blk_a, blk_b, blk_pair_ptr, blk_odo_ptr, blk_odo, bmax, colmax, env_idx, tw_cmax1, blk_order;
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
    for (int b = 0; b < nblk; ++b) {
        long long wt = blk_pair_ptr[b + 1] - blk_pair_ptr[b] + 8;
        if (blk_a[b] == blk_b[b]) wt += pose_ptr[blk_a[b] + 1] - pose_ptr[blk_a[b]];
        byw[b] = {-wt, b};
    }
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
            const int np = blk_pair_ptr[b + 1] - blk_pair_ptr[b], ne = blk_a[b] == blk_b[b] ? pose_ptr[blk_a[b] + 1] - pose_ptr[blk_a[b]] : 0;
            if (no >= PK_MAXOWN || off + 2 * np + ne > arena_ints) break;
            off += 2 * np + ne; ++no;
        }
        if (no < (int)l.size()) ++w.uncached;
    }
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
    a.E = E; a.nlevels = nlevels; a.fx = fx;
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
