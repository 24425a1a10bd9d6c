// The host's half of the SE(3)-XYZ window BA's initializeOptimization (se3_ba.cu), plain C++ so that it also compiles for a
// host test (tests/native/se3_plan_profile.cpp): which keyframes are free, the reduced system's RCM order and 6 x 6 block
// envelope (global_ba_plan.h over the block graph of the window), and every fixed-order gather list of the kernel.
#pragma once
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

#include "global_ba_plan.h"

namespace se2gpu {
namespace se3ba {

struct Plan {
    gba::Plan G;                 // the block graph: odometry links first, then the co-observation pairs of free keyframes
    std::vector<int> flags;      // [N] bit 0 fixed, bit 1 prior (as given)
    // the odometry's contributions to H and b, G's gather lists without the co-observation links (those enter through the
    // Schur complement)
    std::vector<int> diag_ptr;   // [nf + 1]
    std::vector<int> diag_code;  // odometry * 4 + gba::kFromDiag / kToDiag, ascending
    std::vector<int64_t> off_blk;  // [S] envelope block of each off-diagonal block an odometry link touches
    std::vector<int> off_ptr;    // [S + 1]
    std::vector<int> off_code;   // odometry * 4 + gba::kOffDiag / kOffDiagT, ascending
    std::vector<int> kf_ptr, kf_edges;  // [nf + 1], the projection edges of the keyframe at each position, ascending
    std::vector<int> pt_ptr, pt_edges;  // [L + 1], each point's projection edges, ascending
    // Schur pairs of every envelope block: the diagonal block of p lists (e, e) for p's edges in ascending edge order; block
    // (p, q), p > q, lists (a, b) with a to p and b to q on one point, in ascending point order
    std::vector<int64_t> pair_ptr;  // [env blocks + 1]
    std::vector<int> pair_a, pair_b;
};

// N keyframes with fixed / prior [N], O odometry links from / to, L points and E projection edges e_pt / e_kf (indices
// already checked)
inline Plan make_plan(int N, const uint8_t* fixed, const uint8_t* prior, int O, const int* from, const int* to, int L, int E,
                      const int* e_pt, const int* e_kf) {
    Plan P;
    // a keyframe no edge touches is not in the graph g2o optimises; a free one that is takes part in the reduced system
    std::vector<uint8_t> active(N, 0), fx(N, 1);
    for (int v = 0; v < N; ++v) active[v] = prior[v] ? 1 : 0;
    for (int o = 0; o < O; ++o) active[from[o]] = active[to[o]] = 1;
    for (int e = 0; e < E; ++e) active[e_kf[e]] = 1;
    for (int v = 0; v < N; ++v) fx[v] = (fixed[v] || !active[v]) ? 1 : 0;
    std::vector<int>& pt_ptr = P.pt_ptr;
    std::vector<int>& pt_edges = P.pt_edges;
    pt_ptr.assign(L + 1, 0);
    pt_edges.resize(E);
    for (int e = 0; e < E; ++e) ++pt_ptr[e_pt[e] + 1];
    for (int j = 0; j < L; ++j) pt_ptr[j + 1] += pt_ptr[j];
    {
        std::vector<int> f(pt_ptr.begin(), pt_ptr.end() - 1);
        for (int e = 0; e < E; ++e) pt_edges[f[e_pt[e]]++] = e;
    }
    // the block graph: odometry links, then every pair of free keyframes that observe a common point
    std::vector<int> gf(from, from + O), gt(to, to + O);
    {
        std::vector<std::pair<int, int>> pr;
        for (int j = 0; j < L; ++j)
            for (int q = pt_ptr[j]; q < pt_ptr[j + 1]; ++q)
                for (int r = q + 1; r < pt_ptr[j + 1]; ++r) {
                    const int u = e_kf[pt_edges[q]], v = e_kf[pt_edges[r]];
                    if (!fx[u] && !fx[v]) pr.push_back({std::min(u, v), std::max(u, v)});
                }
        std::sort(pr.begin(), pr.end());
        pr.erase(std::unique(pr.begin(), pr.end()), pr.end());
        for (const auto& x : pr) { gf.push_back(x.first); gt.push_back(x.second); }
    }
    P.G = gba::make_plan(N, fx.data(), (int)gf.size(), gf.data(), gt.data());
    const gba::Plan& G = P.G;
    const int nf = G.n_free;
    // odometry contributions only
    P.diag_ptr.assign(nf + 1, 0);
    P.off_ptr.assign(1, 0);
    for (int p = 0; p < nf; ++p) {
        for (int q = G.diag_ptr[p]; q < G.diag_ptr[p + 1]; ++q)
            if ((G.diag_code[q] >> 2) < O) P.diag_code.push_back(G.diag_code[q]);
        P.diag_ptr[p + 1] = (int)P.diag_code.size();
    }
    for (size_t s = 0; s < G.off_blk.size(); ++s) {
        const size_t before = P.off_code.size();
        for (int q = G.off_ptr[s]; q < G.off_ptr[s + 1]; ++q)
            if ((G.off_code[q] >> 2) < O) P.off_code.push_back(G.off_code[q]);
        if (P.off_code.size() != before) { P.off_blk.push_back(G.off_blk[s]); P.off_ptr.push_back((int)P.off_code.size()); }
    }
    // projection edges per position, ascending
    P.kf_ptr.assign(nf + 1, 0);
    {
        std::vector<std::vector<int>> by(nf);
        for (int e = 0; e < E; ++e)
            if (G.pos[e_kf[e]] >= 0) by[G.pos[e_kf[e]]].push_back(e);
        for (int p = 0; p < nf; ++p) { P.kf_edges.insert(P.kf_edges.end(), by[p].begin(), by[p].end()); P.kf_ptr[p + 1] = (int)P.kf_edges.size(); }
    }
    // the Schur pairs
    const int64_t env = G.env_blocks();
    std::vector<std::vector<std::pair<int, int>>> pb(env);
    for (int p = 0; p < nf; ++p)
        for (int q = P.kf_ptr[p]; q < P.kf_ptr[p + 1]; ++q) pb[G.blk(p, p)].push_back({P.kf_edges[q], P.kf_edges[q]});
    for (int j = 0; j < L; ++j)
        for (int q = pt_ptr[j]; q < pt_ptr[j + 1]; ++q)
            for (int r = pt_ptr[j]; r < pt_ptr[j + 1]; ++r) {
                const int ea = pt_edges[q], eb = pt_edges[r], pa = G.pos[e_kf[ea]], pq = G.pos[e_kf[eb]];
                if (pa < 0 || pq < 0 || pa <= pq) continue;
                pb[G.blk(pa, pq)].push_back({ea, eb});
            }
    P.pair_ptr.assign(env + 1, 0);
    for (int64_t k = 0; k < env; ++k) {
        for (const auto& x : pb[k]) { P.pair_a.push_back(x.first); P.pair_b.push_back(x.second); }
        P.pair_ptr[k + 1] = (int64_t)P.pair_a.size();
    }
    P.flags.resize(N);
    for (int v = 0; v < N; ++v) P.flags[v] = (fixed[v] ? 1 : 0) | (prior[v] ? 2 : 0);
    return P;
}

}  // namespace se3ba
}  // namespace se2gpu
