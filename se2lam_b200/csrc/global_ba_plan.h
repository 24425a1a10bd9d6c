// Symbolic phase of the global pose graph (global_ba.cu), plain C++ so that it also compiles for a host test
// (tests/native/global_ba_plan_host.cpp). Built on the host once per call, because every GlobalBA sees new keyframes and new
// feature edges:
//  1. the block graph of the free vertices (an edge between two free vertices couples their 6 x 6 blocks);
//  2. its reverse Cuthill-McKee order: components in order of their lowest-degree, lowest-index vertex, neighbours visited
//     by ascending (degree, index), so the order depends on the topology alone;
//  3. the block envelope of the lower triangle in that order: row p holds blocks first[p] .. p, and an envelope LDL^T never
//     fills outside it;
//  4. fixed-order gather lists: for every free vertex and every off-diagonal nonzero block, the edge contributions in
//     ascending edge index, so H and b are summed in one order on every run.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace se2gpu {
namespace gba {

// contribution codes: edge * 4 + kind
enum Kind { kFromDiag = 0, kToDiag = 1, kOffDiag = 2, kOffDiagT = 3 };  // H_ii, H_jj, H_ij, H_ij^T

struct Plan {
    int n_free = 0;
    std::vector<int> pos;        // [N] vertex -> RCM position, -1 when fixed
    std::vector<int> vert;       // [n_free] position -> vertex
    std::vector<int> first;      // [n_free] first block column of block row p
    std::vector<int64_t> rowoff; // [n_free + 1] block offset of row p in the envelope
    std::vector<int> col_ptr;    // [n_free + 1] rows p > k with first[p] <= k, per column k ...
    std::vector<int> col_rows;   // ... ascending
    std::vector<int> diag_ptr;   // [n_free + 1] contributions to the diagonal block and to b of position p ...
    std::vector<int> diag_code;  // ... edge * 4 + kFromDiag / kToDiag, ascending edge
    std::vector<int64_t> off_blk;  // [S] envelope block of each nonzero off-diagonal block, in envelope order
    std::vector<int> off_ptr;    // [S + 1]
    std::vector<int> off_code;   // edge * 4 + kOffDiag / kOffDiagT, ascending edge
    int64_t env_blocks() const { return rowoff.empty() ? 0 : rowoff.back(); }
    int64_t blk(int p, int q) const { return rowoff[p] + (q - first[p]); }  // block (p, q), first[p] <= q <= p
};

// N vertices, fixed [N] (nonzero = fixed), E edges from / to (indices already checked)
inline Plan make_plan(int N, const uint8_t* fixed, int E, const int* from, const int* to) {
    Plan P;
    P.pos.assign(N, -1);
    std::vector<int> fidx(N, -1), fverts;
    for (int v = 0; v < N; ++v)
        if (!fixed[v]) { fidx[v] = (int)fverts.size(); fverts.push_back(v); }
    const int n = (int)fverts.size();
    P.n_free = n;
    // 1. adjacency of the free vertices, duplicates merged
    std::vector<std::vector<int>> adj(n);
    for (int e = 0; e < E; ++e) {
        const int a = fidx[from[e]], b = fidx[to[e]];
        if (a < 0 || b < 0 || a == b) continue;
        adj[a].push_back(b);
        adj[b].push_back(a);
    }
    std::vector<int> deg(n);
    for (int a = 0; a < n; ++a) {
        std::sort(adj[a].begin(), adj[a].end());
        adj[a].erase(std::unique(adj[a].begin(), adj[a].end()), adj[a].end());
        deg[a] = (int)adj[a].size();
    }
    // 2. Cuthill-McKee by breadth-first search, then reversed
    std::vector<int> seeds(n), order;
    for (int a = 0; a < n; ++a) seeds[a] = a;
    std::stable_sort(seeds.begin(), seeds.end(), [&](int x, int y) { return deg[x] < deg[y]; });
    std::vector<char> seen(n, 0);
    order.reserve(n);
    for (int s : seeds) {
        if (seen[s]) continue;
        seen[s] = 1;
        size_t head = order.size();
        order.push_back(s);
        while (head < order.size()) {
            const int a = order[head++];
            std::vector<int> nb;
            for (int b : adj[a])
                if (!seen[b]) { seen[b] = 1; nb.push_back(b); }
            std::sort(nb.begin(), nb.end(), [&](int x, int y) { return deg[x] != deg[y] ? deg[x] < deg[y] : x < y; });
            order.insert(order.end(), nb.begin(), nb.end());
        }
    }
    std::reverse(order.begin(), order.end());
    P.vert.resize(n);
    std::vector<int> fpos(n);
    for (int p = 0; p < n; ++p) { fpos[order[p]] = p; P.vert[p] = fverts[order[p]]; P.pos[fverts[order[p]]] = p; }
    // 3. the envelope
    P.first.resize(n);
    for (int p = 0; p < n; ++p) {
        int f = p;
        for (int b : adj[order[p]]) f = std::min(f, fpos[b]);
        P.first[p] = f;
    }
    P.rowoff.assign(n + 1, 0);
    for (int p = 0; p < n; ++p) P.rowoff[p + 1] = P.rowoff[p] + (p - P.first[p] + 1);
    std::vector<int> cnt(n + 1, 0);
    for (int p = 0; p < n; ++p)
        for (int k = P.first[p]; k < p; ++k) ++cnt[k + 1];
    P.col_ptr.assign(n + 1, 0);
    for (int k = 0; k < n; ++k) P.col_ptr[k + 1] = P.col_ptr[k] + cnt[k + 1];
    P.col_rows.resize(P.col_ptr[n]);
    std::vector<int> fill(P.col_ptr.begin(), P.col_ptr.end() - 1);
    for (int p = 0; p < n; ++p)
        for (int k = P.first[p]; k < p; ++k) P.col_rows[fill[k]++] = p;
    // 4. gather lists
    std::vector<std::vector<int>> dg(n);
    std::vector<std::pair<int64_t, int>> off;  // (envelope block, code)
    for (int e = 0; e < E; ++e) {
        const int a = P.pos[from[e]], b = P.pos[to[e]];
        if (a >= 0) dg[a].push_back(e * 4 + kFromDiag);
        if (b >= 0) dg[b].push_back(e * 4 + kToDiag);
        if (a >= 0 && b >= 0) off.push_back(a > b ? std::make_pair(P.blk(a, b), e * 4 + kOffDiag) : std::make_pair(P.blk(b, a), e * 4 + kOffDiagT));
    }
    P.diag_ptr.assign(n + 1, 0);
    for (int p = 0; p < n; ++p) {
        P.diag_ptr[p + 1] = P.diag_ptr[p] + (int)dg[p].size();
        P.diag_code.insert(P.diag_code.end(), dg[p].begin(), dg[p].end());
    }
    std::stable_sort(off.begin(), off.end(), [](const std::pair<int64_t, int>& x, const std::pair<int64_t, int>& y) { return x.first < y.first; });
    P.off_ptr.push_back(0);
    for (size_t i = 0; i < off.size(); ++i) {
        if (i == 0 || off[i].first != off[i - 1].first) {
            if (i) P.off_ptr.push_back((int)i);
            P.off_blk.push_back(off[i].first);
        }
        P.off_code.push_back(off[i].second);
    }
    if (!off.empty()) P.off_ptr.push_back((int)off.size());
    return P;
}

}  // namespace gba
}  // namespace se2gpu
