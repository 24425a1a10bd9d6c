// Host check of the global pose graph's symbolic phase (se2lam_b200/csrc/global_ba_plan.h): on synthetic topologies the
// reverse Cuthill-McKee order is a valid permutation of the free vertices, two plans of one graph are identical, the
// envelope bounds every nonzero block, the column lists are the envelope's transpose, and every edge contribution is in
// exactly one gather list. A chain closed into a ring keeps a band of two blocks. Prints "ok" and returns 0 on success.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <set>
#include <vector>

#include "../../se2lam_b200/csrc/global_ba_plan.h"

using se2gpu::gba::Plan;

static int g_fail = 0;
#define CHECK(c, ...) do { if (!(c)) { std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); ++g_fail; } } while (0)

struct Graph { int N; std::vector<uint8_t> fixed; std::vector<int> from, to; const char* name; };

static bool same(const Plan& a, const Plan& b) {
    return a.n_free == b.n_free && a.pos == b.pos && a.vert == b.vert && a.first == b.first && a.rowoff == b.rowoff &&
           a.col_ptr == b.col_ptr && a.col_rows == b.col_rows && a.diag_ptr == b.diag_ptr && a.diag_code == b.diag_code &&
           a.off_blk == b.off_blk && a.off_ptr == b.off_ptr && a.off_code == b.off_code;
}

static void check(const Graph& g) {
    const int E = (int)g.from.size();
    const Plan P = se2gpu::gba::make_plan(g.N, g.fixed.data(), E, g.from.data(), g.to.data());
    CHECK(same(P, se2gpu::gba::make_plan(g.N, g.fixed.data(), E, g.from.data(), g.to.data())), "%s: plan not deterministic", g.name);
    int nf = 0;
    for (int v = 0; v < g.N; ++v) nf += !g.fixed[v];
    CHECK(P.n_free == nf && (int)P.vert.size() == nf, "%s: %d free vertices, plan has %d", g.name, nf, P.n_free);
    std::vector<int> seen(nf, 0);
    for (int v = 0; v < g.N; ++v) {
        if (g.fixed[v]) { CHECK(P.pos[v] == -1, "%s: fixed vertex %d has a position", g.name, v); continue; }
        CHECK(P.pos[v] >= 0 && P.pos[v] < nf, "%s: position of %d out of range", g.name, v);
        if (P.pos[v] < 0 || P.pos[v] >= nf) continue;
        ++seen[P.pos[v]];
        CHECK(P.vert[P.pos[v]] == v, "%s: vert is not the inverse of pos at %d", g.name, v);
    }
    for (int p = 0; p < nf; ++p) CHECK(seen[p] == 1, "%s: position %d taken %d times", g.name, p, seen[p]);
    for (int p = 0; p < nf; ++p) {
        CHECK(P.first[p] >= 0 && P.first[p] <= p, "%s: first[%d] = %d", g.name, p, P.first[p]);
        CHECK(P.rowoff[p + 1] - P.rowoff[p] == p - P.first[p] + 1, "%s: row %d length", g.name, p);
    }
    // the envelope bounds every nonzero block, and every edge's contributions are listed exactly once
    std::vector<int> diag_hits(4 * E, 0), off_hits(4 * E, 0);
    for (int e = 0; e < E; ++e) {
        const int a = P.pos[g.from[e]], b = P.pos[g.to[e]];
        if (a >= 0 && b >= 0) CHECK(P.first[std::max(a, b)] <= std::min(a, b), "%s: edge %d outside the envelope", g.name, e);
    }
    for (int p = 0; p < nf; ++p)
        for (int q = P.diag_ptr[p]; q < P.diag_ptr[p + 1]; ++q) {
            const int code = P.diag_code[q], e = code >> 2, k = code & 3;
            ++diag_hits[code];
            CHECK(P.pos[k == 0 ? g.from[e] : g.to[e]] == p, "%s: diagonal contribution of edge %d at the wrong block", g.name, e);
            if (q > P.diag_ptr[p]) CHECK(P.diag_code[q - 1] < code, "%s: diagonal list of %d not ascending", g.name, p);
        }
    for (size_t s = 0; s < P.off_blk.size(); ++s) {
        if (s) CHECK(P.off_blk[s - 1] < P.off_blk[s], "%s: off-diagonal blocks not in envelope order", g.name);
        for (int q = P.off_ptr[s]; q < P.off_ptr[s + 1]; ++q) {
            const int code = P.off_code[q], e = code >> 2, a = P.pos[g.from[e]], b = P.pos[g.to[e]];
            ++off_hits[code];
            CHECK(P.off_blk[s] == P.blk(std::max(a, b), std::min(a, b)), "%s: edge %d gathered into the wrong block", g.name, e);
            CHECK(((code & 3) == se2gpu::gba::kOffDiag) == (a > b), "%s: edge %d transposed wrongly", g.name, e);
            if (q > P.off_ptr[s]) CHECK(P.off_code[q - 1] < code, "%s: off-diagonal list not ascending", g.name);
        }
    }
    for (int e = 0; e < E; ++e) {
        const bool fa = P.pos[g.from[e]] >= 0, fb = P.pos[g.to[e]] >= 0;
        CHECK(diag_hits[4 * e] == (int)fa && diag_hits[4 * e + 1] == (int)fb, "%s: diagonal contributions of edge %d", g.name, e);
        CHECK(off_hits[4 * e + 2] + off_hits[4 * e + 3] == (int)(fa && fb), "%s: off-diagonal contribution of edge %d", g.name, e);
    }
    // the column lists are the transpose of the envelope
    int cnt = 0;
    for (int k = 0; k < nf; ++k)
        for (int q = P.col_ptr[k]; q < P.col_ptr[k + 1]; ++q) {
            const int i = P.col_rows[q];
            CHECK(i > k && P.first[i] <= k, "%s: column %d lists row %d", g.name, k, i);
            if (q > P.col_ptr[k]) CHECK(P.col_rows[q - 1] < i, "%s: column %d not ascending", g.name, k);
            ++cnt;
        }
    CHECK(cnt == P.env_blocks() - nf, "%s: column lists hold %d blocks, the envelope %lld", g.name, cnt, (long long)(P.env_blocks() - nf));
}

static int bandwidth(const Graph& g) {
    const Plan P = se2gpu::gba::make_plan(g.N, g.fixed.data(), (int)g.from.size(), g.from.data(), g.to.data());
    int b = 0;
    for (int p = 0; p < P.n_free; ++p) b = std::max(b, p - P.first[p]);
    return b;
}

int main() {
    std::vector<Graph> gs;
    std::mt19937 rng(7);
    auto chain = [](int N, const char* name) {
        Graph g{N, std::vector<uint8_t>(N, 0), {}, {}, name};
        g.fixed[0] = 1;
        for (int i = 0; i + 1 < N; ++i) { g.from.push_back(i); g.to.push_back(i + 1); }
        return g;
    };
    gs.push_back(chain(1, "one vertex"));
    gs.push_back(chain(10, "chain"));
    {
        Graph g = chain(300, "ring");
        g.from.push_back(299); g.to.push_back(1);
        gs.push_back(g);
    }
    {
        Graph g = chain(500, "chain with hops and loops");
        for (int i = 0; i < 500; ++i)
            for (int h = 2; h <= 5; ++h)
                if (i + h < 500) { g.from.push_back(i + h); g.to.push_back(i); }
        for (int k = 0; k < 40; ++k) { const int j = 100 + (int)(rng() % 400), i = (int)(rng() % (j - 20)); g.from.push_back(i); g.to.push_back(j); }
        gs.push_back(g);
    }
    {
        Graph g = chain(60, "duplicates, antiparallel edges, isolated and extra fixed vertices");
        for (int i = 0; i + 1 < 40; ++i) { g.from.push_back(i + 1); g.to.push_back(i); g.from.push_back(i); g.to.push_back(i + 1); }
        g.fixed[30] = 1;
        g.fixed[45] = 1;
        g.from.resize(g.from.size() - 2); g.to.resize(g.to.size() - 2);
        gs.push_back(g);
    }
    {
        Graph g{200, std::vector<uint8_t>(200, 0), {}, {}, "random"};
        g.fixed[0] = 1;
        for (int k = 0; k < 900; ++k) {
            const int a = (int)(rng() % 200), b = (int)(rng() % 200);
            if (a != b) { g.from.push_back(a); g.to.push_back(b); }
        }
        gs.push_back(g);
    }
    {
        Graph g{4, std::vector<uint8_t>(4, 1), {0, 1}, {1, 2}, "all fixed"};
        gs.push_back(g);
    }
    for (const Graph& g : gs) check(g);
    const int bw = bandwidth(gs[2]);
    CHECK(bw <= 2, "ring: bandwidth %d blocks", bw);
    if (g_fail) return 1;
    std::printf("ok\n");
    return 0;
}
