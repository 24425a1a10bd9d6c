// The shape of the SE(3)-XYZ window BA's reduced system, from the plan se2lam_b200/csrc/se3_ba_plan.h builds for the
// kernel. Reads on stdin
//   N O L E, then N fixed flags, N prior flags, O odometry links "from to" and E projection edges "point keyframe",
// and prints "nf max_column_rows off_diag off_diag_t components": the number of free keyframes, the most rows any envelope
// column holds below its pivot, how many odometry contributions the off-diagonal gather reads as H_ij (kOffDiag) and as
// H_ij^T (kOffDiagT), and the number of connected components of the free keyframes' block graph (odometry and
// co-observation).
#include <cstdio>
#include <numeric>
#include <vector>

#include "../../se2lam_b200/csrc/se3_ba_plan.h"

namespace gba = se2gpu::gba;

static int root(std::vector<int>& p, int v) {
    while (p[v] != v) v = p[v] = p[p[v]];
    return v;
}

// n values, or n pairs (a, b) with a < na and b < nb
static bool read(int n, std::vector<int>& a, int na, std::vector<int>* b = nullptr, int nb = 0) {
    a.resize(n);
    if (b) b->resize(n);
    for (int i = 0; i < n; ++i)
        if (std::scanf("%d", &a[i]) != 1 || a[i] < 0 || a[i] >= na || (b && (std::scanf("%d", &(*b)[i]) != 1 || (*b)[i] < 0 || (*b)[i] >= nb)))
            return false;
    return true;
}

int main() {
    int N = 0, O = 0, L = 0, E = 0;
    if (std::scanf("%d %d %d %d", &N, &O, &L, &E) != 4 || N < 0 || O < 0 || L < 0 || E < 0) return 2;
    std::vector<int> fixed, prior, from, to, e_pt, e_kf;
    if (!read(N, fixed, 2) || !read(N, prior, 2) || !read(O, from, N, &to, N) || !read(E, e_pt, L, &e_kf, N)) return 2;
    const std::vector<uint8_t> fx(fixed.begin(), fixed.end()), pr(prior.begin(), prior.end());
    const se2gpu::se3ba::Plan P = se2gpu::se3ba::make_plan(N, fx.data(), pr.data(), O, from.data(), to.data(), L, E, e_pt.data(), e_kf.data());
    const gba::Plan& G = P.G;
    int max_rows = 0;
    for (int k = 0; k < G.n_free; ++k) max_rows = std::max(max_rows, G.col_ptr[k + 1] - G.col_ptr[k]);
    long long off = 0, off_t = 0;
    for (int c : P.off_code) ((c & 3) == gba::kOffDiag ? off : off_t) += 1;
    // components: the odometry between free keyframes, and every Schur pair (two edges of one point to free keyframes)
    std::vector<int> parent(N);
    std::iota(parent.begin(), parent.end(), 0);
    for (int o = 0; o < O; ++o)
        if (G.pos[from[o]] >= 0 && G.pos[to[o]] >= 0) parent[root(parent, from[o])] = root(parent, to[o]);
    for (size_t q = 0; q < P.pair_a.size(); ++q) parent[root(parent, e_kf[P.pair_a[q]])] = root(parent, e_kf[P.pair_b[q]]);
    int comps = 0;
    for (int v = 0; v < N; ++v) comps += G.pos[v] >= 0 && root(parent, v) == v;
    std::printf("%d %d %lld %lld %d\n", G.n_free, max_rows, off, off_t, comps);
    return 0;
}
