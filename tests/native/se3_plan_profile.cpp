// The shape of the SE(3)-XYZ window BA's reduced system (se2lam_b200/csrc/se3_ba.cu), from the block graph its make_plan
// passes to global_ba_plan.h: odometry links first, then the co-observation pairs of free keyframes. Reads on stdin
//   N O M, then N fixed flags (nonzero: fixed or not in the graph), then M links "from to" (the first O are odometry),
// and prints "nf max_column_rows off_diag off_diag_t components": the number of free keyframes, the most rows any envelope
// column holds below its pivot, how many odometry contributions env_factor's caller gathers as H_ij (kOffDiag) and as
// H_ij^T (kOffDiagT), and the number of connected components of the free keyframes' block graph.
#include <cstdio>
#include <numeric>
#include <vector>

#include "../../se2lam_b200/csrc/global_ba_plan.h"

namespace gba = se2gpu::gba;

static int root(std::vector<int>& p, int v) {
    while (p[v] != v) v = p[v] = p[p[v]];
    return v;
}

int main() {
    int N = 0, O = 0, M = 0;
    if (std::scanf("%d %d %d", &N, &O, &M) != 3 || N < 0 || O < 0 || M < O) return 2;
    std::vector<uint8_t> fixed(N);
    for (int v = 0; v < N; ++v) {
        int f = 0;
        if (std::scanf("%d", &f) != 1) return 2;
        fixed[v] = f ? 1 : 0;
    }
    std::vector<int> from(M), to(M);
    for (int e = 0; e < M; ++e)
        if (std::scanf("%d %d", &from[e], &to[e]) != 2 || from[e] < 0 || from[e] >= N || to[e] < 0 || to[e] >= N) return 2;
    const gba::Plan P = gba::make_plan(N, fixed.data(), M, from.data(), to.data());
    int max_rows = 0;
    for (int k = 0; k < P.n_free; ++k) max_rows = std::max(max_rows, P.col_ptr[k + 1] - P.col_ptr[k]);
    long long off = 0, off_t = 0;
    for (int c : P.off_code)
        if ((c >> 2) < O) ((c & 3) == gba::kOffDiag ? off : off_t) += 1;
    std::vector<int> parent(N);
    std::iota(parent.begin(), parent.end(), 0);
    for (int e = 0; e < M; ++e)
        if (P.pos[from[e]] >= 0 && P.pos[to[e]] >= 0) parent[root(parent, from[e])] = root(parent, to[e]);
    int comps = 0;
    for (int v = 0; v < N; ++v) comps += P.pos[v] >= 0 && root(parent, v) == v;
    std::printf("%d %d %lld %lld %d\n", P.n_free, max_rows, off, off_t, comps);
    return 0;
}
