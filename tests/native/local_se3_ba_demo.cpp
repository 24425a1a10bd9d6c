// Drives include/se2lam/local_se3_ba.h the way LocalMapper::removeOutlierChi2 would.
// "lists": reads int L, int E, E x (int point, int kf, byte outlier) from argv[2] and writes the vnOutlierIdxAll lists to
// argv[3] as int L, then per point int n and its n keyframes (no device needed).
// "run": reads a window from argv[2] (int N, O, L, E; Tcw, fixed, prior, odo_from, odo_to, odo_measure, odo_info, xyz,
// edge_point, edge_kf, uv, inv_sigma2; then the se2gpu_se3_ba_params bytes) and writes int rc, status, iterations, double
// chi2[E], byte outlier[E] and the lists as above to argv[3].
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "se2lam/local_se3_ba.h"

template <class T>
static bool rd(FILE* f, std::vector<T>& v, size_t n) { v.resize(n); return n == 0 || fread(v.data(), sizeof(T), n, f) == n; }
template <class T>
static bool rd1(FILE* f, T* p) { return fread(p, sizeof(T), 1, f) == 1; }

static void write_lists(FILE* g, const std::vector<std::vector<int>>& lists) {
    const int L = (int)lists.size();
    fwrite(&L, 4, 1, g);
    for (const auto& l : lists) {
        const int n = (int)l.size();
        fwrite(&n, 4, 1, g);
        if (n) fwrite(l.data(), 4, (size_t)n, g);
    }
}

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    const std::string mode = argv[1];
    FILE* f = fopen(argv[2], "rb");
    FILE* g = fopen(argv[3], "wb");
    if (!f || !g) return 2;
    if (mode == "lists") {
        int L = 0, E = 0;
        if (!rd1(f, &L) || !rd1(f, &E)) return 2;
        std::vector<int> pt((size_t)E), kf((size_t)E);
        std::vector<unsigned char> out((size_t)E);
        for (int e = 0; e < E; ++e)
            if (!rd1(f, &pt[(size_t)e]) || !rd1(f, &kf[(size_t)e]) || !rd1(f, &out[(size_t)e])) return 2;
        write_lists(g, se2gpu::se3_outlier_lists(L, pt, kf, out));
        return 0;
    }
    int N, O, L, E;
    if (!rd1(f, &N) || !rd1(f, &O) || !rd1(f, &L) || !rd1(f, &E)) return 2;
    se2gpu::LocalSE3Window w;
    if (!rd(f, w.Tcw, 16 * (size_t)N) || !rd(f, w.fixed, N) || !rd(f, w.prior, N) || !rd(f, w.odo_from, O) || !rd(f, w.odo_to, O) ||
        !rd(f, w.odo_measure, 16 * (size_t)O) || !rd(f, w.odo_info, 36 * (size_t)O) || !rd(f, w.xyz, 3 * (size_t)L) ||
        !rd(f, w.edge_point, E) || !rd(f, w.edge_kf, E) || !rd(f, w.uv, 2 * (size_t)E) || !rd(f, w.inv_sigma2, E))
        return 2;
    se2gpu_se3_ba_params prm;
    if (!rd1(f, &prm)) return 2;
    se2gpu::LocalSE3BAContext ctx;
    se2gpu::LocalSE3Result r;
    const int rc = ctx.run(w, prm, &r);
    fwrite(&rc, 4, 1, g); fwrite(&r.status, 4, 1, g); fwrite(&r.iterations, 4, 1, g);
    if (E) { fwrite(r.chi2.data(), 8, (size_t)E, g); fwrite(r.outlier.data(), 1, (size_t)E, g); }
    write_lists(g, r.outlier_kfs);
    return rc ? 1 : 0;
}
