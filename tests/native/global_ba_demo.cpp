// Drives include/se2lam/global_ba.h the way GlobalMapper::GlobalBA would. Reads a graph and map points from argv[1], runs
// GlobalBA twice on one context (the second run must give the same bytes), checks the cv::Mat form of every pose, and
// writes the results to argv[2].
// Input: int N, float Tbc[16], N x float Tcw[16], N fixed bytes, int E, E x (int from, to, float measure[16], info[36]),
// int M, M x (int kf, float view[3]). Output: int status, iterations, float Tcw[N*16], float pos[M*3].
#include <cstdio>
#include <cstring>
#include <vector>

#include "se2lam/cv_compat.h"
#include "se2lam/global_ba.h"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int N = 0, E = 0, M = 0;
    float Tbc[16];
    if (!rd(f, &N, 1) || !rd(f, Tbc, 16)) return 2;
    std::vector<float> Tcw(16 * (size_t)N);
    std::vector<unsigned char> fixed((size_t)N);
    if (!rd(f, Tcw.data(), Tcw.size()) || !rd(f, fixed.data(), fixed.size()) || !rd(f, &E, 1)) return 2;
    std::vector<se2gpu::GlobalBAEdge> edges((size_t)E);
    for (auto& e : edges)
        if (!rd(f, &e.from, 1) || !rd(f, &e.to, 1) || !rd(f, e.measure, 16) || !rd(f, e.info, 36)) return 2;
    if (!rd(f, &M, 1)) return 2;
    std::vector<int> kf((size_t)M);
    std::vector<float> view(3 * (size_t)M);
    for (int m = 0; m < M; ++m)
        if (!rd(f, &kf[(size_t)m], 1) || !rd(f, &view[3 * (size_t)m], 3)) return 2;
    fclose(f);
    const se2gpu_global_ba_params prm = se2gpu::global_ba_params(Tbc, 1e6f, 1e6f, 1.f, 15);
    se2gpu::GlobalBAContext ctx(0);
    if (!ctx.ok()) { fprintf(stderr, "se2gpu_global_ba_create: %s\n", se2gpu_last_error()); return 1; }
    se2gpu::GlobalBAResult r, again;
    int rc = ctx.GlobalBA(Tcw, fixed, edges, prm, &r);
    if (rc < 0) { fprintf(stderr, "GlobalBA: %d %s\n", rc, se2gpu_last_error()); return 1; }
    rc = ctx.GlobalBA(Tcw, fixed, edges, prm, &again);
    if (rc < 0 || again.status != r.status || again.iterations != r.iterations || again.Tcw != r.Tcw) {
        fprintf(stderr, "a second run on the same context differs\n");
        return 1;
    }
    for (int k = 0; k < N; ++k) {
        const cv::Mat T = se2gpu::global_ba_pose<cv::Mat>(r, k);
        if (std::memcmp(&T.at<float>(0, 0), &r.Tcw[16 * (size_t)k], 16 * sizeof(float))) { fprintf(stderr, "pose %d differs\n", k); return 1; }
    }
    std::vector<float> pos;
    rc = se2gpu::update_map_points(kf, view, r.Tcw, &pos);
    if (rc < 0) { fprintf(stderr, "update_map_points: %d %s\n", rc, se2gpu_last_error()); return 1; }
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(&r.status, sizeof(int), 1, o);
    fwrite(&r.iterations, sizeof(int), 1, o);
    fwrite(r.Tcw.data(), sizeof(float), r.Tcw.size(), o);
    fwrite(pos.data(), sizeof(float), pos.size(), o);
    fclose(o);
    return 0;
}
