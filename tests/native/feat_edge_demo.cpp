// Drives include/se2lam/feat_edge.h the way GlobalMapper::CreateFeatEdge and Map::UpdateFeatGraph would. Reads a batch of
// keyframe pairs from argv[1] and writes every pair's result to argv[2]; the first pair also goes through the cv::Mat
// form and must give the same constraint.
// Input: int matched, int B, float Tbc[16], then per pair float Tcw0[16], Tcw1[16], int P, P x (float pos[3], z0[3], z1[3],
// double info0[9], info1[9]). Output per pair: int ret, status, iterations, float measure[16], info[36], P outlier bytes.
#include <cstdio>
#include <cstring>
#include <vector>

#include "se2lam/cv_compat.h"
#include "se2lam/feat_edge.h"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int matched = 0, B = 0;
    float Tbc[16];
    if (!rd(f, &matched, 1) || !rd(f, &B, 1) || !rd(f, Tbc, 16)) return 2;
    std::vector<se2gpu::FeatEdgePair> pairs((size_t)B);
    for (auto& pr : pairs) {
        int P = 0;
        if (!rd(f, pr.Tcw0, 16) || !rd(f, pr.Tcw1, 16) || !rd(f, &P, 1)) return 2;
        pr.points.resize((size_t)P);
        for (auto& q : pr.points)
            if (!rd(f, q.pos, 3) || !rd(f, q.z0, 3) || !rd(f, q.z1, 3) || !rd(f, q.info0, 9) || !rd(f, q.info1, 9)) return 2;
    }
    fclose(f);
    const se2gpu_feat_edge_params prm = se2gpu::feat_edge_params(Tbc, 1e6f, 1e6f, 1.f);
    std::vector<se2gpu::FeatEdgeResult> out;
    const int rc = se2gpu::create_feat_edges(pairs, matched != 0, prm, &out);
    if (rc < 0) { fprintf(stderr, "create_feat_edges: %d %s\n", rc, se2gpu_last_error()); return 1; }
    if (B) {
        cv::Mat measure, info;
        const int ret = se2gpu::CreateFeatEdge(pairs[0], matched != 0, prm, &measure, &info);
        if (ret != out[0].ret) { fprintf(stderr, "single pair returned %d, the batch %d\n", ret, out[0].ret); return 1; }
        if (ret == 0 && (std::memcmp(&measure.at<float>(0, 0), out[0].measure, sizeof out[0].measure) ||
                         std::memcmp(&info.at<float>(0, 0), out[0].info, sizeof out[0].info))) {
            fprintf(stderr, "single pair and batch differ\n");
            return 1;
        }
    }
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    for (const auto& r : out) {
        fwrite(&r.ret, sizeof(int), 1, o);
        fwrite(&r.status, sizeof(int), 1, o);
        fwrite(&r.iterations, sizeof(int), 1, o);
        fwrite(r.measure, sizeof(float), 16, o);
        fwrite(r.info, sizeof(float), 36, o);
        fwrite(r.outlier.data(), 1, r.outlier.size(), o);
    }
    fclose(o);
    return 0;
}
