// Drives include/se2lam/localizer_ba.h the way Localizer::DoLocalBA would: one keyframe, its keypoints and the observed
// map points. Reads a problem from argv[1], writes the returned Tcw, iteration count and status to argv[2].
// Input: int n_kp, n_kp keypoints (28 B each), int E, E x (float x, y, z, int kp_index), int nlevels, nlevels floats,
// float fx, cx, cy, float Tbc[16], float delta, float Tcw[16].
#include <cstdio>
#include <vector>

#include "se2lam/localizer_ba.h"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int n_kp = 0, E = 0, nl = 0;
    rd(f, &n_kp, 1);
    std::vector<se2gpu_keypoint> kp((size_t)n_kp);
    rd(f, kp.data(), kp.size());
    rd(f, &E, 1);
    std::vector<se2gpu::PoseObservation> obs((size_t)E);
    rd(f, obs.data(), obs.size());
    rd(f, &nl, 1);
    std::vector<float> inv_sigma2((size_t)nl);
    rd(f, inv_sigma2.data(), inv_sigma2.size());
    float K[3], Tbc[16], delta, Tcw[16];
    rd(f, K, 3); rd(f, Tbc, 16); rd(f, &delta, 1);
    if (!rd(f, Tcw, 16)) return 2;
    fclose(f);
    int status = -1;
    const int iters = se2gpu::localizer_ba(Tcw, kp, n_kp ? kp[0].octave : 0, obs, inv_sigma2, K[0], K[1], K[2], Tbc, delta, &status);
    if (iters < 0) { fprintf(stderr, "localizer_ba: %d %s\n", iters, se2gpu_last_error()); return 1; }
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(Tcw, sizeof(float), 16, o);
    fwrite(&iters, sizeof(int), 1, o);
    fwrite(&status, sizeof(int), 1, o);
    fclose(o);
    return 0;
}
