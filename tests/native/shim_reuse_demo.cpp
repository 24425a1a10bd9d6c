// One SlamOptimizer kept across several local BAs, the way include/se2lam/g2o_compat.h keeps its device context while the
// capacity suffices: every window is loaded with the reference's helper calls (Map::loadLocalGraph, src/Map.cpp:891-1053),
// initializeOptimization(0), optimize(N), and read back with estimateVertexSE2 / estimateVertexSBAXYZ.
// usage: shim_reuse_demo <in.bin> <out.bin> reuse|fresh
//   reuse: one optimizer, clear() between windows; fresh: a new optimizer per window (the reference's pattern)
// in:  int nwin, then per window: P L E O iters, the arrays of tests/native/shim_demo.cpp, fx cx cy, Tbc[12], delta, and the
//      Huber delta of the last EdgeSE2XYZ (!= delta: initializeOptimization must reject the graph)
// out: per window: int initialized, int done, poses [3P], points [3L]; then the reload that adds one edge with another Huber
//      delta to the last accepted window (no clear(), like LocalMapper::removeOutlierChi2's second initializeOptimization):
//      int initialized, int done, poses, points
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "se2lam/optimizer.h"

using namespace se2lam;

template <class T> static void rd(FILE* f, T* p, size_t n) { if (fread(p, sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); } }
template <class T> static void wr(FILE* f, const T* p, size_t n) { fwrite(p, sizeof(T), n, f); }

struct Window {
    int P, L, E, O, iters;
    std::vector<double> poses, points, uv, info, om, oinf, cam, Tbc;
    std::vector<unsigned char> fixed;
    std::vector<int> ep, el, oi, oj;
    double delta, delta_last;
};

static Window read_window(FILE* fi) {
    Window w;
    rd(fi, &w.P, 1); rd(fi, &w.L, 1); rd(fi, &w.E, 1); rd(fi, &w.O, 1); rd(fi, &w.iters, 1);
    w.poses.resize(3 * w.P); w.points.resize(3 * w.L); w.uv.resize(2 * w.E); w.info.resize(3 * w.E); w.om.resize(3 * w.O);
    w.oinf.resize(6 * w.O); w.cam.resize(3); w.Tbc.resize(12); w.fixed.resize(w.P);
    w.ep.resize(w.E); w.el.resize(w.E); w.oi.resize(w.O); w.oj.resize(w.O);
    rd(fi, w.poses.data(), w.poses.size()); rd(fi, w.fixed.data(), w.fixed.size()); rd(fi, w.points.data(), w.points.size());
    rd(fi, w.ep.data(), w.ep.size()); rd(fi, w.el.data(), w.el.size()); rd(fi, w.uv.data(), w.uv.size()); rd(fi, w.info.data(), w.info.size());
    rd(fi, w.oi.data(), w.oi.size()); rd(fi, w.oj.data(), w.oj.size()); rd(fi, w.om.data(), w.om.size()); rd(fi, w.oinf.data(), w.oinf.size());
    rd(fi, w.cam.data(), 3); rd(fi, w.Tbc.data(), 12); rd(fi, &w.delta, 1); rd(fi, &w.delta_last, 1);
    return w;
}

static g2o::SE3Quat body_to_camera(const Window& w) {
    g2o::Matrix3D Rbc; g2o::Vector3D tbc;
    for (int i = 0; i < 9; ++i) Rbc.d[i] = w.Tbc[i];
    for (int i = 0; i < 3; ++i) tbc[i] = w.Tbc[9 + i];
    return g2o::SE3Quat(Rbc, tbc);
}

// Map::loadLocalGraph's calls for one window (vertex ids: poses 0..P-1, landmarks P+1..)
static CamPara* load(SlamOptimizer& optimizer, const Window& w) {
    const float K[9] = {(float)w.cam[0], 0.f, (float)w.cam[1], 0.f, (float)w.cam[0], (float)w.cam[2], 0.f, 0.f, 1.f};
    CamPara* campr = addCamPara(optimizer, K, 0);
    for (int i = 0; i < w.P; ++i) addVertexSE2(optimizer, g2o::SE2(w.poses[3 * i], w.poses[3 * i + 1], w.poses[3 * i + 2]), i, w.fixed[i] != 0);
    for (int o = 0; o < w.O; ++o) {
        g2o::Matrix3D inf;
        const double* q = &w.oinf[6 * o];
        inf(0, 0) = q[0]; inf(0, 1) = inf(1, 0) = q[1]; inf(0, 2) = inf(2, 0) = q[2]; inf(1, 1) = q[3]; inf(1, 2) = inf(2, 1) = q[4]; inf(2, 2) = q[5];
        addEdgeSE2(optimizer, g2o::makeVector3D(w.om[3 * o], w.om[3 * o + 1], w.om[3 * o + 2]), w.oi[o], w.oj[o], inf);
    }
    const int maxKFid = w.P + 1;
    const g2o::SE3Quat bTc = body_to_camera(w);
    for (int j = 0; j < w.L; ++j) addVertexSBAXYZ(optimizer, g2o::makeVector3D(w.points[3 * j], w.points[3 * j + 1], w.points[3 * j + 2]), maxKFid + j);
    for (int e = 0; e < w.E; ++e) {
        g2o::Matrix2D inf; inf(0, 0) = w.info[3 * e]; inf(0, 1) = inf(1, 0) = w.info[3 * e + 1]; inf(1, 1) = w.info[3 * e + 2];
        addEdgeSE2XYZ(optimizer, g2o::makeVector2D(w.uv[2 * e], w.uv[2 * e + 1]), w.ep[e], maxKFid + w.el[e], campr, bTc, inf,
                      e + 1 == w.E ? w.delta_last : w.delta);
    }
    return campr;
}

static void run(SlamOptimizer& optimizer, const Window& w, FILE* fo) {
    const int initialized = optimizer.initializeOptimization(0) ? 1 : 0;     // LocalMapper.cpp:259
    const int done = optimizer.optimize(w.iters);                            // LocalMapper.cpp:260
    wr(fo, &initialized, 1); wr(fo, &done, 1);
    for (int i = 0; i < w.P; ++i) { g2o::Vector3D vp = estimateVertexSE2(optimizer, i).toVector(); wr(fo, vp.d, 3); }        // Map.cpp:768
    for (int j = 0; j < w.L; ++j) { g2o::Vector3D p = estimateVertexSBAXYZ(optimizer, w.P + 1 + j); wr(fo, p.d, 3); }        // Map.cpp:777
}

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    const bool reuse = strcmp(argv[3], "reuse") == 0;
    FILE* fi = fopen(argv[1], "rb"); FILE* fo = fopen(argv[2], "wb");
    if (!fi || !fo) return 2;
    int nwin = 0;
    rd(fi, &nwin, 1);
    std::vector<Window> wins;
    for (int k = 0; k < nwin; ++k) wins.push_back(read_window(fi));

    SlamOptimizer* shared = new SlamOptimizer;
    initOptimizer(*shared);
    int last_ok = -1;
    for (int k = 0; k < nwin; ++k) {
        SlamOptimizer* opt = shared;
        if (reuse) opt->clear();
        else { opt = new SlamOptimizer; initOptimizer(*opt); }
        load(*opt, wins[k]);
        run(*opt, wins[k], fo);
        if (wins[k].delta_last == wins[k].delta) last_ok = k;
        if (!reuse) delete opt;
    }
    // the last accepted window once more, then one more edge with another Huber delta on the SAME graph (no clear()):
    // initializeOptimization rejects it, and optimize must not run the window loaded before
    SlamOptimizer* opt = reuse ? shared : new SlamOptimizer;
    if (!reuse) initOptimizer(*opt);
    if (reuse) opt->clear();
    const Window& w = wins[last_ok];
    CamPara* campr = load(*opt, w);
    opt->initializeOptimization(0);
    opt->optimize(w.iters);
    g2o::Matrix2D inf; inf(0, 0) = inf(1, 1) = 1.0;
    addEdgeSE2XYZ(*opt, g2o::makeVector2D(w.uv[0], w.uv[1]), w.ep[0], w.P + 1 + w.el[0], campr, body_to_camera(w), inf, 2 * w.delta + 1);
    run(*opt, w, fo);
    if (!reuse) delete opt;
    delete shared;
    fclose(fi); fclose(fo);
    return 0;
}
