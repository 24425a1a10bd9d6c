// Header-only forwarder of the SE(3)-XYZ window BA to se2gpu_se3_ba: the graph Map::loadLocalGraph (reference
// src/Map.cpp:414-566) or Map::loadLocalGraphOnlyBa (:568-698) builds, optimize(iterations), and the per-edge chi2 cut of
// LocalMapper::removeOutlierChi2 (src/LocalMapper.cpp:172-230). The caller flattens what the loaders walk: the local
// keyframes then the reference keyframes (index = vertex id), each local keyframe's odometry link into the window, and
// for every local map point with isGoodPrl() its observations in the window. The result's outlier lists have the shape of
// removeOutlierChi2's vnOutlierIdxAll, ready for Map::removeLocalOutlierMP. INTEGRATION.md section 10 shows the replaced
// bodies.
#pragma once

#include <vector>

#include "../se2gpu.h"

namespace se2gpu {

struct LocalSE3Window {
    std::vector<float> Tcw;                  // [N*16] KeyFrame::getPose(), row-major
    std::vector<unsigned char> fixed, prior; // [N] fixed vertex; has addPlaneMotionSE3Expmap's prior (loadLocalGraph only)
    std::vector<int> odo_from, odo_to;       // [O] mOdoMeasureFrom: vertex of the source keyframe, vertex of the keyframe
    std::vector<float> odo_measure, odo_info; // [O*16] measure, [O*36] info in KeyFrame's [trans rot] order
    std::vector<float> xyz;                  // [L*3] MapPoint::getPos()
    std::vector<int> edge_point, edge_kf;    // [E] point index, keyframe vertex
    std::vector<float> uv, inv_sigma2;       // [E*2] keyPointsUn[ftrIdx].pt, [E] mvInvLevelSigma2[octave]
};

struct LocalSE3Result {
    int status = 0, iterations = 0;          // SE2GPU_SE3_BA_*, LM iterations done
    std::vector<double> chi2;                // [E] each edge's raw chi2 at the final estimate
    std::vector<unsigned char> outlier;      // [E] chi2 > params.chi2_cut
    std::vector<std::vector<int>> outlier_kfs;  // [L] vnOutlierIdxAll: per point, the keyframe vertices of its outlier edges
};

// removeOutlierChi2's vnOutlierIdxAll from the per-edge flags: edges keep their order within each point
inline std::vector<std::vector<int>> se3_outlier_lists(int L, const std::vector<int>& edge_point, const std::vector<int>& edge_kf,
                                                       const std::vector<unsigned char>& outlier) {
    std::vector<std::vector<int>> lists((size_t)L);
    for (size_t e = 0; e < outlier.size(); ++e)
        if (outlier[e]) lists[(size_t)edge_point[e]].push_back(edge_kf[e]);
    return lists;
}

// The context of LocalMapper: its device buffers grow to the largest window seen, so keep one for the mapper's life.
class LocalSE3BAContext {
  public:
    explicit LocalSE3BAContext(int device = 0) : h_(se2gpu_se3_ba_create(device)) {}
    ~LocalSE3BAContext() { se2gpu_se3_ba_destroy(h_); }
    LocalSE3BAContext(const LocalSE3BAContext&) = delete;
    LocalSE3BAContext& operator=(const LocalSE3BAContext&) = delete;
    bool ok() const { return h_ != nullptr; }

    // optimize(prm.iterations) on the window and the outlier cut. Returns 0 or a negative se2gpu error.
    int run(const LocalSE3Window& w, const se2gpu_se3_ba_params& prm, LocalSE3Result* out) {
        if (!h_) return SE2GPU_ERR_NO_DEVICE;
        const int N = (int)w.fixed.size(), O = (int)w.odo_from.size(), L = (int)(w.xyz.size() / 3), E = (int)w.edge_point.size();
        if (w.Tcw.size() != 16 * (size_t)N || w.prior.size() != (size_t)N || w.odo_to.size() != (size_t)O ||
            w.odo_measure.size() != 16 * (size_t)O || w.odo_info.size() != 36 * (size_t)O || w.xyz.size() != 3 * (size_t)L ||
            w.edge_kf.size() != (size_t)E || w.uv.size() != 2 * (size_t)E || w.inv_sigma2.size() != (size_t)E)
            return SE2GPU_ERR_INVALID;
        out->chi2.assign((size_t)E, 0.0);
        out->outlier.assign((size_t)E, 0);
        const int rc = se2gpu_se3_ba(h_, N, w.Tcw.data(), w.fixed.data(), w.prior.data(), O, w.odo_from.data(), w.odo_to.data(),
                                     w.odo_measure.data(), w.odo_info.data(), L, w.xyz.data(), E, w.edge_point.data(),
                                     w.edge_kf.data(), w.uv.data(), w.inv_sigma2.data(), &prm, out->chi2.data(),
                                     out->outlier.data(), &out->status, &out->iterations, nullptr, nullptr, nullptr, nullptr,
                                     nullptr);
        if (rc) return rc;
        out->outlier_kfs = se3_outlier_lists(L, w.edge_point, w.edge_kf, out->outlier);
        return 0;
    }

  private:
    se2gpu_se3_ba_ctx* h_;
};

}  // namespace se2gpu
