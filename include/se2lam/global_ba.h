// Header-only forwarder of GlobalMapper::GlobalBA (reference src/GlobalMapper.cpp:328-535) to se2gpu_global_ba and its
// map-point write-back to se2gpu_global_ba_update_points. The caller flattens what the reference walks: the non-null
// keyframes (index = position in the list, fixed = mIdKF == 0), the odometry constraint of each keyframe and its
// mFtrMeasureFrom entries whose target is in the list, and for each non-null map point observed by its main keyframe that
// keyframe's index and mViewMPs[idx]. INTEGRATION.md section 9 shows the replaced body. cv::Mat is the project's own
// (OpenCV, or cv_compat.h in the tests).
#pragma once

#include <cstring>
#include <vector>

#include "../se2gpu.h"

namespace se2gpu {

// one EdgeSE3 (addEdgeSE3): an odometry or a feature constraint from keyframe `from` to keyframe `to`
struct GlobalBAEdge {
    int from, to;
    float measure[16];  // SE3Constraint::measure, row-major 4 x 4
    float info[36];     // SE3Constraint::info, row-major 6 x 6
};

struct GlobalBAResult {
    int status = 0, iterations = 0;  // SE2GPU_GLOBAL_BA_*, LM iterations done
    std::vector<float> Tcw;          // [N*16] the pose each keyframe's setPose receives
};

inline se2gpu_global_ba_params global_ba_params(const float* Tbc, float xrot_info, float yrot_info, float z_info, int iterations) {
    se2gpu_global_ba_params p = SE2GPU_GLOBAL_BA_PARAMS_INIT;
    std::memcpy(p.Tbc, Tbc, sizeof p.Tbc);
    p.xrot_info = xrot_info; p.yrot_info = yrot_info; p.z_info = z_info; p.iterations = iterations;
    return p;
}

// The solver context of GlobalMapper: its device buffers grow to the largest map seen, so keep one for the mapper's life.
class GlobalBAContext {
  public:
    explicit GlobalBAContext(int device = 0) : h_(se2gpu_global_ba_create(device)), device_(device) {}
    ~GlobalBAContext() { se2gpu_global_ba_destroy(h_); }
    GlobalBAContext(const GlobalBAContext&) = delete;
    GlobalBAContext& operator=(const GlobalBAContext&) = delete;
    bool ok() const { return h_ != nullptr; }
    int device() const { return device_; }

    // GlobalBA's graph and optimize(params.iterations): Tcw [N*16] (KeyFrame::Tcw, row-major), fixed [N]. Returns 0 or a
    // negative se2gpu error.
    int GlobalBA(const std::vector<float>& Tcw, const std::vector<unsigned char>& fixed, const std::vector<GlobalBAEdge>& edges,
                 const se2gpu_global_ba_params& prm, GlobalBAResult* out) {
        if (!h_) return SE2GPU_ERR_NO_DEVICE;
        const int N = (int)fixed.size(), E = (int)edges.size();
        if (Tcw.size() != 16 * (size_t)N) return SE2GPU_ERR_INVALID;
        std::vector<int> from((size_t)E), to((size_t)E);
        std::vector<float> measure(16 * (size_t)E), info(36 * (size_t)E);
        for (int e = 0; e < E; ++e) {
            from[(size_t)e] = edges[(size_t)e].from;
            to[(size_t)e] = edges[(size_t)e].to;
            std::memcpy(&measure[16 * (size_t)e], edges[(size_t)e].measure, sizeof edges[(size_t)e].measure);
            std::memcpy(&info[36 * (size_t)e], edges[(size_t)e].info, sizeof edges[(size_t)e].info);
        }
        out->Tcw.assign(16 * (size_t)N, 0.f);
        return se2gpu_global_ba(h_, N, Tcw.data(), fixed.data(), E, from.data(), to.data(), measure.data(), info.data(), &prm,
                                out->Tcw.data(), &out->status, &out->iterations, nullptr, nullptr);
    }

  private:
    se2gpu_global_ba_ctx* h_;
    int device_;
};

// keyframe k's new pose as a 4 x 4 CV_32F matrix, for KeyFrame::setPose
template <class Mat>
inline Mat global_ba_pose(const GlobalBAResult& r, int k) {
    Mat T(4, 4, CV_32FC1);
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) T.template at<float>(i, j) = r.Tcw[16 * (size_t)k + (size_t)(i * 4 + j)];
    return T;
}

// GlobalBA's map-point write-back: kf [M] the main keyframe's index, view [M*3] its mViewMPs[idx], Tcw [N*16] the new poses;
// pos [M*3] receives MapPoint::setPos. Returns 0 or a negative se2gpu error.
inline int update_map_points(const std::vector<int>& kf, const std::vector<float>& view, const std::vector<float>& Tcw,
                             std::vector<float>* pos, int device = 0) {
    const int M = (int)kf.size();
    if (view.size() != 3 * (size_t)M || Tcw.size() % 16) return SE2GPU_ERR_INVALID;
    pos->assign(3 * (size_t)M, 0.f);
    return se2gpu_global_ba_update_points(M, kf.data(), view.data(), (int)(Tcw.size() / 16), Tcw.data(), pos->data(), device);
}

}  // namespace se2gpu
