// Header-only forwarder of Localizer::DoLocalBA (reference src/Localizer.cpp:233-302) to se2gpu_pose_ba: takes what
// DoLocalBA has at hand - the keyframe pose, its keypoints, the (map point position, keypoint index) pair of every
// observed map point that is !isNull() && isGoodPrl(), mvInvLevelSigma2, K, Tbc and the Huber delta - and returns the
// float Tcw that DoLocalBA writes back with setPose. INTEGRATION.md section 7 shows the replaced body.
#pragma once

#include <cstring>
#include <vector>

#include "../se2gpu.h"

namespace se2gpu {

struct PoseObservation {
    float x, y, z;  // MapPoint::getPos()
    int kp_index;   // KeyFrame::getObservations()[pMP]
};

// Tcw [16] row-major in/out. uv of observation i is keyPointsUn[obs[i].kp_index].pt; every edge's information is
// invLevelSigma2[octave0] with octave0 = keyPoints[0].octave (what MapPoint::getOctave returns for the Localizer's new
// keyframe). Returns the number of LM iterations done (>= 0) or a negative se2gpu error; *status (may be NULL) receives
// SE2GPU_POSE_BA_*.
inline int localizer_ba(float* Tcw, const std::vector<se2gpu_keypoint>& keyPointsUn, int octave0, const std::vector<PoseObservation>& obs,
                        const std::vector<float>& invLevelSigma2, float fx, float cx, float cy, const float* Tbc, float huber_delta,
                        int* status = nullptr, float xrot_info = 1e6f, float yrot_info = 1e6f, float z_info = 1.f, int iterations = 30,
                        int device = 0) {
    const int E = (int)obs.size();
    if (octave0 < 0 || octave0 >= (int)invLevelSigma2.size()) return SE2GPU_ERR_INVALID;
    std::vector<float> xyz(3 * (size_t)E), uv(2 * (size_t)E), info((size_t)E, invLevelSigma2[(size_t)octave0]);
    for (int e = 0; e < E; ++e) {
        const PoseObservation& o = obs[(size_t)e];
        if (o.kp_index < 0 || o.kp_index >= (int)keyPointsUn.size()) return SE2GPU_ERR_INVALID;
        xyz[3 * (size_t)e] = o.x; xyz[3 * (size_t)e + 1] = o.y; xyz[3 * (size_t)e + 2] = o.z;
        uv[2 * (size_t)e] = keyPointsUn[(size_t)o.kp_index].x; uv[2 * (size_t)e + 1] = keyPointsUn[(size_t)o.kp_index].y;
    }
    se2gpu_pose_ba_params p;
    p.fx = fx; p.cx = cx; p.cy = cy;
    std::memcpy(p.Tbc, Tbc, sizeof p.Tbc);
    p.huber_delta = huber_delta;
    p.xrot_info = xrot_info; p.yrot_info = yrot_info; p.z_info = z_info;
    p.iterations = iterations;
    const int edge_ptr[2] = {0, E};
    int iters = 0, st = 0;
    const int rc = se2gpu_pose_ba(1, Tcw, edge_ptr, E ? xyz.data() : nullptr, E ? uv.data() : nullptr, E ? info.data() : nullptr, &p,
                                  nullptr, &iters, &st, nullptr, device);
    if (rc < 0) return rc;
    if (status) *status = st;
    return iters;
}

}  // namespace se2gpu
