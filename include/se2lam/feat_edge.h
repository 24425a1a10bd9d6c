// Header-only forwarder of GlobalMapper::CreateFeatEdge (reference src/GlobalMapper.cpp:737-843, both overloads) and of
// the loop of Map::UpdateFeatGraph (src/Map.cpp:857-889) to se2gpu_feat_edge. The caller flattens what the reference reads
// through compareViewMPs / getFtrIdx (first overload) or mapMatch (second overload): per co-observed point its world
// position and, for each of the two keyframes, mViewMPs[idx] and mViewMPsInfo[idx]. INTEGRATION.md section 8 shows the
// replaced bodies. cv::Mat is the project's own (OpenCV, or cv_compat.h in the tests).
#pragma once

#include <cstring>
#include <vector>

#include "../se2gpu.h"

namespace se2gpu {

// one co-observed map point (first overload) or one match whose two map points exist (second overload)
struct FeatEdgePoint {
    float pos[3];      // MapPoint::getPos(); for a match, of the point seen in the first keyframe
    float z0[3];       // pKFFrom->mViewMPs[idx0]
    float z1[3];       // pKFTo->mViewMPs[idx1]
    double info0[9];   // pKFFrom->mViewMPsInfo[idx0], row-major
    double info1[9];   // pKFTo->mViewMPsInfo[idx1]
};

struct FeatEdgePair {
    float Tcw0[16], Tcw1[16];            // KeyFrame::getPose() of from / to, row-major
    std::vector<FeatEdgePoint> points;
};

struct FeatEdgeResult {
    int ret;                             // what CreateFeatEdge returns: 0, or 1 for too few points (measure / info untouched)
    int status, iterations;              // SE2GPU_FEAT_EDGE_*, LM iterations done
    float measure[16], info[36];         // SE3Constraint::measure (4 x 4) and ::info (6 x 6), row-major
    std::vector<unsigned char> outlier;  // second overload: sIdMPin1Outlier as one byte per match
};

inline se2gpu_feat_edge_params feat_edge_params(const float* Tbc, float xrot_info, float yrot_info, float z_info) {
    se2gpu_feat_edge_params p = SE2GPU_FEAT_EDGE_PARAMS_INIT;
    std::memcpy(p.Tbc, Tbc, sizeof p.Tbc);
    p.xrot_info = xrot_info; p.yrot_info = yrot_info; p.z_info = z_info;
    return p;
}

// All pairs of one keyframe (Map::UpdateFeatGraph) or a batch of verified loops in one launch. matched = false is
// CreateFeatEdge(from, to, cnstr), matched = true is CreateFeatEdge(from, to, mapMatch, cnstr). Returns 0 or a negative
// se2gpu error; out[b] belongs to pairs[b].
inline int create_feat_edges(const std::vector<FeatEdgePair>& pairs, bool matched, const se2gpu_feat_edge_params& prm,
                             std::vector<FeatEdgeResult>* out, int device = 0) {
    const int B = (int)pairs.size();
    std::vector<int> ptr((size_t)B + 1, 0);
    for (int b = 0; b < B; ++b) ptr[(size_t)b + 1] = ptr[(size_t)b] + (int)pairs[(size_t)b].points.size();
    const size_t P = (size_t)ptr[(size_t)B];
    std::vector<float> T0(16 * (size_t)B), T1(16 * (size_t)B), xyz(3 * P), z0(3 * P), z1(3 * P), measure(16 * (size_t)B), info(36 * (size_t)B);
    std::vector<double> i0(9 * P), i1(9 * P);
    std::vector<int> status((size_t)B), iters((size_t)B);
    std::vector<unsigned char> outlier(P ? P : 1);
    size_t j = 0;
    for (int b = 0; b < B; ++b) {
        std::memcpy(&T0[16 * (size_t)b], pairs[(size_t)b].Tcw0, 16 * sizeof(float));
        std::memcpy(&T1[16 * (size_t)b], pairs[(size_t)b].Tcw1, 16 * sizeof(float));
        for (const FeatEdgePoint& q : pairs[(size_t)b].points) {
            std::memcpy(&xyz[3 * j], q.pos, sizeof q.pos);
            std::memcpy(&z0[3 * j], q.z0, sizeof q.z0);
            std::memcpy(&z1[3 * j], q.z1, sizeof q.z1);
            std::memcpy(&i0[9 * j], q.info0, sizeof q.info0);
            std::memcpy(&i1[9 * j], q.info1, sizeof q.info1);
            ++j;
        }
    }
    out->assign((size_t)B, FeatEdgeResult());
    if (B == 0) return SE2GPU_OK;
    const int rc = se2gpu_feat_edge(B, matched ? 1 : 0, T0.data(), T1.data(), ptr.data(), xyz.data(), z0.data(), z1.data(), i0.data(),
                                    i1.data(), &prm, measure.data(), info.data(), status.data(), iters.data(), nullptr, outlier.data(),
                                    nullptr, nullptr, device);
    if (rc < 0) return rc;
    for (int b = 0; b < B; ++b) {
        FeatEdgeResult& r = (*out)[(size_t)b];
        r.status = status[(size_t)b]; r.iterations = iters[(size_t)b];
        r.ret = r.status == SE2GPU_FEAT_EDGE_TOO_FEW ? 1 : 0;
        std::memcpy(r.measure, &measure[16 * (size_t)b], sizeof r.measure);
        std::memcpy(r.info, &info[36 * (size_t)b], sizeof r.info);
        r.outlier.assign(outlier.begin() + ptr[(size_t)b], outlier.begin() + ptr[(size_t)b + 1]);
    }
    return SE2GPU_OK;
}

// One pair, with the reference's return value; measure (4 x 4 CV_32F) and info (6 x 6 CV_32F) are written only when it
// returns 0, as SE3CnstrOutput is. A negative return is a se2gpu error.
template <class Mat>
inline int CreateFeatEdge(const FeatEdgePair& pair, bool matched, const se2gpu_feat_edge_params& prm, Mat* measure, Mat* info,
                          std::vector<unsigned char>* outlier = nullptr, int device = 0) {
    std::vector<FeatEdgeResult> out;
    const int rc = create_feat_edges(std::vector<FeatEdgePair>(1, pair), matched, prm, &out, device);
    if (rc < 0) return rc;
    if (outlier) *outlier = out[0].outlier;
    if (out[0].ret) return out[0].ret;
    *measure = Mat(4, 4, CV_32FC1);
    *info = Mat(6, 6, CV_32FC1);
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) measure->template at<float>(r, c) = out[0].measure[r * 4 + c];
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) info->template at<float>(r, c) = out[0].info[r * 6 + c];
    return 0;
}

}  // namespace se2gpu
