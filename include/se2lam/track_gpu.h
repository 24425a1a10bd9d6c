// Header-only forwarder of se2gpu_tracker_* (include/se2gpu.h) shaped like Track::mTrack's body (reference
// src/Track.cpp:124-160): one call runs the extraction, MatchByWindow, removeOutliers, updateFramePose, doTriangulate and
// needNewKF of one frame (or of B frames of B streams) with the state on the device; the caller keeps KeyFrame creation,
// LocalMapper::addNewKF and setAbortBA. INTEGRATION.md section 12 shows Track.cpp driving it.
#pragma once
#include <stdexcept>
#include <string>
#include <vector>

#include "../se2gpu.h"

namespace se2lam {
namespace gpu {

class TrackGpu {
  public:
    TrackGpu(int max_streams, int max_w, int max_h, const se2gpu_tracker_params& p, int device = 0)
        : h_(se2gpu_tracker_create(max_streams, max_w, max_h, &p, device)) {
        if (!h_) throw std::runtime_error(std::string("se2gpu_tracker_create: ") + se2gpu_last_error());
    }
    ~TrackGpu() { se2gpu_tracker_destroy(h_); }
    TrackGpu(const TrackGpu&) = delete;
    TrackGpu& operator=(const TrackGpu&) = delete;

    // mCreateFrame for streams 0 .. B-1: out[b].new_kf = the frame has more than 100 keypoints
    void first(int B, const uint8_t* frames, bool on_device, int w, int h, int stride, const float* odom, se2gpu_track_result* out) {
        check(se2gpu_tracker_first(h_, B, frames, on_device, w, h, stride, (size_t)stride * h, odom, out));
    }
    // mTrack for streams 0 .. B-1 (mCreateFrame for those without a reference frame)
    void track(int B, const uint8_t* frames, bool on_device, int w, int h, int stride, const float* odom, const se2gpu_track_kf* kf,
               se2gpu_track_result* out) {
        check(se2gpu_tracker_step(h_, B, frames, on_device, w, h, stride, (size_t)stride * h, odom, kf, out));
    }
    // resetLocalTrack for the streams whose keyframe the caller just made
    void resetLocalTrack(const std::vector<int>& streams, const std::vector<const float*>& d_view_mp) {
        check(se2gpu_tracker_reset(h_, (int)streams.size(), streams.data(), d_view_mp.data()));
    }
    se2gpu_track_state state(int b) {
        se2gpu_track_state s;
        check(se2gpu_tracker_state(h_, b, &s));
        return s;
    }

  private:
    static void check(int rc) {
        if (rc != SE2GPU_OK) throw std::runtime_error(std::string("se2gpu_tracker: ") + se2gpu_last_error());
    }
    se2gpu_tracker* h_;
};

}  // namespace gpu
}  // namespace se2lam
