// Header-only forwarder of se2gpu_loc_* (include/se2gpu.h) shaped like Localizer::run's loop (reference
// src/Localizer.cpp:32-176): one call of localize() runs ReadFrameInfo, UpdatePoseCurr and, for the tracked streams,
// MatchLocalMap, DoLocalBA, UpdateCovisKFCurr, UpdateLocalMap(1) and DetectIfLost for B streams against the map uploaded
// at construction. The caller keeps DetectLoopClose / VerifyLoopClose (ComputeBoW, SearchByBoW, RemoveMatchOutlierRansac)
// and runs relocalize() for the streams it verified; WriteTrajFile reads the returned Tcw. INTEGRATION.md section 13 shows
// the loop.
#pragma once
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "../se2gpu.h"

namespace se2lam {
namespace gpu {

class LocalizerGpu {
  public:
    LocalizerGpu(int max_streams, int max_w, int max_h, const se2gpu_loc_params& p, const se2gpu_loc_map& map, int device = 0)
        : h_(se2gpu_loc_create(max_streams, max_w, max_h, &p, &map, device)) {
        if (!h_) throw std::runtime_error(std::string("se2gpu_loc_create: ") + se2gpu_last_error());
    }
    ~LocalizerGpu() { se2gpu_loc_destroy(h_); }
    LocalizerGpu(const LocalizerGpu&) = delete;
    LocalizerGpu& operator=(const LocalizerGpu&) = delete;

    // one iteration of Localizer::run's loop for streams 0 .. B-1 (frames of `stride` bytes per row, odom [B*3])
    void localize(int B, const uint8_t* frames, bool on_device, int w, int h, int stride, const float* odom, se2gpu_loc_result* out) {
        check(se2gpu_loc_step(h_, B, frames, on_device, w, h, stride, (size_t)stride * h, odom, out));
    }
    // the verified branch (Localizer.cpp:123-139) for one stream that was lost when its last step began: mapMatchGood as
    // VerifyLoopClose leaves it (idxCurr -> idxLoop, ascending idxCurr), kf_loop the index of mpKFLoop in the flattened map
    se2gpu_loc_result relocalize(int stream, int kf_loop, const std::map<int, int>& mapMatchGood) {
        std::vector<int> cur, loop;
        for (const auto& m : mapMatchGood) { cur.push_back(m.first); loop.push_back(m.second); }
        const int ptr[2] = {0, (int)cur.size()};
        se2gpu_loc_result r;
        check(se2gpu_loc_relocalize(h_, 1, &stream, &kf_loop, ptr, cur.data(), loop.data(), &r, nullptr));
        return r;
    }
    se2gpu_loc_stream_state state(int b) {
        se2gpu_loc_stream_state s;
        check(se2gpu_loc_state(h_, b, &s));
        return s;
    }

  private:
    static void check(int rc) {
        if (rc != SE2GPU_OK) throw std::runtime_error(std::string("se2gpu_loc: ") + se2gpu_last_error());
    }
    se2gpu_loc* h_;
};

}  // namespace gpu
}  // namespace se2lam
