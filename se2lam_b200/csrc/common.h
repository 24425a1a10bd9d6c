// Shared host-side helpers of libse2gpu (error reporting, launch accounting, device selection, memory ownership).
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/se2gpu.h"

namespace se2gpu {

extern thread_local std::string g_last_error;
extern std::atomic<unsigned long long> g_launches;

inline int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define SE2_CUDA(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            return ::se2gpu::fail(SE2GPU_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                  __FILE__, __LINE__);                                                   \
    } while (0)

// every kernel launch of the library goes through this so that se2gpu_launch_count() is exact
#define SE2_LAUNCH(kernel, grid, block, smem, stream, ...)      \
    do {                                                        \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__); \
        ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed); \
    } while (0)

// size of the library's per-device tables (host workspaces, default matchers, prepared kernels)
constexpr int kMaxDevices = 64;

// the number of devices; a machine without one is SE2GPU_ERR_NO_DEVICE
inline int count_devices(int* n) {
    *n = 0;
    const cudaError_t e = cudaGetDeviceCount(n);
    if (e != cudaSuccess || *n <= 0) return fail(SE2GPU_ERR_NO_DEVICE, "no CUDA device available (%s)", cudaGetErrorString(e));
    return SE2GPU_OK;
}

// the device check of the handle-less _device entry points (they run on the caller's current device)
inline int require_device() {
    int n;
    return count_devices(&n);
}

inline int select_device(int device) {
    int n;
    { const int rc = count_devices(&n); if (rc) return rc; }
    if (device < 0 || device >= n) return fail(SE2GPU_ERR_INVALID, "device %d out of range (%d devices)", device, n);
    SE2_CUDA(cudaSetDevice(device));
    return SE2GPU_OK;
}

// Accumulates per-group kernel time with CUDA events recorded on the launching stream.
struct Profiler {
    static constexpr int MAXG = 16, MAXEV = 4096;
    bool on = false;
    int nev = 0;
    cudaEvent_t ev[MAXEV][2];
    int grp[MAXEV];
    bool created = false;
    double ms[MAXG] = {0};
    int launches[MAXG] = {0};
    void enable(bool e) {
        if (e && !created) { for (int i = 0; i < MAXEV; ++i) { cudaEventCreate(&ev[i][0]); cudaEventCreate(&ev[i][1]); } created = true; }
        on = e; nev = 0;
        for (int g = 0; g < MAXG; ++g) { ms[g] = 0; launches[g] = 0; }
    }
    void flush() {
        for (int i = 0; i < nev; ++i) {
            cudaEventSynchronize(ev[i][1]);
            float t = 0;
            cudaEventElapsedTime(&t, ev[i][0], ev[i][1]);
            ms[grp[i]] += t; launches[grp[i]]++;
        }
        nev = 0;
    }
    inline void begin(int g, cudaStream_t s) { if (on) { if (nev == MAXEV) flush(); grp[nev] = g; cudaEventRecord(ev[nev][0], s); } }
    inline void end(cudaStream_t s) { if (on) { cudaEventRecord(ev[nev][1], s); ++nev; } }
    ~Profiler() { if (created) for (int i = 0; i < MAXEV; ++i) { cudaEventDestroy(ev[i][0]); cudaEventDestroy(ev[i][1]); } }
};

// NVTX ranges around every kernel group and host entry point (visible in Nsight Systems / ncu --nvtx; a no-op when no tool is attached)
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
#define SE2_NVTX_CAT2(a, b) a##b
#define SE2_NVTX_CAT(a, b) SE2_NVTX_CAT2(a, b)
#define SE2_NVTX(name) ::se2gpu::NvtxRange SE2_NVTX_CAT(_se2_nvtx_, __LINE__)(name)

template <class T>
inline cudaError_t dev_alloc(T** p, size_t count) {
    return cudaMalloc((void**)p, (count ? count : 1) * sizeof(T));
}

// The device buffers of a handle: everything alloc() hands out is freed when the list is destroyed.
class DeviceBuffers {
  public:
    DeviceBuffers() = default;
    DeviceBuffers(const DeviceBuffers&) = delete;
    DeviceBuffers& operator=(const DeviceBuffers&) = delete;
    ~DeviceBuffers() { for (void* p : bufs_) cudaFree(p); }
    template <class T>
    cudaError_t alloc(T** p, size_t count) {
        const cudaError_t e = dev_alloc(p, count);
        if (e == cudaSuccess) bufs_.push_back((void*)*p);
        return e;
    }
    // a buffer that grows: *p, when this list owns it, is freed (its contents are not kept) and replaced by `count` elements
    template <class T>
    cudaError_t regrow(T** p, size_t count) {
        const auto it = std::find(bufs_.begin(), bufs_.end(), (void*)*p);
        if (*p && it != bufs_.end()) { cudaFree(*it); bufs_.erase(it); }
        *p = nullptr;
        return alloc(p, count);
    }

  private:
    std::vector<void*> bufs_;
};

// Device memory of one call of a host-buffer entry point. The constructor selects the device and takes that device's
// grow-only workspace, under its mutex, for the whole call. upload / output / inout / scratch hand out 256-byte aligned
// pieces of it; a piece that does not fit takes a temporary block, freed with the stage, and the workspace then grows to
// the call's high-water mark, so a later call of the same size allocates nothing. Copies are synchronous on the legacy
// default stream. The first CUDA error is kept: status() reports it as SE2GPU_ERR_CUDA (or select_device's failure), and
// once it is set no further piece, copy or launch check does anything.
struct Workspace;
class HostStage {
  public:
    explicit HostStage(int device);
    ~HostStage();
    HostStage(const HostStage&) = delete;
    HostStage& operator=(const HostStage&) = delete;

    int status() const;
    void check(cudaError_t e, const char* what);       // e.g. check(cudaGetLastError(), "kernel launch")
    template <class T>
    T* scratch(size_t count) { return static_cast<T*>(take(count * sizeof(T))); }
    template <class T>
    T* upload(const T* h, size_t count) {
        T* d = scratch<T>(count);
        if (d && count) check(cudaMemcpy(d, h, count * sizeof(T), cudaMemcpyHostToDevice), "cudaMemcpy to the device");
        return d;
    }
    template <class T>
    T* output(T* h, size_t count) {             // copied back to h by finish()
        T* d = scratch<T>(count);
        if (d) outs_.push_back({h, d, count * sizeof(T)});
        return d;
    }
    template <class T>
    T* inout(T* h, size_t count) {
        T* d = upload<T>(h, count);
        if (d) outs_.push_back({h, d, count * sizeof(T)});
        return d;
    }
    int finish();                               // copies the outputs back; status()

  private:
    struct Out { void* host; const void* dev; size_t bytes; };
    void* take(size_t bytes);
    Workspace* ws_ = nullptr;
    std::unique_lock<std::mutex> lock_;
    int rc_ = SE2GPU_OK;
    cudaError_t err_ = cudaSuccess;
    const char* what_ = "";
    size_t used_ = 0, high_ = 0;
    std::vector<void*> temps_;
    std::vector<Out> outs_;
};

// page-locked bump arena: uploads staged through it are real asynchronous DMA transfers (a cudaMemcpyAsync from a
// pageable std::vector is staged by the driver and returns only after the host-side copy)
struct PinnedArena {
    uint8_t* base = nullptr; size_t cap = 0, used = 0;
    ~PinnedArena() { if (base) cudaFreeHost(base); }
    bool reserve(size_t bytes) {
        used = 0;
        if (bytes <= cap) return true;
        if (base) cudaFreeHost(base);
        base = nullptr; cap = 0;
        if (cudaMallocHost((void**)&base, bytes + bytes / 4) != cudaSuccess) { cudaGetLastError(); return false; }
        cap = bytes + bytes / 4;
        return true;
    }
    template <typename T>
    T* alloc(size_t count) {       // page-locked array built in place (nullptr when the arena is exhausted / unavailable)
        const size_t bytes = (count * sizeof(T) + 63) & ~(size_t)63;
        if (!base || used + bytes > cap) return nullptr;
        T* p = reinterpret_cast<T*>(base + used);
        used += bytes;
        return p;
    }
    bool owns(const void* p) const { return base && p >= (const void*)base && p < (const void*)(base + cap); }
    template <typename T>
    int up(T* dst, const T* src, size_t count, cudaStream_t s) {
        if (!count) return SE2GPU_OK;
        const size_t bytes = count * sizeof(T);
        const void* from = src;
        if (base && used + bytes <= cap) { memcpy(base + used, src, bytes); from = base + used; used += (bytes + 63) & ~(size_t)63; }
        SE2_CUDA(cudaMemcpyAsync(dst, from, bytes, cudaMemcpyHostToDevice, s));
        return SE2GPU_OK;
    }
};

// Element offsets of the arrays that share one device buffer, each starting on a 32-element boundary: `o.x = L.take(n)`
// names the next n elements x, and L.size is the buffer's length.
struct Layout {
    size_t size = 0;
    size_t take(size_t n) {
        const size_t o = size;
        size += (n + 31) & ~(size_t)31;
        return o;
    }
};

// A Layout whose arrays are host data, packed (zero-padded) into one vector for one upload.
template <class T>
struct Packed : Layout {
    std::vector<T> data;
    template <class U>
    size_t put(const U* p, size_t n) {
        const size_t o = take(n);
        data.resize(size);
        std::copy(p, p + n, data.begin() + o);
        return o;
    }
    template <class V>
    size_t put(const V& v) { return put(v.data(), v.size()); }
};

// The context of a solver that plans each call on the host (global_ba.cu, se3_ba.cu): its device, a blocking stream for
// the host entries, grow-only device buffers for the plan (ints, long longs) and the work (doubles), and the pinned arena
// the plan goes up through. create_plan_context makes one; delete destroys it once its last call has completed.
struct PlanContext {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t uploaded = nullptr;  // the last plan upload out of the pinned arena has completed
    cudaEvent_t done = nullptr;      // the last kernel, which reads the plan and work buffers, has completed
    DeviceBuffers bufs;
    int* d_int = nullptr; size_t cap_int = 0;
    long long* d_ll = nullptr; size_t cap_ll = 0;
    double* d_dbl = nullptr; size_t cap_dbl = 0;
    PinnedArena arena;

    ~PlanContext() {
        cudaSetDevice(device);
        if (done) cudaEventSynchronize(done);
        if (stream) cudaStreamSynchronize(stream);
        if (uploaded) cudaEventDestroy(uploaded);
        if (done) cudaEventDestroy(done);
        if (stream) cudaStreamDestroy(stream);
    }

    template <class T>
    int grow(T** p, size_t* cap, size_t need) {
        if (need <= *cap && *p) return SE2GPU_OK;
        SE2_CUDA(cudaEventSynchronize(done));  // an earlier call, on any stream, may still read the buffer
        SE2_CUDA(bufs.regrow(p, need));
        *cap = need;
        return SE2GPU_OK;
    }

    // Grows d_int / d_ll to the plan and copies it there on stream s, ordered against the calls before on any stream:
    //  * the plan goes up through the pinned arena, so the previous call's copies out of it must have completed;
    //  * the previous call's kernel may run on another stream, and this call's copies and kernel overwrite what it reads,
    //    so s waits for it.
    // The caller launches its kernel on s and then records `done` there.
    int upload_plan(const std::vector<int>& ints, const std::vector<long long>& lls, cudaStream_t s) {
        { const int rc = grow(&d_int, &cap_int, ints.size()); if (rc) return rc; }
        { const int rc = grow(&d_ll, &cap_ll, lls.size()); if (rc) return rc; }
        SE2_CUDA(cudaEventSynchronize(uploaded));
        SE2_CUDA(cudaStreamWaitEvent(s, done, 0));
        arena.reserve(4 * ints.size() + 8 * lls.size() + 128);
        { const int rc = arena.up(d_int, ints.data(), ints.size(), s); if (rc) return rc; }
        { const int rc = arena.up(d_ll, lls.data(), lls.size(), s); if (rc) return rc; }
        SE2_CUDA(cudaEventRecord(uploaded, s));
        return SE2GPU_OK;
    }
};

template <class Ctx>
Ctx* create_plan_context(int device) {
    if (select_device(device)) return nullptr;
    Ctx* h = new Ctx;
    h->device = device;
    if (cudaStreamCreate(&h->stream) != cudaSuccess || cudaEventCreateWithFlags(&h->uploaded, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming) != cudaSuccess) {
        fail(SE2GPU_ERR_CUDA, "cudaStreamCreate / cudaEventCreate failed");
        delete h;
        return nullptr;
    }
    return h;
}

// n SE(3) links between N nodes (the global graph's edges, the window's odometry): from / to in range and distinct; with
// measure [16 n] and info [36 n] (host entries) also every measurement finite and every information finite and symmetric.
// `link` and `node` name them in the message.
inline int check_se3_links(int N, int n, const int* from, const int* to, const float* measure, const float* info, const char* link,
                           const char* node) {
    for (int e = 0; e < n; ++e) {
        if (from[e] < 0 || from[e] >= N || to[e] < 0 || to[e] >= N) return fail(SE2GPU_ERR_INVALID, "%s %d: %s out of range", link, e, node);
        if (from[e] == to[e]) return fail(SE2GPU_ERR_INVALID, "%s %d: from == to", link, e);
        if (!measure) continue;
        for (int k = 0; k < 16; ++k)
            if (!std::isfinite(measure[16 * (size_t)e + k])) return fail(SE2GPU_ERR_INVALID, "%s %d: measurement not finite", link, e);
        const float* I = info + 36 * (size_t)e;
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
                if (!std::isfinite(I[r * 6 + c])) return fail(SE2GPU_ERR_INVALID, "%s %d: information not finite", link, e);
                if (I[r * 6 + c] != I[c * 6 + r]) return fail(SE2GPU_ERR_INVALID, "%s %d: information not symmetric", link, e);
            }
    }
    return SE2GPU_OK;
}

// ---------------------------------------------------------------------------------------------- shared device helpers
// number of valid entries: *d_n clamped to [0, cap], or cap when there is no device-side count
__device__ __forceinline__ int count_of(const int* d_n, int cap) { return d_n ? min(max(*d_n, 0), cap) : cap; }

// exclusive prefix sum over the CTA of one value per thread (blockDim.x a multiple of 32); `total` receives the sum.
// s_warp: [32] ints of shared memory. Every thread of the CTA calls it; it ends with a barrier, so s_warp may be reused.
__device__ __forceinline__ int block_exclusive_sum(int x, int& total, int* s_warp) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        int v = lane < nw ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
        if (lane < nw) s_warp[lane] = v;
    }
    __syncthreads();
    const int excl = (w ? s_warp[w - 1] : 0) + inc - x;
    total = s_warp[nw - 1];
    __syncthreads();
    return excl;
}

// Hamming distance of two 256-bit ORB descriptors (8 x 32 bit, 16-byte aligned)
__device__ __forceinline__ int hamming256(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b) {
    const uint4 a0 = *reinterpret_cast<const uint4*>(a), a1 = *reinterpret_cast<const uint4*>(a + 4);
    const uint4 b0 = *reinterpret_cast<const uint4*>(b), b1 = *reinterpret_cast<const uint4*>(b + 4);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// ---------------------------------------------------------------------------------------------- entries shared between units
// Track::doTriangulate over B streams (geom.cu); see se2gpu_track_triangulate_batch_device. observed_tab / view_mp_tab, when
// set, give each stream's keyframe arrays by pointer (device memory) instead of at b * cap in observed / view_mp.
struct TrackTriArgs {
    const se2gpu_keypoint* kp_kf; int cap; const int* d_n;
    const se2gpu_keypoint* kp_fr; int cap_fr;
    int* matches;
    const uint8_t* observed; const float* view_mp;
    const uint8_t* const* observed_tab; const float* const* view_mp_tab;
    const float* Tcr; const int* gate; const float* K;
    float lower, upper, min_cos;
    float* local_mps; uint8_t* good_prl; int* counts;
};
int track_triangulate_launch(const TrackTriArgs& a, int B, cudaStream_t s);
float track_min_cos(int min_parallax_deg);
// Localizer::DoLocalBA for B streams (pose_ba.cu): stream b's keypoints d_kp + b * cap_kf (d_n[b] of them) with their map
// points d_obs_mp + b * cap_kf (-1: none); edges at b * cap_kf in d_xyz / d_uv / d_w, their count in d_edges[b];
// d_best [B * n_mp]. d_run[b] == 0 leaves stream b as it is (NO_EDGES); min_obs >= 0 gates at that many observations.
int loc_local_ba(int B, const se2gpu_keypoint* d_kp, int cap_kf, const int* d_n, const int* d_obs_mp, int n_mp, const float* d_mp_xyz,
                 const uint8_t* d_mp_use, const float* d_inv_sigma2, int nlevels, const int* d_run, int min_obs, int* d_best,
                 float* d_xyz, float* d_uv, float* d_w, int* d_edges, int* d_skip, int* d_n_obs, float* d_Tcw,
                 const se2gpu_pose_ba_params* params, int* d_iterations, int* d_status, cudaStream_t s);
// The set-up a stream capture must not contain, done ahead of one: the extractor's geometry tables and undistortion map for
// a w x hgt frame (orb.cu), the outlier kernel's table and shared-memory limit (fundam.cu); and whether MatchByWindow on
// cap1 x cap2 keypoints on `device` takes the shared-memory resolve, whose launches hold no host-to-device copy (matcher.cu;
// answered before any matcher is made, so a refused handle allocates nothing for it).
int orb_prepare_shape(se2gpu_orb* h, int w, int hgt, cudaStream_t s);
int fundam_prepare();
// GlobalMapper::RemoveMatchOutlierRansac (src/GlobalMapper.cpp:1207-1248) for `batch` keyframe pairs (fundam.cu): pair b's
// current keypoints at d_kp1 + b * cap1, its loop keyframe's at d_kp2 + d_slot2[b] * cap2 (negative: an empty pair), the
// matches d_matches12 + b * cap1 kept where cv::findFundamentalMat's mask is 1, all cleared when fewer than 10 are given.
// cap1 <= kFundamMaxPairs, checked by the caller.
constexpr int kFundamMaxPairs = 8192;
int remove_outliers_loop(int batch, const se2gpu_keypoint* d_kp1, int cap1, const se2gpu_keypoint* d_kp2, int cap2,
                         const int* d_slot2, int* d_matches12, cudaStream_t s);
bool matcher_window_capturable(int device, int cap1, int cap2);

}  // namespace se2gpu
