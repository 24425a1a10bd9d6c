#include "common.h"

namespace se2gpu {
thread_local std::string g_last_error;
std::atomic<unsigned long long> g_launches{0};

// the grow-only device block of one device's host-buffer entry points
struct Workspace {
    std::mutex mu;
    char* base = nullptr;
    size_t cap = 0;
};
static Workspace g_workspace[kMaxDevices];

HostStage::HostStage(int device) {
    rc_ = select_device(device);
    if (rc_ == SE2GPU_OK && device < kMaxDevices) {
        ws_ = &g_workspace[device];
        lock_ = std::unique_lock<std::mutex>(ws_->mu);
    }
}

HostStage::~HostStage() {
    for (void* p : temps_) cudaFree(p);
    if (ws_ && high_ > ws_->cap) {
        cudaFree(ws_->base);
        ws_->base = nullptr;
        ws_->cap = 0;
        if (cudaMalloc((void**)&ws_->base, high_) == cudaSuccess) ws_->cap = high_;
        else cudaGetLastError();                // the next call stages through temporary blocks again
    }
}

int HostStage::status() const {
    if (rc_) return rc_;
    if (err_ != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "%s failed: %s", what_, cudaGetErrorString(err_));
    return SE2GPU_OK;
}

void HostStage::check(cudaError_t e, const char* what) {
    if (e == cudaSuccess || err_ != cudaSuccess) return;
    err_ = e;
    what_ = what;
    cudaGetLastError();
}

void* HostStage::take(size_t bytes) {
    if (rc_ || err_ != cudaSuccess) return nullptr;
    const size_t n = ((bytes ? bytes : 1) + 255) & ~(size_t)255;
    high_ += n;
    if (ws_ && used_ + n <= ws_->cap) {
        void* p = ws_->base + used_;
        used_ += n;
        return p;
    }
    void* p = nullptr;
    check(cudaMalloc(&p, n), "cudaMalloc");
    if (!p) return nullptr;
    temps_.push_back(p);
    return p;
}

int HostStage::finish() {
    for (const Out& o : outs_)
        if (o.bytes) check(cudaMemcpy(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost), "cudaMemcpy to the host");
    return status();
}

}  // namespace se2gpu

extern "C" {

int se2gpu_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

const char* se2gpu_last_error(void) { return se2gpu::g_last_error.c_str(); }

unsigned long long se2gpu_launch_count(void) { return se2gpu::g_launches.load(); }

}  // extern "C"
