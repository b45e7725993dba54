// cuda_owner.h — move-only owners of the CUDA runtime resources the renderer holds (host only): a device buffer, a pinned
// host buffer, an event, a stream.  Each frees its resource in its destructor and converts to the raw handle.  A failed
// creation is reported through fail() and the runtime's recorded error is read, so that the next call does not report
// it again.
#ifndef GLAVA_B200_CUDA_OWNER_H
#define GLAVA_B200_CUDA_OWNER_H

#include "internal.h"

#include <cuda_runtime.h>

namespace glb {

template <typename H, cudaError_t (*Release)(H)>
class Owner {
public:
    Owner() = default;
    Owner(Owner&& o) noexcept : h_(o.h_) { o.h_ = H(); }
    Owner& operator=(Owner&& o) noexcept {
        if (this != &o) { reset(); h_ = o.h_; o.h_ = H(); }
        return *this;
    }
    Owner(const Owner&) = delete;
    Owner& operator=(const Owner&) = delete;
    ~Owner() { reset(); }
    void reset() {
        if (h_) Release(h_);
        h_ = H();
    }
    H get() const { return h_; }

protected:
    // takes ownership of what `create` made; on failure stays empty and reports `what`
    int adopt(cudaError_t e, H h, const char* what, size_t bytes) {
        reset();
        if (e != cudaSuccess) {
            cudaGetLastError();
            if (!bytes) return fail(GLAVA_B200_ECUDA, "%s: %s", what, cudaGetErrorString(e));
            return fail(GLAVA_B200_ECUDA, "%s(%zu bytes): %s", what, bytes, cudaGetErrorString(e));
        }
        h_ = h;
        return 0;
    }
    H h_ = H();
};

// device memory as T[] (a buffer of 0 bytes takes 16)
template <typename T = void>
class DevBuf : public Owner<void*, cudaFree> {
public:
    int alloc(size_t bytes) {
        void* p = nullptr;
        if (bytes == 0) bytes = 16;
        const cudaError_t e = cudaMalloc(&p, bytes);
        return adopt(e, p, "cudaMalloc", bytes);
    }
    operator T*() const { return static_cast<T*>(h_); }
};

// pinned host memory as T[]
template <typename T>
class PinnedBuf : public Owner<void*, cudaFreeHost> {
public:
    int alloc(size_t bytes) {
        void* p = nullptr;
        const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
        return adopt(e, p, "cudaHostAlloc", bytes);
    }
    operator T*() const { return static_cast<T*>(h_); }
};

class Event : public Owner<cudaEvent_t, cudaEventDestroy> {
public:
    int create(unsigned flags = cudaEventDisableTiming) {
        cudaEvent_t e = nullptr;
        const cudaError_t err = cudaEventCreateWithFlags(&e, flags);
        return adopt(err, e, "cudaEventCreateWithFlags", 0);
    }
    operator cudaEvent_t() const { return h_; }
};

class Stream : public Owner<cudaStream_t, cudaStreamDestroy> {
public:
    int create(int priority) {
        cudaStream_t s = nullptr;
        const cudaError_t e = cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, priority);
        return adopt(e, s, "cudaStreamCreateWithPriority", 0);
    }
    operator cudaStream_t() const { return h_; }
};

}  // namespace glb

#endif
