// Owning handles of the CUDA resources an engine holds: each releases its resource in its destructor and is move-only.
// The buffers grow with ensure(): a buffer sized by the largest request so far, reallocated only when a request exceeds
// it, keeping none of its old contents.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <memory>

namespace bgr {

struct CudaFree { void operator()(void* p) const { cudaFree(p); } };
struct CudaFreeHost { void operator()(void* p) const { cudaFreeHost(p); } };
struct CudaEventDestroy { void operator()(cudaEvent_t ev) const { cudaEventDestroy(ev); } };

// Device memory of `count` elements of T.
template <class T> class DeviceBuffer {
  public:
    // Holds at least `count` elements afterwards; frees and reallocates only when it held fewer.
    cudaError_t ensure(size_t count) {
        if (count <= n_) return cudaSuccess;
        p_.reset();
        n_ = 0;
        void* p = nullptr;
        const cudaError_t ce = cudaMalloc(&p, count * sizeof(T));
        if (ce != cudaSuccess) return ce;
        p_.reset(static_cast<T*>(p));
        n_ = count;
        return cudaSuccess;
    }
    T* get() const { return p_.get(); }

  private:
    std::unique_ptr<T, CudaFree> p_;
    size_t n_ = 0;
};

// Page-locked host memory of `count` elements of T, mapped into the device address space: get() on the host, dev() in
// kernels.
template <class T> class MappedHostBuffer {
  public:
    cudaError_t ensure(size_t count) {
        if (count <= n_) return cudaSuccess;
        p_.reset();
        n_ = 0;
        dev_ = nullptr;
        void* p = nullptr;
        cudaError_t ce = cudaHostAlloc(&p, count * sizeof(T), cudaHostAllocMapped);
        if (ce != cudaSuccess) return ce;
        p_.reset(static_cast<T*>(p));
        void* d = nullptr;
        ce = cudaHostGetDevicePointer(&d, p, 0);
        if (ce != cudaSuccess) { p_.reset(); return ce; }
        dev_ = static_cast<T*>(d);
        n_ = count;
        return cudaSuccess;
    }
    T* get() const { return p_.get(); }
    T* dev() const { return dev_; }

  private:
    std::unique_ptr<T, CudaFreeHost> p_;
    T* dev_ = nullptr;
    size_t n_ = 0;
};

// An event without timing, created by the first ensure().
class Event {
  public:
    cudaError_t ensure() {
        if (ev_) return cudaSuccess;
        cudaEvent_t ev = nullptr;
        const cudaError_t ce = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (ce == cudaSuccess) ev_.reset(ev);
        return ce;
    }
    cudaEvent_t get() const { return ev_.get(); }

  private:
    std::unique_ptr<CUevent_st, CudaEventDestroy> ev_;
};

}  // namespace bgr
