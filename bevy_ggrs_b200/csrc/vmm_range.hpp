// Strided device ranges: every buffer of an engine whose size follows its row capacity.
//
// Engines created with BGR_CFG_GROWABLE reserve one virtual range of `n` strides once (the CUDA virtual memory
// management API); memory is mapped under a prefix of every stride, and growing maps more under each stride behind what
// is there.  No byte moves and no address changes, so pointers handed to queued launches stay valid while the range
// grows.  Other engines allocate the `n` strides with one cudaMalloc, all of it mapped.  The driver entry points come
// through cudaGetDriverEntryPoint: the library keeps static cudart as its only link-time dependency.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

namespace bgr {

struct VmmApi {
    PFN_cuMemAddressReserve_v10020 reserve = nullptr;
    PFN_cuMemAddressFree_v10020 address_free = nullptr;
    PFN_cuMemCreate_v10020 create = nullptr;
    PFN_cuMemRelease_v10020 release = nullptr;
    PFN_cuMemMap_v10020 map = nullptr;
    PFN_cuMemUnmap_v10020 unmap = nullptr;
    PFN_cuMemSetAccess_v10020 set_access = nullptr;
    PFN_cuMemGetAllocationGranularity_v10020 granularity = nullptr;
    PFN_cuGetErrorString_v6000 error_string = nullptr;
};

// The entry points, resolved once per process; nullptr (and *why) when the driver does not provide them.
inline const VmmApi* vmm_api(std::string* why) {
    static VmmApi api;
    static bool done = false, ok = false;
    if (!done) {
        done = true;
        ok = true;
        auto get = [&](const char* name, auto* fn) {
            void* p = nullptr;
            cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
            if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
                cudaGetLastError();
                ok = false;
                return;
            }
            *fn = reinterpret_cast<std::remove_pointer_t<decltype(fn)>>(p);
        };
        get("cuMemAddressReserve", &api.reserve);
        get("cuMemAddressFree", &api.address_free);
        get("cuMemCreate", &api.create);
        get("cuMemRelease", &api.release);
        get("cuMemMap", &api.map);
        get("cuMemUnmap", &api.unmap);
        get("cuMemSetAccess", &api.set_access);
        get("cuMemGetAllocationGranularity", &api.granularity);
        get("cuGetErrorString", &api.error_string);
    }
    if (!ok && why) *why = "the CUDA driver does not provide the virtual memory management entry points";
    return ok ? &api : nullptr;
}

inline std::string vmm_error(const VmmApi* api, const char* what, CUresult r) {
    const char* s = nullptr;
    if (api->error_string) api->error_string(r, &s);
    return std::string(what) + ": " + (s ? s : "unknown CUDA driver error");
}

inline size_t round_up(size_t v, size_t to) { return (v + to - 1) / to * to; }

// `n` strides of `stride` bytes at `base`; [0, mapped) of every stride is backed by memory.  Owns that memory: it is
// released when the range is destroyed, once the caller has synchronised every stream that used it.
struct StridedRange {
    CUdeviceptr base = 0;
    size_t stride = 0, mapped = 0, zeroed = 0, gran = 0;
    uint32_t n = 0;
    int device = 0;
    bool allocated = false;     // one cudaMalloc (allocate) rather than a reserved address range (reserve)
    std::vector<size_t> steps;  // mapped size after each growth step: every step is one mapping per stride

    StridedRange() = default;
    StridedRange(StridedRange&& o) noexcept { swap(o); }
    StridedRange& operator=(StridedRange&& o) noexcept { StridedRange t(std::move(o)); swap(t); return *this; }
    ~StridedRange() { free(); }

    template <class T = uint8_t> T* ptr() const { return reinterpret_cast<T*>(base); }
    bool empty() const { return base == 0; }

    // Allocates n contiguous strides of exactly `bytes` each, all mapped; map_to cannot grow them.
    bool allocate(uint32_t n_strides, size_t bytes, std::string* err) {
        void* p = nullptr;
        const cudaError_t ce = cudaMalloc(&p, size_t(n_strides) * bytes);
        if (ce != cudaSuccess) { *err = std::string("cudaMalloc: ") + cudaGetErrorString(ce); return false; }
        base = reinterpret_cast<CUdeviceptr>(p);
        n = n_strides;
        stride = mapped = bytes;
        gran = 1;
        allocated = true;
        return true;
    }

    // Reserves n strides of at least `stride_min` bytes each (rounded up to the allocation granularity); maps nothing.
    bool reserve(int dev, uint32_t n_strides, size_t stride_min, std::string* err) {
        const VmmApi* api = vmm_api(err);
        if (!api) return false;
        device = dev;
        n = n_strides;
        gran = granularity(dev, err);
        if (!gran) return false;
        stride = round_up(std::max<size_t>(stride_min, 1), gran);
        const CUresult r = api->reserve(&base, stride * n, gran, 0, 0);
        if (r != CUDA_SUCCESS) { base = 0; *err = vmm_error(api, "cuMemAddressReserve", r); return false; }
        return true;
    }

    static size_t granularity(int dev, std::string* err) {
        const VmmApi* api = vmm_api(err);
        if (!api) return 0;
        CUmemAllocationProp prop = props(dev);
        size_t g = 0;
        const CUresult r = api->granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
        if (r != CUDA_SUCCESS || g == 0) { *err = vmm_error(api, "cuMemGetAllocationGranularity", r); return 0; }
        return g;
    }

    // Maps memory so that every stride holds at least `bytes` (rounded up to the granularity): one physical allocation
    // per stride and step (cuMemMap maps a handle from its start only).  On failure nothing stays mapped that was not
    // mapped before, *err holds the driver's text, and false is returned.  The new bytes are zeroed by zero_new().
    bool map_to(size_t bytes, std::string* err) {
        const size_t target = round_up(bytes, gran);
        if (target <= mapped) return true;
        if (target > stride) { *err = "growth past the reserved address range"; return false; }
        const VmmApi* api = vmm_api(err);
        const size_t delta = target - mapped;
        CUmemAllocationProp prop = props(device);
        CUmemAccessDesc acc{};
        acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        acc.location.id = device;
        acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
        uint32_t done = 0;
        CUresult r = CUDA_SUCCESS;
        for (; done < n; ++done) {
            const CUdeviceptr at = base + size_t(done) * stride + mapped;
            CUmemGenericAllocationHandle h = 0;
            r = api->create(&h, delta, &prop, 0);
            if (r != CUDA_SUCCESS) { *err = vmm_error(api, "cuMemCreate", r); break; }
            r = api->map(at, delta, 0, h, 0);
            api->release(h);  // a mapping keeps its memory until it is unmapped
            if (r != CUDA_SUCCESS) { *err = vmm_error(api, "cuMemMap", r); break; }
            r = api->set_access(at, delta, &acc, 1);
            if (r != CUDA_SUCCESS) { *err = vmm_error(api, "cuMemSetAccess", r); ++done; break; }
        }
        if (r != CUDA_SUCCESS) {
            for (uint32_t i = 0; i < done; ++i) api->unmap(base + size_t(i) * stride + mapped, delta);
            return false;
        }
        mapped = target;
        steps.push_back(mapped);
        return true;
    }

    // Zeroes what was mapped since the last call, on `stream` (ordered behind every launch that used the range).
    cudaError_t zero_new(cudaStream_t stream) {
        const cudaError_t ce = zero(zeroed, mapped, stream);
        if (ce == cudaSuccess) zeroed = mapped;
        return ce;
    }

    // Zeroes [lo, hi) of every stride on `stream`: one memset when that is every stride whole.
    cudaError_t zero(size_t lo, size_t hi, cudaStream_t stream) const {
        if (lo >= hi) return cudaSuccess;
        if (lo == 0 && hi == stride) return cudaMemsetAsync(ptr(), 0, stride * n, stream);
        for (uint32_t i = 0; i < n; ++i) {
            const cudaError_t ce = cudaMemsetAsync(ptr() + size_t(i) * stride + lo, 0, hi - lo, stream);
            if (ce != cudaSuccess) return ce;
        }
        return cudaSuccess;
    }

    // Unmaps the growth steps taken after `bytes` were mapped (a growth that failed later on another range; nothing was
    // enqueued on those bytes yet).
    void shrink(size_t bytes) {
        const VmmApi* api = vmm_api(nullptr);
        while (!steps.empty() && steps.back() > bytes) {
            const size_t hi = steps.back();
            steps.pop_back();
            const size_t lo = steps.empty() ? 0 : steps.back();
            for (uint32_t i = 0; i < n; ++i) api->unmap(base + size_t(i) * stride + lo, hi - lo);
            mapped = lo;
        }
        zeroed = std::min(zeroed, mapped);
    }

    // Releases the memory (the caller has synchronised every stream that used it); the range is empty afterwards.
    void free() {
        if (allocated) cudaFree(ptr());
        else if (base) {
            shrink(0);
            vmm_api(nullptr)->address_free(base, stride * n);
        }
        base = 0;
        stride = mapped = zeroed = gran = 0;
        n = 0;
        allocated = false;
        steps.clear();
    }

  private:
    void swap(StridedRange& o) noexcept {
        std::swap(base, o.base); std::swap(stride, o.stride); std::swap(mapped, o.mapped); std::swap(zeroed, o.zeroed);
        std::swap(gran, o.gran); std::swap(n, o.n); std::swap(device, o.device); std::swap(allocated, o.allocated);
        steps.swap(o.steps);
    }

    static CUmemAllocationProp props(int dev) {
        CUmemAllocationProp prop{};
        prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
        prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        prop.location.id = dev;
        return prop;
    }
};

}  // namespace bgr
