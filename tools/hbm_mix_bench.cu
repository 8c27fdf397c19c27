// Microbenchmark: what HBM bandwidth does an H100 deliver for the ACCESS MIX of a rollback tick?
// The driver's MEASURED_PEAKS.json number is a 1:1 copy (read N, write N).  A SyncTest tick at d=8
// reads 1 image and writes 9 (1 read : 9 writes).  This tool measures, with CUDA events:
//   copy      1 read : 1 write   (plain 16-byte loads/stores)         == the driver's measurement shape
//   fill      0 read : 1 write
//   fanout    1 read : F writes  (plain stores)                       == the tick's mix: F = 8 Saves (live image deferred)
//   fanout_tma 1 read : F writes (cp.async.bulk global->smem->global)
//   write_bytes (optional): fanout stores only the first write_bytes of each target, the mix of a tick whose Saves store
//   part of the image (stable-plane elision: 33 B read : 8 x ~16 B written); copy, fill and fanout_tma stay whole-image.
// Usage: hbm_mix_bench [image_bytes] [F = 8 or 9] [write_bytes].  Output: one JSON line.  Not part of the product; evidence for the roofline discussion in DESIGN.md.
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__global__ void k_copy(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x)
        __stcs(dst + i, __ldcs(src + i));
}
__global__ void k_fill(uint4* __restrict__ dst, size_t n) {
    uint4 v = make_uint4(1, 2, 3, 4);
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x)
        __stcs(dst + i, v);
}
template <int F>
__global__ void k_fanout(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n, size_t stride, size_t m,
                         unsigned int* sink) {
    unsigned int acc = 0;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
        uint4 v = __ldcs(src + i);
        if (i < m) {
#pragma unroll
            for (int f = 0; f < F; ++f) __stcs(dst + f * stride + i, v);
        } else {
            acc ^= v.x ^ v.y ^ v.z ^ v.w;  // rows past write_bytes are read too: the load cannot sink into the branch
        }
    }
    if (acc == 0x9E3779B9u) *sink = acc;  // keeps the reads observable; practically never stores
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
// one chunk per block iteration: bulk load into smem, F bulk stores, 2 buffers
template <int F>
__global__ void __launch_bounds__(32, 1) k_fanout_tma(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t bytes,
                                                      size_t stride, uint32_t chunk) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar[2];
    if (threadIdx.x == 0) {
        for (int b = 0; b < 2; ++b) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&bar[b])), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const size_t n_chunks = (bytes + chunk - 1) / chunk;
    uint32_t it = 0;
    for (size_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++it) {
        const uint32_t b = it & 1u;
        const uint32_t sz = uint32_t(min(size_t(chunk), bytes - c * chunk));
        asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[b])), "r"(sz) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(smem + size_t(b) * chunk)), "l"(src + c * chunk), "r"(sz), "r"(smem_u32(&bar[b])) : "memory");
        uint32_t ok = 0;
        const uint32_t parity = (it >> 1) & 1u;
        while (!ok)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(smem_u32(&bar[b])), "r"(parity) : "memory");
#pragma unroll
        for (int f = 0; f < F; ++f)
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(dst + f * stride + c * chunk), "r"(smem_u32(smem + size_t(b) * chunk)), "r"(sz) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <class L>
static double time_us(L launch, int iters) {
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    for (int i = 0; i < 3; ++i) launch();
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(a));
    for (int i = 0; i < iters; ++i) launch();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, a, b));
    return double(ms) * 1e3 / iters;
}

template <int F>
static void run(size_t img, size_t write_bytes) {
    const size_t n = img / 16, m = std::min(n, write_bytes / 16), stride_v = (img / 16 + 63) & ~size_t(63);
    uint8_t *src, *dst;
    // large source ring so reads are not served by L2: rotate over 8 source images
    const int NSRC = 8;
    CK(cudaMalloc(&src, stride_v * 16 * NSRC));
    CK(cudaMalloc(&dst, stride_v * 16 * (F + 1) * 2));
    CK(cudaMemset(src, 1, stride_v * 16 * NSRC));
    unsigned int* sink;
    CK(cudaMalloc(&sink, sizeof(unsigned int)));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    int it = 0;
    auto srcp = [&]() { return reinterpret_cast<const uint4*>(src + (size_t(it++ % NSRC)) * stride_v * 16); };
    auto dstp = [&]() { return reinterpret_cast<uint4*>(dst + (size_t(it % 2)) * stride_v * 16 * (F + 1)); };
    const int iters = 50;
    double t_copy = time_us([&] { k_copy<<<sms * 8, 256>>>(srcp(), dstp(), n); }, iters);
    double t_fill = time_us([&] { k_fill<<<sms * 8, 256>>>(dstp(), n * F); }, iters);
    double t_fan = time_us([&] { k_fanout<F><<<sms * 8, 256>>>(srcp(), dstp(), n, stride_v, m, sink); }, iters);
    const uint32_t chunk = 48 * 1024;
    CK(cudaFuncSetAttribute(k_fanout_tma<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(2 * chunk)));
    double t_tma = time_us([&] { k_fanout_tma<F><<<sms * 2, 32, 2 * chunk>>>(reinterpret_cast<const uint8_t*>(srcp()), reinterpret_cast<uint8_t*>(dstp()), n * 16, stride_v * 16, chunk); }, iters);
    CK(cudaGetLastError());
    printf("{\"image_bytes\": %zu, \"write_bytes\": %zu, \"fanout\": %d, \"copy_1r1w\": {\"us\": %.2f, \"gbps\": %.0f}, \"fill_0r1w\": {\"us\": %.2f, \"gbps\": %.0f}, "
           "\"fanout_stg\": {\"us\": %.2f, \"gbps\": %.0f}, \"fanout_tma\": {\"us\": %.2f, \"gbps\": %.0f}}\n",
           n * 16, m * 16, F, t_copy, 2.0 * n * 16 / t_copy / 1e3, t_fill, double(F) * n * 16 / t_fill / 1e3,
           t_fan, (double(n) + double(F) * m) * 16 / t_fan / 1e3, t_tma, double(F + 1) * n * 16 / t_tma / 1e3);
}

int main(int argc, char** argv) {
    const size_t img = (argc > 1 ? size_t(atoll(argv[1])) : size_t(61) * 1000448);  // bytes of one image
    const int F = argc > 2 ? atoi(argv[2]) : 9;
    const size_t wb = argc > 3 ? size_t(atoll(argv[3])) : img;
    if (F == 8) run<8>(img, wb);
    else if (F == 9) run<9>(img, wb);
    else { fprintf(stderr, "fan-out must be 8 or 9\n"); return 2; }
    return 0;
}
