// torch.rand on a CUDA generator, restated element by element, so that a kernel whose draw size lives in device memory draws exactly
// the values the host-sized path gets from torch.rand([N]) at the same (seed, offset).
//
// torch's uniform_ (ATen/native/cuda/DistributionTemplates.h: calc_execution_policy, distribution_elementwise_grid_stride_kernel,
// uniform_and_transform, uniform_kernel) launches blocks of 256 threads on grid = min(ceil(N / 256), SMs * (maxThreadsPerSM / 256)), and
// thread idx of stride = 256 * grid runs curand_init(seed, idx, offset) and, in its k-th loop iteration, one curand_uniform4 whose
// component c is element idx + stride * (4 k + c).  Each value v in (0, 1] becomes v * 1 + 0, then 0 where it is 1 (uniform_kernel).
// The generator's offset then advances by inc(N) = ((N - 1) / (4 stride) + 1) * 4; an empty draw neither runs nor advances it.
// Only the header-only device API of curand_kernel.h is used: the library still links cudart alone.
//
// torch.randint(high, [N]) on a CUDA generator is random_(0, high) -> random_from_to_kernel with range = high and base = 0.  For a range
// below 2^32 (every frame count) it takes the uint32 branch: distribution_nullary_kernel<scalar_t, uint32_t, curand4_engine_calls = 4>
// with dist_func = curand4 and transform uniform_int_from_to(v, range, base) = (int64)(v % range + base).  That kernel calls the same
// calc_execution_policy(N, unroll 4) as uniform_ -- the same grid, stride and offset increment inc(N) -- and the same grid-stride body:
// element idx + stride * (4 k + c) is component c of the k-th curand4 of Philox subsequence idx.  curand_uniform4 is a map of curand4
// applied to that same uint4, so the element mapping and inc() below serve both draws; torch_random4 only leaves the uint4 unmapped.
#pragma once
#include <cstdint>
#include <curand_kernel.h>

#include "nsb_common.cuh"

namespace nsb {

constexpr int64_t kTorchRandBlock = 256;

// torch's grid of a draw of n > 0 values on a device with grid_cap = SMs * (maxThreadsPerSM / 256) blocks, times the block: the stride
__host__ __device__ __forceinline__ int64_t torch_uniform_stride(int64_t n, int64_t grid_cap) {
    const int64_t g = (n + kTorchRandBlock - 1) / kTorchRandBlock;
    return kTorchRandBlock * (g < grid_cap ? g : grid_cap);
}

// torch's cap on the grid of a draw (calc_execution_policy): SMs * (maxThreadsPerSM / 256) blocks, per device
inline int64_t torch_rand_grid_cap() {
    static std::atomic<int64_t> cache[64];
    const int dev = current_device() & 63;
    int64_t c = cache[dev].load(std::memory_order_relaxed);
    if (c == 0) {
        int threads = 0;
        cudaDeviceGetAttribute(&threads, cudaDevAttrMaxThreadsPerMultiProcessor, current_device());
        c = (int64_t)sm_count() * (threads / kTorchRandBlock);
        if (c <= 0) c = 1;
        cache[dev].store(c, std::memory_order_relaxed);
    }
    return c;
}

// the offset increment of a draw of n values (0 for n <= 0)
__host__ __device__ __forceinline__ int64_t torch_uniform_inc(int64_t n, int64_t grid_cap) {
    if (n <= 0) return 0;
    return ((n - 1) / (4 * torch_uniform_stride(n, grid_cap)) + 1) * 4;
}

// the four values thread idx of a draw produces in its k-th iteration: .x .. .w are elements idx + stride * (4 k + 0 .. 3)
__device__ __forceinline__ float4 torch_uniform4(uint64_t seed, uint64_t offset, int64_t idx, int64_t k) {
    curandStatePhilox4_32_10_t s;
    curand_init(seed, (unsigned long long)idx, offset, &s);
    if (k > 0) skipahead((unsigned long long)(4 * k), &s);
    float4 r = curand_uniform4(&s);
    r.x = r.x == 1.f ? 0.f : r.x;
    r.y = r.y == 1.f ? 0.f : r.y;
    r.z = r.z == 1.f ? 0.f : r.z;
    r.w = r.w == 1.f ? 0.f : r.w;
    return r;
}

// element li of a draw of stride `stride` (torch_uniform_stride of the draw's size)
__device__ __forceinline__ float torch_uniform_at(uint64_t seed, uint64_t offset, int64_t li, int64_t stride) {
    const float4 r = torch_uniform4(seed, offset, li % stride, li / (4 * stride));
    const int c = (int)((li / stride) & 3);
    return c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w;
}

// the four uint32 of thread idx's k-th iteration of a torch.randint draw (curand4 of subsequence idx after k calls)
__device__ __forceinline__ uint4 torch_random4(uint64_t seed, uint64_t offset, int64_t idx, int64_t k) {
    curandStatePhilox4_32_10_t s;
    curand_init(seed, (unsigned long long)idx, offset, &s);
    if (k > 0) skipahead((unsigned long long)(4 * k), &s);
    return curand4(&s);
}

// element li of torch.randint(base, base + range, [N]) (range in [1, 2^32)) with stride torch_uniform_stride(N, grid_cap)
__device__ __forceinline__ int64_t torch_randint_at(uint64_t seed, uint64_t offset, int64_t li, int64_t stride, uint64_t range, int64_t base) {
    const uint4 r = torch_random4(seed, offset, li % stride, li / (4 * stride));
    const int c = (int)((li / stride) & 3);
    const uint32_t v = c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w;
    return (int64_t)((uint64_t)v % range) + base;
}

}  // namespace nsb
