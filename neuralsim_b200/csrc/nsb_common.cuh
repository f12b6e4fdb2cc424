// Shared helpers of the neuralsim_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

#include "../../include/neuralsim_b200.h"

namespace nsb {

void set_error(const char *fmt, ...);
extern std::atomic<uint64_t> g_launches;

inline int check_launch(const char *what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
        cudaGetLastError();
        return 1;
    }
    return 0;
}

#define NSB_REQUIRE(cond, ...)        \
    do {                              \
        if (!(cond)) {                \
            nsb::set_error(__VA_ARGS__); \
            return 2;                 \
        }                             \
    } while (0)

inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}

// per DEVICE (a single process may drive several GPUs: render_parallel's worker threads)
inline int sm_count() {
    static std::atomic<int> cache[64];
    const int dev = current_device() & 63;
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n == 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, and the call is not free
bool smem_opt_in_needed(const void *kernel, int dev, int bytes);       // common.cu: remembers (kernel, device) -> bytes already granted
template <typename K>
inline void opt_in_smem(K kernel, int bytes) {
    // keyed by the kernel's ADDRESS: two instantiations of one template share their function-pointer type
    if (smem_opt_in_needed(reinterpret_cast<const void *>(kernel), current_device(), bytes))
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

// Resident CTAs per SM of `kernel` at this block size and dynamic shared memory (cudaOccupancyMaxActiveBlocksPerMultiprocessor), computed
// once per (kernel, device, block, bytes); common.cu.  Call it after opt_in_smem.
int max_active_ctas(const void *kernel, int dev, int block, int smem_bytes);
// A persistent grid sized for `ctas` resident CTAs per SM whose kernel fits fewer would run as serial waves, silently slower.  0 if the
// occupancy calculator agrees, else 2 with the error set.
template <typename K>
inline int require_ctas_per_sm(K kernel, int block, int smem_bytes, int ctas, const char *who) {
    const int got = max_active_ctas(reinterpret_cast<const void *>(kernel), current_device(), block, smem_bytes);
    NSB_REQUIRE(got >= ctas, "%s: %d CTAs per SM fit with %d bytes of dynamic shared memory, the persistent grid assumes %d", who, got, smem_bytes, ctas);
    return 0;
}

// Device-resident counts (nsb_bind_device_counts, include/neuralsim_b200.h): the entry points that support them take the binding of the
// calling thread; the kernels then process min(n_arg, *count) items, n_arg being the capacity the launch was sized for.
struct DevCounts { const int64_t *a, *b; };
DevCounts take_counts();
__device__ __forceinline__ int64_t eff_n(int64_t n, const int64_t *__restrict__ nd) {
    if (nd) { const int64_t v = *nd; return v < n ? (v < 0 ? 0 : v) : n; }
    return n;
}

// Device-resident LoTD level bound (nsb_bind_device_max_level): the level-aware entry points take the binding of the calling thread and
// their kernels read *level instead of the host max_level argument.
const int32_t *take_max_level();

// Grid size for grid-stride kernels: a whole number of waves of `ctas_per_sm` resident CTAs on all SMs.
inline unsigned wave_grid(int64_t work_items, int block, int ctas_per_sm) {
    int64_t need = (work_items + block - 1) / block;
    int64_t wave = (int64_t)sm_count() * ctas_per_sm;
    if (need <= wave) return (unsigned)(need > 0 ? need : 1);
    int64_t waves = (need + wave - 1) / wave;
    if (waves > 8) waves = 8;  // grid-stride loops cover the rest
    return (unsigned)(waves * wave);
}

// Grid size for persistent kernels: one CTA per work unit, at most `ctas_per_sm` resident CTAs on every SM; each CTA loops over the rest.
inline unsigned persistent_grid(int64_t work_units, int ctas_per_sm) {
    const int64_t wave = (int64_t)sm_count() * ctas_per_sm;
    return (unsigned)(work_units < wave ? work_units : wave);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// inclusive warp scan (sum)
__device__ __forceinline__ float warp_scan_incl(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}

__device__ __forceinline__ uint32_t ld_nc_u32(const void *p) {
    uint32_t r;
    asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

}  // namespace nsb
