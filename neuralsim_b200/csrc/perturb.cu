// Perturbed (stratified) samples of the NeuS query with the draw sizes in device memory: torch.rand's values, made in the kernel.
//
// With perturb=True the reference draws, per query (nr3d_lib/graphics/neus/neus_ray_query.py:803, :821, :889):
//   the coarse depths   batch_sample_step_linear(near, far, nc1, perturb=True)   torch.rand([n_rays, nc1])   (graphics/raysample.py:285-310)
//   the marcher         rand_like of the marched samples' deltas                  torch.rand([M])           (occgrid_raymarch.py:96-110)
//   stage i             packed_sample_cdf(..., num_fine[i], perturb=True)        torch.rand([n_hit, nf_i])  (graphics/raysample.py:38-61)
// each from torch's default CUDA generator, draw k at offset base + sum_{j<k} inc(N_j) (torch_uniform.cuh).  These kernels take that
// list of draws as (count slot, multiplier) pairs, N_j = counts[slot_j] * mult_j; the last pair is the kernel's own draw, counts[slot] rows
// of mult values, so each kernel finds its offset and its size on the device and a captured step draws what the host-sized step draws.
//   k_coarse_perturbed     t[r, j] = addcmul(near[r], j + u[r, j], (far[r] - near[r]) / nc1) with torch's roundings
//   k_invert_cdf_perturbed u = addcmul(0, j + u[p, j], 1 / nf), then kernel_packed_invert_cdf (pack_ops_cuda.cu:1634-1682) at u: the
//                          body of nsb_packed_invert_cdf, without a u buffer
// A thread takes one curand_uniform4 and writes the four elements it covers, as torch's own grid-stride kernel does.
#include "neus_device.cuh"
#include "torch_uniform.cuh"

namespace nsb {

constexpr int kMaxDraws = 8;

struct Draws {
    int32_t n;
    int32_t slot[kMaxDraws], mult[kMaxDraws];
};

// this kernel's draw: Philox (seed, offset), its size n and its live rows (counts[slot] clamped to the capacity)
struct Draw {
    uint64_t seed, offset;
    int64_t n, rows;
};

__device__ __forceinline__ Draw find_draw(const int64_t *__restrict__ rng, const int64_t *__restrict__ counts, const Draws &d, int64_t cap_rows,
                                          int64_t grid_cap, int64_t *__restrict__ next_offset) {
    Draw w;
    w.seed = (uint64_t)rng[0];
    w.offset = (uint64_t)rng[1];
    int64_t c = 0, mult = 1;
#pragma unroll
    for (int k = 0; k < kMaxDraws; ++k) {             // unrolled: the draw list stays in registers
        if (k + 1 < d.n) w.offset += (uint64_t)torch_uniform_inc(counts[d.slot[k]] * d.mult[k], grid_cap);
        if (k + 1 == d.n) c = counts[d.slot[k]], mult = d.mult[k];
    }
    w.n = c > 0 ? c * mult : 0;
    w.rows = c < 0 ? 0 : (c < cap_rows ? c : cap_rows);
    if (next_offset && blockIdx.x == 0 && threadIdx.x == 0) *next_offset = (int64_t)(w.offset + (uint64_t)torch_uniform_inc(w.n, grid_cap));
    return w;
}

// grid-stride over the draw's (thread, iteration) units; f(li, u) for every element li < n of the unit
template <typename F>
__device__ __forceinline__ void for_each_uniform(const Draw &w, int64_t grid_cap, F f) {
    if (w.n <= 0) return;
    const int64_t stride = torch_uniform_stride(w.n, grid_cap);
    const int64_t units = ((w.n - 1) / (4 * stride) + 1) * stride;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < units; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t idx = q % stride, k = q / stride;
        const float4 r = torch_uniform4(w.seed, w.offset, idx, k);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int64_t li = idx + stride * (4 * k + c);
            if (li < w.n) f(li, c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w);
        }
    }
}

__global__ void __launch_bounds__(256)
k_coarse_perturbed(const float *__restrict__ near, const float *__restrict__ far, int64_t cap_rows, int nc1, float inv_nc1,
                   const int64_t *__restrict__ rng, const int64_t *__restrict__ counts, Draws d, int64_t grid_cap, float *__restrict__ t,
                   int64_t *__restrict__ next_offset) {
    const Draw w = find_draw(rng, counts, d, cap_rows, grid_cap, next_offset);
    for_each_uniform(w, grid_cap, [&](int64_t li, float u) {
        const int64_t r = li / nc1;
        if (r >= w.rows) return;
        const int j = (int)(li - r * nc1);
        const float n0 = near[r];
        // dt = (far - near) / nc1: torch divides by a host scalar as a product with its fp32 reciprocal (div_true_kernel_cuda);
        // idx = arange + rand; t = addcmul(near, idx, dt): one FMA in torch's kernel (measured bit-equal on an H100; the form with the
        // product rounded first differs in a quarter of the depths)
        const float dt = __fmul_rn(__fsub_rn(far[r], n0), inv_nc1);
        t[li] = __fmaf_rn(__fadd_rn((float)j, u), dt, n0);
    });
}

__global__ void __launch_bounds__(256)
k_invert_cdf_perturbed(const float *__restrict__ bins, const float *__restrict__ cdfs, const int64_t *__restrict__ pi, int64_t cap_packs, int nf,
                       float inv_nf, const int64_t *__restrict__ rng, const int64_t *__restrict__ counts, Draws d, int64_t grid_cap,
                       float *__restrict__ samples, int64_t *__restrict__ next_offset) {
    const Draw w = find_draw(rng, counts, d, cap_packs, grid_cap, next_offset);
    for_each_uniform(w, grid_cap, [&](int64_t li, float r) {
        const int64_t p = li / nf;
        if (p >= w.rows) return;
        const int j = (int)(li - p * nf);
        // batch_sample_step_linear(0, 1, nf, perturb=True): addcmul(0, j + r, (1 - 0) / nf), an FMA with a zero addend: the rounded product
        const float uu = __fmul_rn(__fadd_rn((float)j, r), inv_nf);
        const int64_t b = pi[2 * p];
        samples[li] = invert_cdf_one(bins + b, cdfs + b, (uint32_t)pi[2 * p + 1], uu);
    });
}

// the draw list of an entry point: n_draws (slot, multiplier) pairs, the last one the kernel's own draw of `width` values per row
inline int make_draws(const int32_t *draws_host, int32_t n_draws, int32_t width, const char *who, Draws &d) {
    NSB_REQUIRE(draws_host && n_draws >= 1 && n_draws <= kMaxDraws, "%s: 1 to %d draws, got %d", who, kMaxDraws, n_draws);
    d.n = n_draws;
    for (int k = 0; k < n_draws; ++k) {
        d.slot[k] = draws_host[2 * k];
        d.mult[k] = draws_host[2 * k + 1];
        NSB_REQUIRE(d.slot[k] >= 0 && d.slot[k] < 32 && d.mult[k] >= 1, "%s: draw %d: slot %d / multiplier %d out of range", who, k, d.slot[k], d.mult[k]);
    }
    NSB_REQUIRE(d.mult[n_draws - 1] == width, "%s: the last draw's multiplier %d is not the row width %d", who, d.mult[n_draws - 1], width);
    return 0;
}

// the units of the largest draw a capacity allows: its elements rounded up to a block, or a quarter of them plus one stride
inline unsigned perturbed_grid(int64_t cap_elems) {
    const int64_t a = cap_elems + kTorchRandBlock, b = cap_elems / 4 + kTorchRandBlock * torch_rand_grid_cap();
    return wave_grid(a < b ? a : b, 256, 8);
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int nsb_coarse_depths_perturbed(const float *near, const float *far, int64_t n_rays, int32_t n_samples, const int64_t *rng,
                                           const int64_t *counts, const int32_t *draws_host, int32_t n_draws, float *t, int64_t *next_offset,
                                           void *stream) {
    NSB_REQUIRE(n_rays >= 0 && n_samples >= 1, "nsb_coarse_depths_perturbed: bad size");
    NSB_REQUIRE(n_rays * (int64_t)n_samples < ((int64_t)1 << 31), "nsb_coarse_depths_perturbed: a draw of 2^31 or more values");
    NSB_REQUIRE(rng && counts && (n_rays == 0 || (near && far && t)), "nsb_coarse_depths_perturbed: NULL argument");
    Draws d;
    if (make_draws(draws_host, n_draws, n_samples, "nsb_coarse_depths_perturbed", d)) return 2;
    k_coarse_perturbed<<<perturbed_grid(n_rays * n_samples), 256, 0, STREAM>>>(near, far, n_rays, n_samples, 1.0f / (float)n_samples, rng, counts, d,
                                                                              torch_rand_grid_cap(), t, next_offset);
    return check_launch("nsb_coarse_depths_perturbed");
}

extern "C" int nsb_packed_invert_cdf_perturbed(const float *bins, const float *cdfs, const int64_t *pack_infos, int64_t n_packs, int32_t n_samples,
                                               const int64_t *rng, const int64_t *counts, const int32_t *draws_host, int32_t n_draws, float *samples,
                                               int64_t *next_offset, void *stream) {
    NSB_REQUIRE(n_packs >= 0 && n_samples >= 1, "nsb_packed_invert_cdf_perturbed: bad size");
    NSB_REQUIRE(n_packs * (int64_t)n_samples < ((int64_t)1 << 31), "nsb_packed_invert_cdf_perturbed: a draw of 2^31 or more values");
    NSB_REQUIRE(rng && counts && (n_packs == 0 || (bins && cdfs && pack_infos && samples)), "nsb_packed_invert_cdf_perturbed: NULL argument");
    Draws d;
    if (make_draws(draws_host, n_draws, n_samples, "nsb_packed_invert_cdf_perturbed", d)) return 2;
    k_invert_cdf_perturbed<<<perturbed_grid(n_packs * n_samples), 256, 0, STREAM>>>(bins, cdfs, pack_infos, n_packs, n_samples, 1.0f / (float)n_samples,
                                                                                   rng, counts, d, torch_rand_grid_cap(), samples, next_offset);
    return check_launch("nsb_packed_invert_cdf_perturbed");
}
