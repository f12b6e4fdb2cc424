// Per-ray NeuS stage bodies shared by the stand-alone stage kernels (neus_fused.cu, neus_glue.cu) and -- round 2 -- the persistent per-ray
// kernel (ray_upsample.cu): they take plain pointers, so they run on global packs and on a ray's samples in shared memory alike.
#pragma once
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ float sigmoidf_(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }   // ATen: 1/(1+exp(-x))

// serial transmittance recurrence over one 32-element chunk, replayed by every lane from shuffled alphas
// (w = alpha*T; T *= 1-alpha; stop when T < eps; skip alpha <= thre)  -> this lane's weight, selected flag
__device__ __forceinline__ void replay_chunk(float a, int lim, int lane, float eps, float thre, float &T, bool &stopped, int &cnt,
                                             float &my_w, bool &my_sel) {
    my_w = 0.f;
    my_sel = false;
    if (stopped) return;
    // only the samples with alpha > thre change T; walk those (most chunks of most rays have none: empty space).  The early-stop
    // test `T < eps` of the reference runs before every sample; T only changes at the visited ones, so testing there (and once at
    // the chunk's start) stops at exactly the same sample.
    unsigned live = __ballot_sync(0xffffffffu, lane < lim && a > thre);
    if (T < eps) { stopped = true; return; }
    while (live) {
        const int q = __ffs(live) - 1;
        live &= live - 1;
        const float aq = __shfl_sync(0xffffffffu, a, q);
        if (q == lane) { my_w = __fmul_rn(aq, T); my_sel = true; }
        T = __fmul_rn(T, __fsub_rn(1.f, aq));
        ++cnt;
        if (T < eps) { stopped = (live != 0) || (q + 1 < lim); break; }
    }
}

// ------------------------------------------------------------------------------------------------ up-sampling cdf
__device__ __forceinline__ float upsample_alpha_at(const float *__restrict__ sdf, const float *__restrict__ dep, int64_t b, int64_t n,
                                                   int64_t k, float inv_s) {
    // interval k of the pack: [k, k+1]; the last element has sdf_diff = delta = 0 (packed_diff's trailing zero)
    const float s0 = sdf[b + k], d0 = dep[b + k];
    const bool last = (k == n - 1);
    const float ds = last ? 0.f : __fsub_rn(sdf[b + k + 1], s0);
    const float dt = last ? 0.f : __fsub_rn(dep[b + k + 1], d0);
    const float dot = __fdiv_rn(ds, __fadd_rn(dt, 1e-5f));
    float prev = 0.f;
    if (k > 0) {
        const float sp = sdf[b + k - 1], dp = dep[b + k - 1];
        prev = __fdiv_rn(__fsub_rn(s0, sp), __fadd_rn(__fsub_rn(d0, dp), 1e-5f));
    }
    const float slope = fminf(fmaxf(fminf(prev, dot), -10.f), 0.f);
    const float mid = __fadd_rn(s0, __fmul_rn(ds, 0.5f));
    const float e0 = __fmaf_rn(slope, __fmul_rn(dt, -0.5f), mid);          // addcmul: mid + slope * (dt * -0.5)
    const float e1 = __fmaf_rn(slope, __fmul_rn(dt, 0.5f), mid);
    const float c0 = sigmoidf_(__fmul_rn(e0, inv_s)), c1 = sigmoidf_(__fmul_rn(e1, inv_s));
    return fmaxf(__fdiv_rn(__fsub_rn(c0, c1), __fadd_rn(c0, 1e-5f)), 0.f);
}

__device__ __forceinline__ float neus_alpha_at(const float *__restrict__ sdf, int64_t b, int64_t n, int64_t k, float inv_s) {
    const float c0 = sigmoidf_(__fmul_rn(sdf[b + k], inv_s));
    if (k == n - 1) return fmaxf(__fdiv_rn(-0.f, __fadd_rn(c0, 1e-5f)), 0.f);
    const float c1 = sigmoidf_(__fmul_rn(sdf[b + k + 1], inv_s));
    return fmaxf(__fdiv_rn(__fsub_rn(c0, c1), __fadd_rn(c0, 1e-5f)), 0.f);      // -(c1 - c0) / (c0 + 1e-5)
}

}  // namespace nsb
