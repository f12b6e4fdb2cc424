// Per-ray NeuS stage bodies: the one statement of each, called by the stand-alone stage kernels (neus_fused.cu, neus_glue.cu), the
// persistent per-ray kernel (ray_upsample.cu) and the `_pack_ops` drop-in (pack_ops.cu).  They take plain pointers, so they run on global
// packs and on a ray's samples in shared memory alike, and the kernels agree bit for bit by construction.
#pragma once
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ float sigmoidf_(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }   // ATen: 1/(1+exp(-x))

// serial transmittance recurrence over one 32-element chunk, replayed by every lane from shuffled alphas
// (w = alpha*T; T *= 1-alpha; stop when T < eps; skip alpha <= thre, so a NaN alpha is visited as in the reference's
// packed_alpha_to_vw)  -> this lane's weight, selected flag
__device__ __forceinline__ void replay_chunk(float a, int lim, int lane, float eps, float thre, float &T, bool &stopped, int &cnt,
                                             float &my_w, bool &my_sel) {
    my_w = 0.f;
    my_sel = false;
    if (stopped) return;
    // only the samples that are not skipped change T; walk those (most chunks of most rays have none: empty space).  The early-stop
    // test `T < eps` of the reference runs before every sample; T only changes at the visited ones, so testing there (and once at
    // the chunk's start) stops at exactly the same sample.
    unsigned live = __ballot_sync(0xffffffffu, lane < lim && !(a <= thre));
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

// ------------------------------------------------------------------------------------------------ sorted search, inverse cdf, merge
// The number of leading elements of a[0, n) for which before(a[i]) holds; a is partitioned by `before` (those come first).  Each caller
// states its comparison: x < v gives the lower bound of v, x <= v or the reference's !(v < x) the upper bound; the two upper-bound forms
// differ when v or a key is NaN.  I is the index type of the caller (32-bit within a pack).
template <class I, class K, class Before>
__device__ __forceinline__ I partition_point(const K *a, I n, Before before) {
    I first = 0, count = n;
    while (count > 0) {
        const I step = count >> 1, it = first + step;
        if (before(a[it])) { first = it + 1; count -= step + 1; } else count = step;
    }
    return first;
}

// bin of v in a sorted pack: its lower bound clamped to n - 1, 0 in an empty pack (binary_search, pack_ops_cuda.cu:1365-1372)
__device__ __forceinline__ uint32_t search_bin(const float *a, uint32_t n, float v) {
    const uint32_t first = partition_point(a, n, [&](float x) { return x < v; });
    return n ? min(first, n - 1) : 0;
}

// warp per ray: the exclusive cdf of the up-sampling weights of a pack, normalised by max(last, 1e-5)
__device__ __forceinline__ void warp_upsample_cdf(const float *sdf, const float *dep, int n, float inv_s, int use_estimate, float eps, float thre,
                                                  float *cdf, int lane) {
    float T = 1.f, carry = 0.f, last_excl = 0.f;
    bool stopped = false;
    int cnt = 0;
    for (int k0 = 0; k0 < n; k0 += 32) {
        const int k = k0 + lane;
        float a = 0.f;
        if (k < n) a = use_estimate ? upsample_alpha_at(sdf, dep, 0, n, k, inv_s) : neus_alpha_at(sdf, 0, n, k, inv_s);
        float w;
        bool sel;
        replay_chunk(a, min(32, n - k0), lane, eps, thre, T, stopped, cnt, w, sel);
        const float inc = warp_scan_incl(w, lane) + carry;
        const float excl = inc - w;
        if (k < n) cdf[k] = excl;
        if (k == n - 1) last_excl = excl;
        carry = __shfl_sync(0xffffffffu, inc, 31);
    }
    last_excl = __shfl_sync(0xffffffffu, last_excl, (n - 1) & 31);
    const float norm = fmaxf(last_excl, 1e-5f);
    __syncwarp();
    for (int k = lane; k < n; k += 32) cdf[k] = __fdiv_rn(cdf[k], norm);
    __syncwarp();
}

// inverse-cdf sample of uu in a pack of bins bb / cdf cc (kernel_packed_invert_cdf, pack_ops_cuda.cu:1634-1682); its bin into *bin if given.
// An empty pack reads bb[0].
__device__ __forceinline__ float invert_cdf_one(const float *bb, const float *cc, uint32_t n, float uu, uint32_t *bin = nullptr) {
    const uint32_t pos = search_bin(cc, n, uu);
    if (bin) *bin = pos;
    if (pos == 0) return bb[0];
    const float c0 = cc[pos - 1], pmf = __fsub_rn(cc[pos], c0);
    // nvcc fuses the reference's b0 + t * (b1 - b0) into one FMA
    return pmf < 1.0e-5f ? bb[pos - 1] : __fmaf_rn(__fdiv_rn(__fsub_rn(uu, c0), pmf), __fsub_rn(bb[pos], bb[pos - 1]), bb[pos - 1]);
}

// warp per ray: merge sorted a and b with their payloads (sdf_m may be NULL: depths only).  Merged position of a_i = i + #{b <= a_i}, of
// b_j = j + #{a < b_j}: a b goes before an equal a (kernel_merge_two_packs_sorted_aligned's rule).
__device__ __forceinline__ void warp_merge(const float *dep_a, const float *sdf_a, int na, const float *dep_b, const float *sdf_b, int nb,
                                           float *dep_m, float *sdf_m, int lane) {
    for (int i = lane; i < na; i += 32) {
        const float v = dep_a[i];
        const int lo = partition_point(dep_b, nb, [&](float x) { return x <= v; });
        dep_m[i + lo] = v;
        if (sdf_m) sdf_m[i + lo] = sdf_a[i];
    }
    for (int j = lane; j < nb; j += 32) {
        const float v = dep_b[j];
        const int lo = partition_point(dep_a, na, [&](float x) { return x < v; });
        dep_m[j + lo] = v;
        if (sdf_m) sdf_m[j + lo] = sdf_b[j];
    }
    __syncwarp();
}

}  // namespace nsb
