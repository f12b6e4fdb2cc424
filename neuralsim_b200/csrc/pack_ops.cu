// Packed-tensor ("ragged per-ray arrays") operators for sm_90a.
//
// Replaces the reference's `_pack_ops` extension (nr3d_lib/csrc/pack_ops/pack_ops_cuda.cu).
// The reference runs ONE THREAD PER PACK with serial inner loops, so neighbouring threads stride by the pack
// length (uncoalesced) and every wrapper syncs the host.  Here a WARP owns a pack: lanes sweep the pack in
// 32-element, fully coalesced chunks; reductions / scans use shuffles with a running carry; nothing
// synchronises with the host.  Index-valued results (search, merge, compaction) are bit-exact with the
// reference's serial semantics; fp32 sums differ only by summation order.
#include "neus_device.cuh"

namespace nsb {

constexpr int kWarpsPerBlock = 8;
constexpr int kBlock = kWarpsPerBlock * 32;

__device__ __forceinline__ int64_t warp_id_global() { return ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int64_t warps_total() { return ((int64_t)gridDim.x * blockDim.x) >> 5; }

inline unsigned warp_grid(int64_t n_packs) { return wave_grid(n_packs * 32, kBlock, 8); }

// ------------------------------------------------------------------ broadcast binary ops
template <int OP>
__device__ __forceinline__ float bin_arith(float a, float b) {
    if (OP == NSB_OP_ADD) return a + b;
    if (OP == NSB_OP_SUB) return a - b;
    if (OP == NSB_OP_MUL) return a * b;
    return __fdiv_rn(a, b);
}
template <int OP>
__device__ __forceinline__ bool bin_cmp(float a, float b) {
    if (OP == NSB_OP_GT) return a > b;
    if (OP == NSB_OP_GEQ) return a >= b;
    if (OP == NSB_OP_LT) return a < b;
    if (OP == NSB_OP_LEQ) return a <= b;
    if (OP == NSB_OP_EQ) return a == b;
    return a != b;
}

template <int OP>
__global__ void __launch_bounds__(kBlock)
k_packed_binary(const float *__restrict__ feats, const float *__restrict__ other, const int64_t *__restrict__ pi,
                int64_t n_packs, int C, void *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p] * C, n = pi[2 * p + 1] * C;
        for (int64_t k = lane; k < n; k += 32) {
            const float o = other[p * C + (k % C)];
            if (OP <= NSB_OP_DIV) ((float *)out)[b + k] = bin_arith<OP>(feats[b + k], o);
            else ((uint8_t *)out)[b + k] = bin_cmp<OP>(feats[b + k], o);
        }
    }
}

// ------------------------------------------------------------------ sum
__global__ void __launch_bounds__(kBlock)
k_packed_sum(const float *__restrict__ feats, const int64_t *__restrict__ pi, int64_t n_packs, int C,
             float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        if (C == 1) {
            float acc = 0.f;
            for (int64_t k = lane; k < n; k += 32) acc += feats[b + k];
            acc = warp_sum(acc);
            if (lane == 0) out[p] = acc;
        } else {
            // lanes sweep the flattened [n*C] range; lane l always sees channel (l + 32*iter) % C
            for (int c0 = 0; c0 < C; ++c0) {
                float acc = 0.f;
                for (int64_t k = lane; k < n; k += 32) acc += feats[(b + k) * C + c0];
                acc = warp_sum(acc);
                if (lane == 0) out[p * C + c0] = acc;
            }
        }
    }
}

// ------------------------------------------------------------------ cumsum (inclusive/exclusive, forward/reverse)
__global__ void __launch_bounds__(kBlock)
k_packed_cumsum(const float *__restrict__ feats, const int64_t *__restrict__ pi, int64_t n_packs, int C, int exclusive,
                int reverse, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        for (int c0 = 0; c0 < C; ++c0) {
            float carry = 0.f;
            for (int64_t k0 = 0; k0 < n; k0 += 32) {
                const int64_t k = k0 + lane;
                const int64_t src = reverse ? (n - 1 - k) : k;
                const float v = (k < n) ? feats[(b + src) * C + c0] : 0.f;
                const float s = warp_scan_incl(v, lane);
                const float inc = s + carry;
                // exclusive: inc - v, except at an inf or NaN v, where that is NaN; there the sum of the elements before it
                const float s_prev = __shfl_up_sync(0xffffffffu, s, 1);
                const float exc = isfinite(v) ? inc - v : (lane ? s_prev + carry : carry);
                if (k < n) out[(b + src) * C + c0] = exclusive ? exc : inc;
                carry = __shfl_sync(0xffffffffu, inc, 31);
            }
        }
    }
}

// ------------------------------------------------------------------ forward / backward difference
__global__ void __launch_bounds__(kBlock)
k_packed_diff(const float *__restrict__ feats, const int64_t *__restrict__ pi, int64_t n_packs, int C,
              const float *__restrict__ edge_val, const float *__restrict__ edge_fill, int backward,
              float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        const int64_t tot = n * C;
        for (int64_t k = lane; k < tot; k += 32) {
            const int64_t e = k / C;
            const int c0 = (int)(k - e * C);
            float r;
            if (!backward) {
                if (e < n - 1) r = feats[(b + e + 1) * C + c0] - feats[(b + e) * C + c0];
                else if (edge_val) r = edge_val[p * C + c0] - feats[(b + e) * C + c0];
                else if (edge_fill) r = edge_fill[p * C + c0];
                else r = 0.f;
            } else {
                if (e > 0) r = feats[(b + e) * C + c0] - feats[(b + e - 1) * C + c0];
                else if (edge_val) r = feats[(b + e) * C + c0] - edge_val[p * C + c0];
                else if (edge_fill) r = edge_fill[p * C + c0];
                else r = 0.f;
            }
            out[(b + e) * C + c0] = r;
        }
    }
}

// ------------------------------------------------------------------ sorted search (partition_point, search_bin: neus_device.cuh)
__global__ void __launch_bounds__(256)
k_packed_searchsorted(const float *__restrict__ bins, const float *__restrict__ vals, const int64_t *__restrict__ pi,
                      int64_t n_packs, int n_vals, int64_t *__restrict__ out) {
    const int64_t total = n_packs * n_vals, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t p = t / n_vals;
        const int64_t b = pi[2 * p];
        out[t] = b + search_bin(bins + b, (uint32_t)pi[2 * p + 1], vals[t]);
    }
}

__global__ void __launch_bounds__(256)
k_packed_invert_cdf(const float *__restrict__ bins, const float *__restrict__ cdfs, const float *__restrict__ u,
                    const int64_t *__restrict__ pi, int64_t n_packs, int n_samples, float *__restrict__ samples,
                    int64_t *__restrict__ bin_idx) {
    // kernel_packed_invert_cdf, pack_ops_cuda.cu:1634-1682, one thread per (pack, sample)
    const int64_t total = n_packs * n_samples, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t p = t / n_samples;
        const int64_t b = pi[2 * p];
        const uint32_t n = (uint32_t)pi[2 * p + 1];
        uint32_t pos;
        samples[t] = invert_cdf_one(bins + b, cdfs + b, n, u[t], &pos);
        if (bin_idx) bin_idx[t] = (int64_t)pos + b;
    }
}

// ------------------------------------------------------------------ merge of two sorted, aligned packs
// Closed form of kernel_try_merge_two_packs_sorted_aligned (pack_ops_cuda.cu:1506-1571) for b_sorted.  The reference searches b_j
// in a[last:], from the bin i of the b before it; a and b are ascending with any NaNs last (torch.sort's order).  A NaN b_j finds
// nothing below it there and takes the bin of the last number in b (0 if b has none), so with m the count of numbers in b:
//   i_j = lower_bound(a, key_j),  key_j = b[j] for j < m, else b[m - 1] (NaN when m = 0, whose lower bound is 0)
//   pidx_b[j] = out_begin + j + i_j
//   pidx_a[i] = out_begin + i + #{ j : i_j <= i } = out_begin + i + (c < m ? c : bn),  c = #{ j < m : !(a[i] < b[j]) }
// so every element is independent and a warp sweeps both packs coalesced.
__global__ void __launch_bounds__(kBlock)
k_merge_sorted_aligned(const float *__restrict__ va, const int64_t *__restrict__ pia, const float *__restrict__ vb,
                       const int64_t *__restrict__ pib, const int64_t *__restrict__ pio, int64_t n_packs,
                       int64_t *__restrict__ pidx_a, int64_t *__restrict__ pidx_b) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t ab = pia[2 * p], bb = pib[2 * p], ob = pio[2 * p];
        const uint32_t an = (uint32_t)pia[2 * p + 1], bn = (uint32_t)pib[2 * p + 1];
        const uint32_t m = partition_point(vb + bb, bn, [](float x) { return !isnan(x); });
        for (uint32_t i = lane; i < an; i += 32) {
            const float v = va[ab + i];
            const uint32_t c = partition_point(vb + bb, m, [&](float x) { return !(v < x); });
            pidx_a[ab + i] = ob + i + (c < m ? c : bn);
        }
        for (uint32_t j = lane; j < bn; j += 32) {
            const float v = (j < m || m == 0) ? vb[bb + j] : vb[bb + m - 1];
            pidx_b[bb + j] = ob + j + partition_point(va + ab, an, [&](float x) { return x < v; });
        }
    }
}

// b not sorted: the reference's serial bookkeeping (one thread per pack), kept verbatim in behaviour.
__global__ void __launch_bounds__(128)
k_merge_unsorted_b(const float *__restrict__ va, const int64_t *__restrict__ pia, const float *__restrict__ vb,
                   const int64_t *__restrict__ pib, const int64_t *__restrict__ pio, int64_t n_packs,
                   int64_t *__restrict__ pidx_a, int64_t *__restrict__ pidx_b) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_packs) return;
    const int64_t ab = pia[2 * p], bb = pib[2 * p], ob = pio[2 * p];
    const uint32_t an = (uint32_t)pia[2 * p + 1], bn = (uint32_t)pib[2 * p + 1];
    int64_t *ia = pidx_a + ab, *ib = pidx_b + bb;
    for (uint32_t i = 0; i < an; ++i) ia[i] = 0;
    for (uint32_t j = 0; j < bn; ++j) {
        const float v = vb[bb + j];
        const uint32_t i = partition_point(va + ab, an, [&](float x) { return x < v; });
        ib[j] = i;
        if (i < an) ia[i]++;
    }
    if (an > 0) {
        ia[0] += ob;
        for (uint32_t i = 1; i < an; ++i) ia[i] += ia[i - 1] + 1;
    }
    int64_t acc = 1, last = -1;
    for (uint32_t j = 0; j < bn; ++j) {
        const int64_t i = ib[j];
        if (i == last) ++acc; else acc = 0;
        ib[j] = acc + (i == 0 ? ob : ia[i - 1] + 1);
        last = i;
    }
}

// ------------------------------------------------------------------ alpha compositing weights
// w_j = alpha_j * T, T *= 1 - alpha_j, stop when T < eps, skip alpha <= thre (pack_ops_cuda.cu:1736-1793).
// The transmittance recurrence is evaluated in the reference's serial order (so the early-stop decision and the
// compaction selector are bit-exact), but by a whole warp: a 32-alpha chunk is loaded coalesced, every lane
// replays the chunk's recurrence from shuffled values and keeps the weight of its own element (replay_chunk).
__global__ void __launch_bounds__(kBlock)
k_alpha_to_vw_fwd(const float *__restrict__ alphas, const int64_t *__restrict__ pi, int64_t n_packs, float eps, float thre,
                  float *__restrict__ weights, int64_t *__restrict__ num_steps, uint8_t *__restrict__ selector) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        float T = 1.f;
        int cnt = 0;
        bool stopped = false;
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            const float a = (k < n) ? alphas[b + k] : 0.f;
            float my_w;
            bool my_sel;
            replay_chunk(a, (int)min((int64_t)32, n - k0), lane, eps, thre, T, stopped, cnt, my_w, my_sel);
            if (k < n) {
                if (weights) weights[b + k] = my_w;
                if (selector) selector[b + k] = my_sel ? 1 : 0;
            }
        }
        if (num_steps && lane == 0) num_steps[p] = cnt;
    }
}

// Backward (pack_ops_cuda.cu:1795-1848): grad_alpha_j = (gw_j*T_j - sum_{k>=j} gw_k w_k) / max(1-alpha_j, 1e-10)
// for the samples the forward visited (note `alpha < thre` here vs `<=` in the forward, as in the reference).
__global__ void __launch_bounds__(kBlock)
k_alpha_to_vw_bwd(const float *__restrict__ weights, const float *__restrict__ gw, const float *__restrict__ alphas,
                  const int64_t *__restrict__ pi, int64_t n_packs, float eps, float thre, float *__restrict__ ga) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        float accum = 0.f;
        for (int64_t k = lane; k < n; k += 32) accum += gw[b + k] * weights[b + k];
        accum = warp_sum(accum);
        float T = 1.f;
        bool stopped = false;
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            const float a = (k < n) ? alphas[b + k] : 0.f;
            const float gwk = (k < n) ? gw[b + k] : 0.f;
            const float gww = (k < n) ? gwk * weights[b + k] : 0.f;
            float my_g = 0.f;
            if (!stopped) {
                const int lim = (int)min((int64_t)32, n - k0);
                for (int q = 0; q < lim; ++q) {
                    const float aq = __shfl_sync(0xffffffffu, a, q);
                    const float gq = __shfl_sync(0xffffffffu, gww, q);
                    if (T < eps) { stopped = true; break; }
                    if (aq < thre) continue;
                    if (q == lane) my_g = __fdiv_rn(gwk * T - accum, fmaxf(1.f - aq, 1e-10f));
                    accum -= gq;
                    T *= (1.f - aq);
                }
            }
            if (k < n) ga[b + k] = my_g;
        }
    }
}

// ------------------------------------------------------------------ producers
__global__ void __launch_bounds__(kBlock)
k_interleave_linstep(const float *__restrict__ start, const int64_t *__restrict__ num_steps, const int64_t *__restrict__ cum,
                     const float *__restrict__ step, float step_scalar, int64_t n_packs, float *__restrict__ out,
                     int64_t *__restrict__ nidx) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t n = num_steps[p], b = cum[p] - n;
        const float s0 = start[p], st = step ? step[p] : step_scalar;
        for (int64_t j = lane; j < n; j += 32) {
            out[b + j] = __fmaf_rn((float)j, st, s0);          // one FMA, as nvcc compiles the reference's start + j*step
            if (nidx) nidx[b + j] = p;
        }
    }
}

__global__ void __launch_bounds__(kBlock)
k_interleave_arange(const int64_t *__restrict__ num_steps, const int64_t *__restrict__ cum, int64_t n_packs,
                    int64_t *__restrict__ out, int64_t *__restrict__ nidx) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t n = num_steps[p], b = cum[p] - n;
        for (int64_t j = lane; j < n; j += 32) {
            out[b + j] = j;
            if (nidx) nidx[b + j] = p;
        }
    }
}

__global__ void __launch_bounds__(256) k_mark_boundaries(const int64_t *__restrict__ ids, int64_t n, int32_t *__restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = (i == 0 || ids[i] != ids[i - 1]) ? 1 : 0;
}

// ------------------------------------------------------------------ per-pack sort (ascending, stable by index, NaN last)
// The sort's total order: every number before NaN, NaNs tied among themselves (numpy's and torch's order); -0 and +0 tie.
__device__ __forceinline__ bool sort_before(float x, float y) { return x < y || (!isnan(x) && isnan(y)); }
__device__ __forceinline__ bool sort_tie(float x, float y) { return x == y || (isnan(x) && isnan(y)); }

// Warp-cooperative rank sort: rank_i = #{k : v_k before v_i, or v_k tied with v_i and k < i}, a bijection onto [0, n) of the
// pack, so element i goes straight to vals[b + rank_i].  O(n^2/32) per pack, meant for the short per-ray packs of the N-object
// merge (buffer_compose_renderer.py:687); src is a copy of vals, read through L1.  Elements outside every pack are not touched.
__global__ void __launch_bounds__(kBlock)
k_packed_sort_rank(const float *__restrict__ src, const int64_t *__restrict__ pi, int64_t n_packs, float *__restrict__ vals,
                   int64_t *__restrict__ idx) {
    const int lane = threadIdx.x & 31;
    for (int64_t p = warp_id_global(); p < n_packs; p += warps_total()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        for (int64_t i = lane; i < n; i += 32) {
            const float vi = src[b + i];
            int64_t r = 0;
            for (int64_t k = 0; k < n; ++k) {
                const float vk = src[b + k];
                r += sort_before(vk, vi) || (sort_tie(vk, vi) && k < i);
            }
            vals[b + r] = vi;
            if (idx) idx[b + r] = b + i;
        }
    }
}

}  // namespace nsb

// ================================================================================================ C ABI
using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int nsb_packed_binary(int op, const float *feats, const float *other, const int64_t *pack_infos,
                                 int64_t n_packs, int32_t feat_dim, void *out, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(feats && other && pack_infos && out && feat_dim >= 1, "nsb_packed_binary: bad argument");
    const unsigned g = warp_grid(n_packs);
#define CASE(OP) case OP: k_packed_binary<OP><<<g, kBlock, 0, STREAM>>>(feats, other, pack_infos, n_packs, feat_dim, out); break;
    switch (op) {
        CASE(NSB_OP_ADD) CASE(NSB_OP_SUB) CASE(NSB_OP_MUL) CASE(NSB_OP_DIV) CASE(NSB_OP_GT) CASE(NSB_OP_GEQ)
        CASE(NSB_OP_LT) CASE(NSB_OP_LEQ) CASE(NSB_OP_EQ) CASE(NSB_OP_NEQ)
        default: set_error("nsb_packed_binary: unknown op %d", op); return 2;
    }
#undef CASE
    return check_launch("nsb_packed_binary");
}

extern "C" int nsb_packed_sum(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim, float *out,
                              void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(feats && pack_infos && out && feat_dim >= 1, "nsb_packed_sum: bad argument");
    k_packed_sum<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(feats, pack_infos, n_packs, feat_dim, out);
    return check_launch("nsb_packed_sum");
}

extern "C" int nsb_packed_cumsum(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim,
                                 int exclusive, int reverse, float *out, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(feats && pack_infos && out && feat_dim >= 1, "nsb_packed_cumsum: bad argument");
    k_packed_cumsum<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(feats, pack_infos, n_packs, feat_dim, exclusive, reverse, out);
    return check_launch("nsb_packed_cumsum");
}

extern "C" int nsb_packed_diff(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim,
                               const float *appends, const float *last_fill, int backward, float *out, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(feats && pack_infos && out && feat_dim >= 1, "nsb_packed_diff: bad argument");
    k_packed_diff<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(feats, pack_infos, n_packs, feat_dim, appends, last_fill, backward, out);
    return check_launch("nsb_packed_diff");
}

extern "C" int nsb_packed_searchsorted(const float *bins, const float *vals, const int64_t *pack_infos, int64_t n_packs,
                                       int32_t n_vals, int64_t *out_idx, void *stream) {
    if (n_packs == 0 || n_vals == 0) return 0;
    NSB_REQUIRE(bins && vals && pack_infos && out_idx, "nsb_packed_searchsorted: bad argument");
    k_packed_searchsorted<<<wave_grid(n_packs * n_vals, 256, 8), 256, 0, STREAM>>>(bins, vals, pack_infos, n_packs, n_vals, out_idx);
    return check_launch("nsb_packed_searchsorted");
}

extern "C" int nsb_packed_invert_cdf(const float *bins, const float *cdfs, const float *u, const int64_t *pack_infos,
                                     int64_t n_packs, int32_t n_samples, float *samples, int64_t *bin_idx, void *stream) {
    if (n_packs == 0 || n_samples == 0) return 0;
    NSB_REQUIRE(bins && cdfs && u && pack_infos && samples, "nsb_packed_invert_cdf: bad argument");
    k_packed_invert_cdf<<<wave_grid(n_packs * n_samples, 256, 8), 256, 0, STREAM>>>(bins, cdfs, u, pack_infos, n_packs,
                                                                                     n_samples, samples, bin_idx);
    return check_launch("nsb_packed_invert_cdf");
}

extern "C" int nsb_merge_two_packs_sorted_aligned(const float *vals_a, const int64_t *pack_infos_a, const float *vals_b,
                                                  const int64_t *pack_infos_b, const int64_t *pack_infos_out,
                                                  int64_t n_packs, int b_sorted, int64_t *pidx_a, int64_t *pidx_b,
                                                  void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(vals_a && vals_b && pack_infos_a && pack_infos_b && pack_infos_out && pidx_a && pidx_b,
                "nsb_merge_two_packs_sorted_aligned: bad argument");
    if (b_sorted)
        k_merge_sorted_aligned<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(vals_a, pack_infos_a, vals_b, pack_infos_b,
                                                                          pack_infos_out, n_packs, pidx_a, pidx_b);
    else
        k_merge_unsorted_b<<<(unsigned)((n_packs + 127) / 128), 128, 0, STREAM>>>(vals_a, pack_infos_a, vals_b, pack_infos_b,
                                                                                  pack_infos_out, n_packs, pidx_a, pidx_b);
    return check_launch("nsb_merge_two_packs_sorted_aligned");
}

extern "C" int nsb_packed_alpha_to_vw_forward(const float *alphas, const int64_t *pack_infos, int64_t n_packs,
                                              float early_stop_eps, float alpha_thre, float *weights, int64_t *num_steps,
                                              uint8_t *selector, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(alphas && pack_infos, "nsb_packed_alpha_to_vw_forward: bad argument");
    k_alpha_to_vw_fwd<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(alphas, pack_infos, n_packs, early_stop_eps, alpha_thre,
                                                                 weights, num_steps, selector);
    return check_launch("nsb_packed_alpha_to_vw_forward");
}

extern "C" int nsb_packed_alpha_to_vw_backward(const float *weights, const float *grad_weights, const float *alphas,
                                               const int64_t *pack_infos, int64_t n_packs, float early_stop_eps,
                                               float alpha_thre, float *grad_alphas, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(weights && grad_weights && alphas && pack_infos && grad_alphas, "nsb_packed_alpha_to_vw_backward: bad argument");
    k_alpha_to_vw_bwd<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(weights, grad_weights, alphas, pack_infos, n_packs,
                                                                 early_stop_eps, alpha_thre, grad_alphas);
    return check_launch("nsb_packed_alpha_to_vw_backward");
}

extern "C" int nsb_interleave_linstep(const float *start, const int64_t *num_steps, const int64_t *cumsum_steps,
                                      const float *step_size, float step_scalar, int64_t n_packs, float *out, int64_t *nidx,
                                      void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(start && num_steps && cumsum_steps && out, "nsb_interleave_linstep: bad argument");
    k_interleave_linstep<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(start, num_steps, cumsum_steps, step_size, step_scalar,
                                                                    n_packs, out, nidx);
    return check_launch("nsb_interleave_linstep");
}

extern "C" int nsb_interleave_arange(const int64_t *num_steps, const int64_t *cumsum_steps, int64_t n_packs, int64_t *out,
                                     int64_t *nidx, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(num_steps && cumsum_steps && out, "nsb_interleave_arange: bad argument");
    k_interleave_arange<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(num_steps, cumsum_steps, n_packs, out, nidx);
    return check_launch("nsb_interleave_arange");
}

extern "C" int nsb_packed_sort(float *vals, int64_t n_vals, const int64_t *pack_infos, int64_t n_packs, int64_t *idx, void *stream) {
    if (n_packs == 0) return 0;
    NSB_REQUIRE(vals && pack_infos, "nsb_packed_sort: bad argument");
    // the packs must end where vals ends (the reference's checkSize); the total lives on the device, in the last pack
    int64_t last[2];
    cudaMemcpyAsync(last, pack_infos + 2 * (n_packs - 1), sizeof(last), cudaMemcpyDeviceToHost, STREAM);
    cudaStreamSynchronize(STREAM);
    const int64_t n = last[0] + last[1];
    if (n != n_vals) {
        set_error("nsb_packed_sort: vals has %lld elements but the last pack ends at %lld", (long long)n_vals, (long long)n);
        return 2;
    }
    if (n == 0) return 0;
    float *tmp = nullptr;
    if (cudaMallocAsync(&tmp, n * sizeof(float), STREAM) != cudaSuccess) {
        set_error("nsb_packed_sort: out of device memory");
        return 3;
    }
    cudaMemcpyAsync(tmp, vals, n * sizeof(float), cudaMemcpyDeviceToDevice, STREAM);
    k_packed_sort_rank<<<warp_grid(n_packs), kBlock, 0, STREAM>>>(tmp, pack_infos, n_packs, vals, idx);
    const int rc = check_launch("nsb_packed_sort");
    cudaFreeAsync(tmp, STREAM);
    return rc;
}

extern "C" int nsb_mark_pack_boundaries(const int64_t *ids, int64_t n, int32_t *out, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(ids && out, "nsb_mark_pack_boundaries: bad argument");
    k_mark_boundaries<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(ids, n, out);
    return check_launch("nsb_mark_pack_boundaries");
}
