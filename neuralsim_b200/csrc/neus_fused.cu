// Fused per-ray NeuS stages for sm_90a: one warp owns one ray (pack) and keeps the ray's state in registers / shuffles.
// Each kernel replaces a chain of ~10-40 ATen / pack_ops launches of the reference's Python layer:
//   k_upsample_cdf      neus_packed_sdf_to_upsample_alpha | neus_packed_sdf_to_alpha -> packed_alpha_to_vw -> packed_cumsum(excl)
//                       -> / clamp_min(last,1e-5)                     (graphics/neus/neus_ray_query.py:873-884, neus_utils.py:164-188)
//   k_neus_alpha_fwd    sigmoid(sdf*inv_s) -> packed_diff -> /(cdf+1e-5) -> clamp_min(0) + the compression pass
//                       (neus_utils.py:88-111, pack_ops.py:286-291);  k_neus_alpha_bwd is its adjoint (d sdf, d inv_s)
//   k_composite_fwd/bwd packed_alpha_to_vw + packed_sum x4 + packed_div + products (single_volume_renderer.py:73-102) and
//                       their autograd rules (pack_ops.py:97-291)
// fp32 arithmetic follows the reference's operation order with explicit roundings where an index-valued result depends on
// it (transmittance recurrence / early stop: bit-exact, as in pack_ops.cu); plain sums differ by summation order only.
#include "neus_device.cuh"

namespace nsb {

constexpr int kNB = 256;   // 8 warps per CTA
__device__ __forceinline__ int64_t gwarp() { return ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int64_t nwarps() { return ((int64_t)gridDim.x * blockDim.x) >> 5; }
inline unsigned pack_grid(int64_t n_packs) { return wave_grid(n_packs * 32, kNB, 8); }

__global__ void __launch_bounds__(kNB)
k_upsample_cdf(const float *__restrict__ sdf, const float *__restrict__ dep, const int64_t *__restrict__ pi, int64_t n_packs, float inv_s,
               int use_estimate, float eps, float thre, float *__restrict__ cdf, const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    n_packs = eff_n(n_packs, n_dev);
    for (int64_t p = gwarp(); p < n_packs; p += nwarps()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        float T = 1.f, carry = 0.f, last_excl = 0.f;
        bool stopped = false;
        int cnt = 0;
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            float a = 0.f;
            if (k < n) a = use_estimate ? upsample_alpha_at(sdf, dep, b, n, k, inv_s) : neus_alpha_at(sdf, b, n, k, inv_s);
            float w;
            bool sel;
            replay_chunk(a, (int)min((int64_t)32, n - k0), lane, eps, thre, T, stopped, cnt, w, sel);
            const float inc = warp_scan_incl(w, lane) + carry;
            const float excl = inc - w;
            if (k < n) cdf[b + k] = excl;
            if (k == n - 1) last_excl = excl;
            carry = __shfl_sync(0xffffffffu, inc, 31);
        }
        last_excl = __shfl_sync(0xffffffffu, last_excl, (int)((n - 1) & 31));
        const float norm = fmaxf(last_excl, 1e-5f);
        __syncwarp();
        for (int64_t k = lane; k < n; k += 32) cdf[b + k] = __fdiv_rn(cdf[b + k], norm);
    }
}

// inverse-cdf sampling at u[0..n_s) shared by all packs (kernel_packed_invert_cdf semantics, pack_ops_cuda.cu:1634-1682)
__global__ void __launch_bounds__(256)
k_invert_cdf_shared_u(const float *__restrict__ bins, const float *__restrict__ cdfs, const float *__restrict__ u, const int64_t *__restrict__ pi,
                      int64_t n_packs, int n_s, float *__restrict__ samples, const int64_t *__restrict__ n_dev) {
    n_packs = eff_n(n_packs, n_dev);
    const int64_t total = n_packs * n_s, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t p = t / n_s;
        const int64_t b = pi[2 * p];
        const uint32_t n = (uint32_t)pi[2 * p + 1];
        const float *bb = bins + b, *cc = cdfs + b;
        const float uu = u[t - p * n_s];
        uint32_t first = 0, count = n;                       // lower bound, clamped to n-1
        while (count > 0) {
            const uint32_t step = count >> 1, it = first + step;
            if (cc[it] < uu) { first = it + 1; count -= step + 1; } else count = step;
        }
        const uint32_t pos = n ? min(first, n - 1) : 0;
        float r;
        if (pos == 0) r = bb[0];
        else {
            const float c0 = cc[pos - 1], pmf = __fsub_rn(cc[pos], c0);
            r = pmf < 1.0e-5f ? bb[pos - 1] : __fmaf_rn(__fdiv_rn(__fsub_rn(uu, c0), pmf), __fsub_rn(bb[pos], bb[pos - 1]), bb[pos - 1]);
        }
        samples[t] = r;
    }
}

// ------------------------------------------------------------------------------------------------ render alpha (+ compression)
__global__ void __launch_bounds__(kNB)
k_neus_alpha_fwd(const float *__restrict__ sdf, const int64_t *__restrict__ pi, int64_t n_packs, const float *__restrict__ inv_s_p, float eps,
                 float thre, float *__restrict__ alpha, uint8_t *__restrict__ selector, int32_t *__restrict__ num_steps,
                 const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    const float inv_s = inv_s_p[0];
    if (n_dev) {                                          // capacity > live packs: the packs in between keep nothing
        const int64_t live = eff_n(n_packs, n_dev);
        for (int64_t p = live + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_packs; p += (int64_t)gridDim.x * blockDim.x) num_steps[p] = 0;
        n_packs = live;
    }
    for (int64_t p = gwarp(); p < n_packs; p += nwarps()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        float T = 1.f;
        bool stopped = false;
        int cnt = 0;
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            const float a = (k < n) ? neus_alpha_at(sdf, b, n, k, inv_s) : 0.f;
            float w;
            bool sel;
            replay_chunk(a, (int)min((int64_t)32, n - k0), lane, eps, thre, T, stopped, cnt, w, sel);
            if (k < n) { alpha[b + k] = a; selector[b + k] = sel ? 1 : 0; }
        }
        if (lane == 0) num_steps[p] = cnt;
    }
}

// adjoint: alpha_i = max(0, (c_i - c_{i+1}) / (c_i + e)), c = sigmoid(s * inv_s)
//   d alpha_i / d c_i = (c_{i+1} + e) / (c_i + e)^2 ,  d alpha_i / d c_{i+1} = -1 / (c_i + e)   (where the clamp is inactive: raw >= 0)
__global__ void __launch_bounds__(kNB)
k_neus_alpha_bwd(const float *__restrict__ sdf, const int64_t *__restrict__ pi, int64_t n_packs, const float *__restrict__ inv_s_p,
                 const float *__restrict__ d_alpha, float *__restrict__ d_sdf, float *__restrict__ d_inv_s, const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    const float inv_s = inv_s_p[0];
    n_packs = eff_n(n_packs, n_dev);
    float acc_invs = 0.f;
    for (int64_t p = gwarp(); p < n_packs; p += nwarps()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        for (int64_t k = lane; k < n; k += 32) {
            const float g_own = (k < n - 1) ? d_alpha[b + k] : 0.f, g_prev = (k > 0) ? d_alpha[b + k - 1] : 0.f;
            if (g_own == 0.f && g_prev == 0.f) { d_sdf[b + k] = 0.f; continue; }     // most samples: compressed away / empty space
            const float s = sdf[b + k];
            const float c = sigmoidf_(s * inv_s);
            float gc = 0.f;                                             // dL/dc_k
            if (k < n - 1) {                                            // as c_i of interval k
                const float c1 = sigmoidf_(sdf[b + k + 1] * inv_s);
                const float den = c + 1e-5f;
                if ((c - c1) / den >= 0.f) gc += g_own * (c1 + 1e-5f) / (den * den);
            }
            if (k > 0) {                                                // as c_{i+1} of interval k-1
                const float cp = sigmoidf_(sdf[b + k - 1] * inv_s);
                const float den = cp + 1e-5f;
                if ((cp - c) / den >= 0.f) gc -= g_prev / den;
            }
            const float dc = c * (1.f - c);
            d_sdf[b + k] = gc * dc * inv_s;
            acc_invs += gc * dc * s;
        }
    }
    acc_invs = warp_sum(acc_invs);
    if (lane == 0 && acc_invs != 0.f) atomicAdd(d_inv_s, acc_invs);
}

// ------------------------------------------------------------------------------------------------ compositing
__global__ void __launch_bounds__(kNB)
k_composite_fwd(const float *__restrict__ alpha, const float *__restrict__ t, const float *__restrict__ rgb, const float *__restrict__ nab,
                const int64_t *__restrict__ pi, int64_t n_packs, float eps, float thre, int normalize_depth, const int64_t *__restrict__ ray_index,
                float *__restrict__ vw, float *__restrict__ mask, float *__restrict__ depth, float *__restrict__ rgb_out, float *__restrict__ nab_out,
                const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    n_packs = eff_n(n_packs, n_dev);
    for (int64_t p = gwarp(); p < n_packs; p += nwarps()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        float T = 1.f;
        bool stopped = false;
        int cnt = 0;
        float sm = 0.f, sd = 0.f, sr[3] = {0.f, 0.f, 0.f}, sn[3] = {0.f, 0.f, 0.f};
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            const float a = (k < n) ? alpha[b + k] : 0.f;
            float w;
            bool sel;
            replay_chunk(a, (int)min((int64_t)32, n - k0), lane, eps, thre, T, stopped, cnt, w, sel);
            if (k < n) {
                vw[b + k] = w;
                sm += w;
                sd = fmaf(w, t[b + k], sd);
                if (rgb) { sr[0] = fmaf(w, rgb[(b + k) * 3], sr[0]); sr[1] = fmaf(w, rgb[(b + k) * 3 + 1], sr[1]); sr[2] = fmaf(w, rgb[(b + k) * 3 + 2], sr[2]); }
                if (nab) { sn[0] = fmaf(w, nab[(b + k) * 3], sn[0]); sn[1] = fmaf(w, nab[(b + k) * 3 + 1], sn[1]); sn[2] = fmaf(w, nab[(b + k) * 3 + 2], sn[2]); }
            }
        }
        sm = warp_sum(sm); sd = warp_sum(sd);
#pragma unroll
        for (int c = 0; c < 3; ++c) { sr[c] = warp_sum(sr[c]); sn[c] = warp_sum(sn[c]); }
        if (lane == 0) {
            const int64_t o = ray_index ? ray_index[p] : p;          // per-pack outputs land at the ray's slot of the full image
            mask[o] = sm;
            depth[o] = normalize_depth ? sd / (sm + 1e-10f) : sd;
            if (rgb) { rgb_out[o * 3] = sr[0]; rgb_out[o * 3 + 1] = sr[1]; rgb_out[o * 3 + 2] = sr[2]; }
            if (nab) { nab_out[o * 3] = sn[0]; nab_out[o * 3 + 1] = sn[1]; nab_out[o * 3 + 2] = sn[2]; }
        }
    }
}

// g_w = gm + gd * (t - depth)/(M+e) [or gd*t] + g_rgb . rgb + g_n . nab ; then the alpha_to_vw adjoint (pack_ops_cuda.cu:1795-1848)
__global__ void __launch_bounds__(kNB)
k_composite_bwd(const float *__restrict__ alpha, const float *__restrict__ t, const float *__restrict__ rgb, const float *__restrict__ nab,
                const float *__restrict__ vw, const int64_t *__restrict__ pi, int64_t n_packs, float eps, float thre, int normalize_depth,
                const float *__restrict__ mask, const float *__restrict__ depth, const float *__restrict__ g_mask, const float *__restrict__ g_depth,
                const float *__restrict__ g_rgb, const float *__restrict__ g_nab, const float *__restrict__ g_vw_ext,
                const int64_t *__restrict__ ray_index, float *__restrict__ d_alpha, float *__restrict__ d_rgb, float *__restrict__ d_nab,
                const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    n_packs = eff_n(n_packs, n_dev);
    for (int64_t p = gwarp(); p < n_packs; p += nwarps()) {
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        const int64_t o = ray_index ? ray_index[p] : p;
        const float gm = g_mask ? g_mask[o] : 0.f, gd = g_depth ? g_depth[o] : 0.f;
        const float M = mask[o], Dp = depth[o];
        const float inv = normalize_depth ? 1.f / (M + 1e-10f) : 1.f;
        float gr[3] = {0.f, 0.f, 0.f}, gn[3] = {0.f, 0.f, 0.f};
        if (g_rgb) { gr[0] = g_rgb[o * 3]; gr[1] = g_rgb[o * 3 + 1]; gr[2] = g_rgb[o * 3 + 2]; }
        if (g_nab) { gn[0] = g_nab[o * 3]; gn[1] = g_nab[o * 3 + 1]; gn[2] = g_nab[o * 3 + 2]; }
        // pass 1: gw per sample (kept in d_alpha as scratch), accum = sum gw * w
        float accum = 0.f;
        for (int64_t k = lane; k < n; k += 32) {
            const float w = vw[b + k];
            float gw = gm + gd * (normalize_depth ? (t[b + k] - Dp) * inv : t[b + k]);
            if (g_vw_ext) gw += g_vw_ext[b + k];
            if (rgb) {
                gw += gr[0] * rgb[(b + k) * 3] + gr[1] * rgb[(b + k) * 3 + 1] + gr[2] * rgb[(b + k) * 3 + 2];
                d_rgb[(b + k) * 3] = w * gr[0]; d_rgb[(b + k) * 3 + 1] = w * gr[1]; d_rgb[(b + k) * 3 + 2] = w * gr[2];
            }
            if (nab) {
                gw += gn[0] * nab[(b + k) * 3] + gn[1] * nab[(b + k) * 3 + 1] + gn[2] * nab[(b + k) * 3 + 2];
                d_nab[(b + k) * 3] = w * gn[0]; d_nab[(b + k) * 3 + 1] = w * gn[1]; d_nab[(b + k) * 3 + 2] = w * gn[2];
            }
            d_alpha[b + k] = gw;
            accum += gw * w;
        }
        accum = warp_sum(accum);
        __syncwarp();
        float T = 1.f;
        bool stopped = false;
        for (int64_t k0 = 0; k0 < n; k0 += 32) {
            const int64_t k = k0 + lane;
            const float a = (k < n) ? alpha[b + k] : 0.f;
            const float gw = (k < n) ? d_alpha[b + k] : 0.f;
            const float gww = (k < n) ? gw * vw[b + k] : 0.f;
            float my_g = 0.f;
            if (!stopped) {
                const int lim = (int)min((int64_t)32, n - k0);
                for (int q = 0; q < lim; ++q) {
                    const float aq = __shfl_sync(0xffffffffu, a, q);
                    const float gq = __shfl_sync(0xffffffffu, gww, q);
                    if (T < eps) { stopped = true; break; }
                    if (aq < thre) continue;
                    if (q == lane) my_g = __fdiv_rn(gw * T - accum, fmaxf(1.f - aq, 1e-10f));
                    accum -= gq;
                    T *= (1.f - aq);
                }
            }
            if (k < n) d_alpha[b + k] = my_g;
        }
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int nsb_neus_upsample_cdf(const float *sdf, const float *depth, const int64_t *pack_infos, int64_t n_packs, float inv_s,
                                     int use_estimate_alpha, float early_stop_eps, float alpha_thre, float *cdf, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(sdf && depth && pack_infos && cdf, "nsb_neus_upsample_cdf: NULL argument");
    k_upsample_cdf<<<pack_grid(n_packs), kNB, 0, STREAM>>>(sdf, depth, pack_infos, n_packs, inv_s, use_estimate_alpha, early_stop_eps, alpha_thre, cdf, dn.a);
    return check_launch("nsb_neus_upsample_cdf");
}

extern "C" int nsb_packed_invert_cdf_shared_u(const float *bins, const float *cdfs, const float *u, const int64_t *pack_infos, int64_t n_packs,
                                              int32_t n_samples, float *samples, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0 || n_samples == 0) return 0;
    NSB_REQUIRE(bins && cdfs && u && pack_infos && samples, "nsb_packed_invert_cdf_shared_u: NULL argument");
    k_invert_cdf_shared_u<<<wave_grid(n_packs * n_samples, 256, 8), 256, 0, STREAM>>>(bins, cdfs, u, pack_infos, n_packs, n_samples, samples, dn.a);
    return check_launch("nsb_packed_invert_cdf_shared_u");
}

extern "C" int nsb_neus_alpha_forward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, float early_stop_eps,
                                      float alpha_thre, float *alpha, uint8_t *selector, int32_t *num_steps, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(sdf && pack_infos && inv_s_dev && alpha && selector && num_steps, "nsb_neus_alpha_forward: NULL argument");
    k_neus_alpha_fwd<<<pack_grid(n_packs), kNB, 0, STREAM>>>(sdf, pack_infos, n_packs, inv_s_dev, early_stop_eps, alpha_thre, alpha, selector, num_steps, dn.a);
    return check_launch("nsb_neus_alpha_forward");
}

extern "C" int nsb_neus_alpha_backward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, const float *d_alpha,
                                       float *d_sdf, float *d_inv_s, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(sdf && pack_infos && inv_s_dev && d_alpha && d_sdf && d_inv_s, "nsb_neus_alpha_backward: NULL argument");
    k_neus_alpha_bwd<<<pack_grid(n_packs), kNB, 0, STREAM>>>(sdf, pack_infos, n_packs, inv_s_dev, d_alpha, d_sdf, d_inv_s, dn.a);
    return check_launch("nsb_neus_alpha_backward");
}

extern "C" int nsb_composite_forward(const float *alpha, const float *t, const float *rgb, const float *nablas, const int64_t *pack_infos,
                                     int64_t n_packs, float early_stop_eps, float alpha_thre, int normalize_depth, const int64_t *ray_index,
                                     float *vw, float *mask, float *depth, float *rgb_out, float *nablas_out, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(alpha && t && pack_infos && vw && mask && depth, "nsb_composite_forward: NULL argument");
    NSB_REQUIRE((!rgb || rgb_out) && (!nablas || nablas_out), "nsb_composite_forward: missing output buffer");
    k_composite_fwd<<<pack_grid(n_packs), kNB, 0, STREAM>>>(alpha, t, rgb, nablas, pack_infos, n_packs, early_stop_eps, alpha_thre, normalize_depth,
                                                            ray_index, vw, mask, depth, rgb_out, nablas_out, dn.a);
    return check_launch("nsb_composite_forward");
}

extern "C" int nsb_composite_backward(const float *alpha, const float *t, const float *rgb, const float *nablas, const float *vw,
                                      const int64_t *pack_infos, int64_t n_packs, float early_stop_eps, float alpha_thre, int normalize_depth,
                                      const float *mask, const float *depth, const float *g_mask, const float *g_depth, const float *g_rgb,
                                      const float *g_nablas, const float *g_vw, const int64_t *ray_index, float *d_alpha, float *d_rgb,
                                      float *d_nablas, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(alpha && t && vw && pack_infos && mask && depth && d_alpha, "nsb_composite_backward: NULL argument");
    NSB_REQUIRE((!rgb || d_rgb) && (!nablas || d_nablas), "nsb_composite_backward: missing output buffer");
    k_composite_bwd<<<pack_grid(n_packs), kNB, 0, STREAM>>>(alpha, t, rgb, nablas, vw, pack_infos, n_packs, early_stop_eps, alpha_thre, normalize_depth,
                                                            mask, depth, g_mask, g_depth, g_rgb, g_nablas, g_vw, ray_index, d_alpha, d_rgb, d_nablas, dn.a);
    return check_launch("nsb_composite_backward");
}
