// The StreetSurf LiDAR loss (app/loss/lidar.py: LidarLoss with DepthLoss and the `neus_unisim` LineOfSightLoss) on the renderer's own
// buffers, without a host read:
//   k_lidar_mask_err     the validity mask and the masked L1 error of every ray (lidar.py:259-266, 280; recon.py:40-53, utils.py:11-34)
//   k_kth_small / _hist  the k-th smallest error, sorted(err)[R // 2] bit for bit (lidar.py:281-283): an 8-bit-digit radix select
//   k_lidar_rows         the outlier discard (lidar.py:284) and the per-ray depth term f(pred, gt) * mask (recon.py:40-53, 119-129)
//   k_lidar_los_rows     one warp per kept ray: sum over its samples of [|t - gt| > eps] vw^2, times the mask (lidar.py:189-210)
//   k_lidar_reduce       one CTA: both terms, reduced over the whole-image rows in one fixed order
//   k_lidar_depth_bwd / k_lidar_los_bwd   their adjoints, the cotangents of the composite's depth and vw
// fp32 arithmetic uses explicit roundings (__f*_rn: no FMA contraction) in the reference's operation order; the sums are deterministic.
// The iteration-dependent scalars live in a device block blk = {w_depth, w_los, epsilon} the host refreshes before each step.
#include "nsb_common.cuh"

namespace nsb {

constexpr int kLidarL1 = 0, kLidarL2Relative = 1;

__device__ __forceinline__ float lidar_fn(int fn, float x, float y) {
    const float d = __fsub_rn(x, y);
    if (fn == kLidarL1) return fabsf(d);
    return __fdiv_rn(__fmul_rn(d, d), __fadd_rn(__fmul_rn(x, x), 0.01f));          // (x - y)^2 / (x^2 + 1e-2)
}

__global__ void __launch_bounds__(256)
k_lidar_mask_err(const float *__restrict__ pred, const float *__restrict__ mask_pred, const float *__restrict__ gt, int64_t n, float thresh,
                 int has_toofar, float toofar, float *__restrict__ mask, float *__restrict__ err) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const float g = gt[r];
        bool m = (mask_pred[r] > thresh) && (g > 0.f);
        if (has_toofar) m = g <= toofar;                   // the reference ASSIGNS here (lidar.py:265-266): the first mask is dropped
        const float mf = m ? 1.f : 0.f;
        mask[r] = mf;
        err[r] = __fmul_rn(fabsf(__fsub_rn(pred[r], g)), mf);
    }
}

// ---------------------------------------------------------------- k-th smallest (radix select on order-preserving keys)
// key(f) orders like torch.sort: negatives, -0, +0, positives, +inf, then NaN (a NaN's sign is dropped: its key is that of |NaN|).
__device__ __forceinline__ uint32_t order_key(float f) {
    const uint32_t b = __float_as_uint(f);
    if (f != f) return b | 0x80000000u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// One digit of the select: in hist[256] (the keys that match `prefix` above bit shift + 8), the digit holding the krem-th key (0-based).
__device__ __forceinline__ void radix_pick(const uint32_t *hist, int shift, uint32_t &prefix, uint32_t &krem) {
    uint32_t below = 0;
    for (int d = 0; d < 256; ++d) {
        const uint32_t c = hist[d];
        if (krem < below + c) {
            prefix |= (uint32_t)d << shift;
            krem -= below;
            return;
        }
        below += c;
    }
}

__device__ __forceinline__ bool radix_match(uint32_t key, uint32_t prefix, int shift) {
    return shift == 24 || (key >> (shift + 8)) == (prefix >> (shift + 8));
}

// small n: one CTA, four passes over the keys with the histogram in shared memory
__global__ void __launch_bounds__(1024)
k_kth_small(const float *__restrict__ v, int64_t n, int64_t k, float *__restrict__ out) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_prefix, s_krem;
    if (threadIdx.x == 0) { s_prefix = 0u; s_krem = (uint32_t)k; }
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int d = threadIdx.x; d < 256; d += blockDim.x) hist[d] = 0u;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t key = order_key(v[i]);
            if (radix_match(key, prefix, shift)) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) radix_pick(hist, shift, s_prefix, s_krem);
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = key_value(s_prefix);
}

// large n: pass `pass` (digit at 24 - 8 pass) histograms into hist[pass][256] (zero-filled by the caller); every CTA replays the picks of
// the earlier passes from their histograms.  k_kth_final replays all four and writes the value.
__device__ __forceinline__ void radix_replay(const uint32_t *__restrict__ hist, int passes, uint32_t k, uint32_t &prefix, uint32_t &krem) {
    prefix = 0u;
    krem = k;
    for (int p = 0; p < passes; ++p) radix_pick(hist + 256 * p, 24 - 8 * p, prefix, krem);
}

__global__ void __launch_bounds__(256)
k_kth_hist(const float *__restrict__ v, int64_t n, int64_t k, int pass, uint32_t *__restrict__ hist) {
    __shared__ uint32_t h[256];
    __shared__ uint32_t s_prefix;
    h[threadIdx.x] = 0u;
    if (threadIdx.x == 0) {
        uint32_t krem;
        radix_replay(hist, pass, (uint32_t)k, s_prefix, krem);
    }
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const int shift = 24 - 8 * pass;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t key = order_key(v[i]);
        if (radix_match(key, prefix, shift)) atomicAdd(&h[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[256 * pass + threadIdx.x], h[threadIdx.x]);
}

__global__ void k_kth_final(const uint32_t *__restrict__ hist, int64_t k, float *__restrict__ out) {
    uint32_t prefix, krem;
    radix_replay(hist, 4, (uint32_t)k, prefix, krem);
    out[0] = key_value(prefix);
}

// ---------------------------------------------------------------- loss rows
__global__ void __launch_bounds__(256)
k_lidar_rows(const float *__restrict__ pred, const float *__restrict__ gt, const float *__restrict__ err, const float *__restrict__ median,
             float factor, int fn, int64_t n, float *__restrict__ mask, float *__restrict__ depth_row, float *__restrict__ los_row) {
    const float thr = median ? __fmul_rn(median[0], factor) : 0.f;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        float m = mask[r];
        if (median && err[r] > thr) m = 0.f;               // strict >: a NaN error keeps its ray (lidar.py:284)
        mask[r] = m;
        if (depth_row) depth_row[r] = __fmul_rn(lidar_fn(fn, pred[r], gt[r]), m);
        if (los_row) los_row[r] = 0.f;                     // rays that keep no sample; k_lidar_los_rows writes the others
    }
}

__global__ void __launch_bounds__(256)
k_lidar_los_rows(const float *__restrict__ t, const float *__restrict__ vw, const int64_t *__restrict__ pi, const int64_t *__restrict__ rih,
                 int64_t n_packs, const float *__restrict__ gt, const float *__restrict__ mask, const float *__restrict__ blk,
                 float *__restrict__ los_row, const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    const float eps = blk[2];
    n_packs = eff_n(n_packs, n_dev);
    for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_packs; p += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const int64_t b = pi[2 * p], ns = pi[2 * p + 1], r = rih[p];
        const float g = gt[r];
        float acc = 0.f;
        for (int64_t k = lane; k < ns; k += 32) {
            const float w = vw[b + k];
            if (fabsf(__fsub_rn(t[b + k], g)) > eps) acc = __fadd_rn(acc, __fmul_rn(w, w));
        }
        acc = warp_sum(acc);
        if (lane == 0) los_row[r] = __fmul_rn(acc, mask[r]);
    }
}

// one CTA of 1024 threads: a fixed-order fp64 sum of each row array (thread i takes rows i, i + 1024, ..; then a fixed tree)
__global__ void __launch_bounds__(1024)
k_lidar_reduce(const float *__restrict__ depth_row, const float *__restrict__ los_row, int64_t n, int64_t n_kept, const float *__restrict__ blk,
               float *__restrict__ out, const int64_t *__restrict__ n_dev) {
    __shared__ double sa[1024], sb[1024];
    double a = 0.0, b = 0.0;
    for (int64_t r = threadIdx.x; r < n; r += 1024) {
        if (depth_row) a += (double)depth_row[r];
        if (los_row) b += (double)los_row[r];
    }
    sa[threadIdx.x] = a;
    sb[threadIdx.x] = b;
    __syncthreads();
    for (int s = 512; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sb[threadIdx.x] += sb[threadIdx.x + s]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int64_t kept = eff_n(n_kept, n_dev);
        out[0] = depth_row ? __fmul_rn(blk[0], (float)(sa[0] / (double)n)) : 0.f;
        out[1] = (los_row && kept > 0) ? __fmul_rn(blk[1], (float)(sb[0] / (double)kept)) : 0.f;
    }
}

// ---------------------------------------------------------------- adjoints (torch autograd's order: mean's backward multiplies by 1/N)
__global__ void __launch_bounds__(256)
k_lidar_depth_bwd(const float *__restrict__ pred, const float *__restrict__ gt, const float *__restrict__ mask, int64_t n, int fn,
                  const float *__restrict__ blk, const float *__restrict__ g_out, float *__restrict__ g_depth) {
    const float g0 = __fmul_rn(__fmul_rn(g_out[0], blk[0]), __fdiv_rn(1.f, (float)n));
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const float x = pred[r], g = __fmul_rn(g0, mask[r]);
        const float d = __fsub_rn(x, gt[r]);
        if (fn == kLidarL1) {
            g_depth[r] = __fmul_rn(g, (float)((d > 0.f) - (d < 0.f)));
        } else {
            // (x - y)^2 / den, den = x^2 + 1e-2: d/d(x - y) = g / den * 2 (x - y); d/d den = -g (num / den) / den, then * 2 x
            const float den = __fadd_rn(__fmul_rn(x, x), 0.01f), num = __fmul_rn(d, d);
            const float ga = __fmul_rn(__fdiv_rn(g, den), __fmul_rn(2.f, d));
            const float gb = __fmul_rn(-g, __fdiv_rn(__fdiv_rn(num, den), den));
            g_depth[r] = __fadd_rn(ga, __fmul_rn(gb, __fmul_rn(2.f, x)));
        }
    }
}

__global__ void __launch_bounds__(256)
k_lidar_los_bwd(const float *__restrict__ t, const float *__restrict__ vw, const int64_t *__restrict__ pi, const int64_t *__restrict__ rih,
                int64_t n_packs, const float *__restrict__ gt, const float *__restrict__ mask, const float *__restrict__ blk,
                const float *__restrict__ g_out, float *__restrict__ g_vw, const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    const float eps = blk[2];
    n_packs = eff_n(n_packs, n_dev);
    if (n_packs == 0) return;
    const float g0 = __fmul_rn(__fmul_rn(g_out[1], blk[1]), __fdiv_rn(1.f, (float)n_packs));
    for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_packs; p += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const int64_t b = pi[2 * p], ns = pi[2 * p + 1], r = rih[p];
        const float g = gt[r], gm = __fmul_rn(g0, mask[r]);
        for (int64_t k = lane; k < ns; k += 32) {
            const float w = vw[b + k];
            const float sel = fabsf(__fsub_rn(t[b + k], g)) > eps ? 1.f : 0.f;
            g_vw[b + k] = __fmul_rn(__fmul_rn(gm, sel), __fmul_rn(2.f, w));
        }
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

static constexpr int64_t kKthSmallMax = 1 << 16;          // up to this many keys, one CTA selects (one launch)

extern "C" int64_t nsb_kth_smallest_scratch_bytes(void) { return 4 * 256 * sizeof(uint32_t); }

extern "C" int nsb_lidar_mask_err(const float *pred, const float *mask_pred, const float *gt, int64_t n, float mask_pred_thresh, int32_t has_toofar,
                                  float discard_toofar, float *mask, float *err, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(pred && mask_pred && gt && mask && err, "nsb_lidar_mask_err: NULL argument");
    k_lidar_mask_err<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(pred, mask_pred, gt, n, mask_pred_thresh, has_toofar, discard_toofar, mask, err);
    return check_launch("nsb_lidar_mask_err");
}

extern "C" int nsb_kth_smallest(const float *v, int64_t n, int64_t k, float *out, void *scratch, void *stream) {
    NSB_REQUIRE(v && out, "nsb_kth_smallest: NULL argument");
    NSB_REQUIRE(n > 0 && n < ((int64_t)1 << 31) && k >= 0 && k < n, "nsb_kth_smallest: k = %lld outside [0, n = %lld) or n >= 2^31",
                (long long)k, (long long)n);
    if (n <= kKthSmallMax) {
        k_kth_small<<<1, 1024, 0, STREAM>>>(v, n, k, out);
        return check_launch("nsb_kth_smallest");
    }
    NSB_REQUIRE(scratch, "nsb_kth_smallest: n > %lld needs the scratch (nsb_kth_smallest_scratch_bytes)", (long long)kKthSmallMax);
    uint32_t *hist = (uint32_t *)scratch;
    cudaMemsetAsync(hist, 0, nsb_kth_smallest_scratch_bytes(), STREAM);
    for (int pass = 0; pass < 4; ++pass) {
        k_kth_hist<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(v, n, k, pass, hist);
        if (check_launch("nsb_kth_smallest")) return 1;
    }
    k_kth_final<<<1, 1, 0, STREAM>>>(hist, k, out);
    return check_launch("nsb_kth_smallest");
}

extern "C" int nsb_lidar_rows(const float *pred, const float *gt, const float *err, const float *median, float median_factor, int32_t fn_type,
                              int64_t n, float *mask, float *depth_row, float *los_row, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(pred && gt && mask && (!median || err), "nsb_lidar_rows: NULL argument");
    NSB_REQUIRE(fn_type == kLidarL1 || fn_type == kLidarL2Relative, "nsb_lidar_rows: fn_type %d is not built", (int)fn_type);
    k_lidar_rows<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(pred, gt, err, median, median_factor, fn_type, n, mask, depth_row, los_row);
    return check_launch("nsb_lidar_rows");
}

extern "C" int nsb_lidar_los_rows(const float *t, const float *vw, const int64_t *pack_infos, const int64_t *rays_inds_hit, int64_t n_packs,
                                  const float *gt, const float *mask, const float *blk, float *los_row, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(t && vw && pack_infos && rays_inds_hit && gt && mask && blk && los_row, "nsb_lidar_los_rows: NULL argument");
    k_lidar_los_rows<<<wave_grid(n_packs * 32, 256, 8), 256, 0, STREAM>>>(t, vw, pack_infos, rays_inds_hit, n_packs, gt, mask, blk, los_row, dn.a);
    return check_launch("nsb_lidar_los_rows");
}

extern "C" int nsb_lidar_loss_reduce(const float *depth_row, const float *los_row, int64_t n, int64_t n_kept, const float *blk, float *out,
                                     void *stream) {
    const DevCounts dn = take_counts();
    NSB_REQUIRE(blk && out && n > 0, "nsb_lidar_loss_reduce: NULL argument or n = 0");
    k_lidar_reduce<<<1, 1024, 0, STREAM>>>(depth_row, los_row, n, n_kept, blk, out, dn.a);
    return check_launch("nsb_lidar_loss_reduce");
}

extern "C" int nsb_lidar_depth_backward(const float *pred, const float *gt, const float *mask, int64_t n, int32_t fn_type, const float *blk,
                                        const float *g_out, float *g_depth, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(pred && gt && mask && blk && g_out && g_depth, "nsb_lidar_depth_backward: NULL argument");
    NSB_REQUIRE(fn_type == kLidarL1 || fn_type == kLidarL2Relative, "nsb_lidar_depth_backward: fn_type %d is not built", (int)fn_type);
    k_lidar_depth_bwd<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(pred, gt, mask, n, fn_type, blk, g_out, g_depth);
    return check_launch("nsb_lidar_depth_backward");
}

extern "C" int nsb_lidar_los_backward(const float *t, const float *vw, const int64_t *pack_infos, const int64_t *rays_inds_hit, int64_t n_packs,
                                      const float *gt, const float *mask, const float *blk, const float *g_out, float *g_vw, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(t && vw && pack_infos && rays_inds_hit && gt && mask && blk && g_out && g_vw, "nsb_lidar_los_backward: NULL argument");
    k_lidar_los_bwd<<<wave_grid(n_packs * 32, 256, 8), 256, 0, STREAM>>>(t, vw, pack_infos, rays_inds_hit, n_packs, gt, mask, blk, g_out, g_vw, dn.a);
    return check_launch("nsb_lidar_los_backward");
}
