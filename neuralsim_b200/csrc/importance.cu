// Error-map importance sampling of a camera's training batch, and the error-map update, inside the step.
//
// The shipped camera configs draw each batch with ImpSampler.sample_img_pixel(n) over one 'rgb' ErrorMap (nr3d_lib/models/importance.py:
// 317-336, 186-231): n_u = int(n * frac_uniform) uniform rays, then n_e = n - n_u from the map, with four draws of torch's generator in
// this order, each at the offset the previous one left (torch_uniform.cuh):
//   D1 randint(n_images, [n_u])            frame of uniform ray j                 (element j)
//   D2 rand([n_u, 2]).clamp_(1e-6, 1-1e-6) x, y of uniform ray j                  (elements 2j, 2j + 1)
//   D3 rand([n_e]).clamp_(...)             searchsorted(cdf_img, .) -> frame      (element j)
//   D4 rand([2, n_e]).clamp_(...)          x, y of map ray j, 2-D inverse cdf     (elements j, n_e + j)
// The inverse cdf of a coordinate is h = searchsorted(cdf, y) (left), ((y - prev) / (cdf[h] - prev) + h) / res, prev = cdf[h - 1] or 0:
// a true division, then the division by the host int res that torch's CUDA kernel makes a product with its fp32 reciprocal.  The pixel
// loader and the camera then snap (xy * WH).long().clamp_(0, WH - 1) (dataio/data_loader/pixel_loader.py:309-318, app/resources/
// observers/cameras.py:297-310) and lift the centre (w + 0.5, h + 0.5) with pinhole_lift (nr3d_lib/graphics/cameras/pinhole.py:71-72).
//   k_imp_sample        thread per ray: the draws, frame, xy, pose index, camera-space direction, ground-truth rows and appearance code
//   k_err_mark          thread per ray: the last ray in batch order of each (corner statement, cell), by atomicMax; the negative-error flag
//   k_err_apply         thread per cell: the four statements in order, each adding its last ray's value, then the marks reset to -1
// ErrorMap.update_error_map (importance.py:87-109) runs `error_map[i, h, w] += v` four times: a gather, an add and an index_put_ without
// accumulate, so a cell hit by several rays in one statement receives old + v of the LAST such ray (CPU torch, CUDA torch under
// use_deterministic_algorithms(True)).  The two launches give exactly that, whatever the thread order.
#include "nsb_common.cuh"
#include "torch_uniform.cuh"

namespace nsb {

struct ImpGt {
    int32_t n;
    int64_t row_bytes[NSB_IMP_MAX_GT];
    uint8_t *dst[NSB_IMP_MAX_GT];
};

__device__ __forceinline__ float clamp_u(float v) {
    // clamp_(1e-6, 1 - 1e-6): the Python doubles as fp32, min(max(v, lo), hi)
    constexpr float lo = (float)1e-6, hi = (float)(1.0 - 1e-6);
    return fminf(fmaxf(v, lo), hi);
}

// torch.searchsorted(cdf[0:n], v, right=False): the first i with cdf[i] >= v (n when none)
__device__ __forceinline__ int64_t search_left(const float *__restrict__ cdf, int64_t n, float v) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (cdf[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// one coordinate of ErrorMap.sample_pixel: -> the bin (clamped into [0, n): a value past the last cdf entry can not occur, cdf[n-1] ~ 1)
__device__ __forceinline__ float invert_1d(const float *__restrict__ cdf, int n, float inv_n, float v, int64_t &bin) {
    int64_t h = search_left(cdf, n, v);
    h = h < n ? h : n - 1;
    const float prev = h > 0 ? cdf[h - 1] : 0.f;
    bin = h;
    return __fmul_rn(__fadd_rn(__fdiv_rn(__fsub_rn(v, prev), __fsub_rn(cdf[h], prev)), (float)h), inv_n);
}

__global__ void __launch_bounds__(256)
k_imp_sample(const int64_t *__restrict__ table, const int64_t *__restrict__ cam, const int64_t *__restrict__ rng, int64_t n, int64_t n_u,
             int res_y, int res_x, float inv_res_y, float inv_res_x, int64_t grid_cap, ImpGt gt, const float *__restrict__ appear_table,
             int n_appear, float *__restrict__ h_appear, int64_t *__restrict__ fidx, float *__restrict__ xy, int64_t *__restrict__ pidx,
             float *__restrict__ dirs, int64_t *__restrict__ rng_next) {
    const int64_t *row = table + (*cam) * NSB_IMP_TABLE_WIDTH;
    const float *cdf_img = (const float *)row[0], *cdf_y = (const float *)row[1], *cdf_x = (const float *)row[2], *intr = (const float *)row[3];
    const int64_t F = row[4], W = row[5], H = row[6];
    const uint64_t seed = (uint64_t)rng[0];
    const int64_t n_e = n - n_u;
    const uint64_t o1 = (uint64_t)rng[1];
    const uint64_t o2 = o1 + (uint64_t)torch_uniform_inc(n_u, grid_cap);
    const uint64_t o3 = o2 + (uint64_t)torch_uniform_inc(2 * n_u, grid_cap);
    const uint64_t o4 = o3 + (uint64_t)torch_uniform_inc(n_e, grid_cap);
    if (rng_next && blockIdx.x == 0 && threadIdx.x == 0) {
        rng_next[0] = rng[0];
        rng_next[1] = (int64_t)(o4 + (uint64_t)torch_uniform_inc(2 * n_e, grid_cap));
    }
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t fi;
        float x, y;
        if (r < n_u) {
            fi = torch_randint_at(seed, o1, r, torch_uniform_stride(n_u, grid_cap), (uint64_t)F, 0);
            const int64_t s2 = torch_uniform_stride(2 * n_u, grid_cap);
            x = clamp_u(torch_uniform_at(seed, o2, 2 * r, s2));
            y = clamp_u(torch_uniform_at(seed, o2, 2 * r + 1, s2));
        } else {
            const int64_t j = r - n_u;
            fi = search_left(cdf_img, F, clamp_u(torch_uniform_at(seed, o3, j, torch_uniform_stride(n_e, grid_cap))));
            fi = fi < F ? fi : F - 1;
            const int64_t s4 = torch_uniform_stride(2 * n_e, grid_cap);
            const float ux = clamp_u(torch_uniform_at(seed, o4, j, s4));
            const float uy = clamp_u(torch_uniform_at(seed, o4, n_e + j, s4));
            int64_t h, w;
            y = invert_1d(cdf_y + fi * res_y, res_y, inv_res_y, uy, h);
            x = invert_1d(cdf_x + (fi * res_y + h) * res_x, res_x, inv_res_x, ux, w);
        }
        fidx[r] = fi;
        xy[2 * r] = x;
        xy[2 * r + 1] = y;
        if (!dirs) continue;                                     // an ErrorMap / ImpSampler draw: no camera
        pidx[r] = row[7] + fi;
        // (xy * WH).long().clamp_(0, WH - 1): the product in fp32, truncated
        int64_t pw = (int64_t)__fmul_rn(x, (float)W), ph = (int64_t)__fmul_rn(y, (float)H);
        pw = pw < 0 ? 0 : (pw > W - 1 ? W - 1 : pw);
        ph = ph < 0 ? 0 : (ph > H - 1 ? H - 1 : ph);
        // pinhole_lift(u, v, 1): x = (u - cx + cy * sk / fy - sk * v / fy) / fx * 1, y = (v - cy) / fy * 1, each op rounded
        const float *K = intr + fi * 9;
        const float fx = K[0], sk = K[1], cx = K[2], fy = K[4], cy = K[5];
        const float u = __fadd_rn((float)pw, 0.5f), v = __fadd_rn((float)ph, 0.5f);
        const float a = __fadd_rn(__fsub_rn(u, cx), __fdiv_rn(__fmul_rn(cy, sk), fy));
        dirs[3 * r] = __fdiv_rn(__fsub_rn(a, __fdiv_rn(__fmul_rn(sk, v), fy)), fx);
        dirs[3 * r + 1] = __fdiv_rn(__fsub_rn(v, cy), fy);
        dirs[3 * r + 2] = 1.f;
        const int64_t pix = (fi * H + ph) * W + pw;
#pragma unroll
        for (int k = 0; k < NSB_IMP_MAX_GT; ++k) {                // unrolled: the key list stays in parameter space
            if (k >= gt.n) break;
            const int64_t b = gt.row_bytes[k];
            const uint8_t *src = (const uint8_t *)row[11 + k] + pix * b;
            uint8_t *dst = gt.dst[k] + r * b;
            for (int64_t i = 0; i < b; ++i) dst[i] = src[i];
        }
        if (h_appear) {
            const float *code = appear_table + (row[8] + fi) * n_appear;
            for (int i = 0; i < n_appear; ++i) h_appear[r * n_appear + i] = code[i];
        }
    }
}

// the cell and value of corner statement s (0: (h, w), 1: (h+1, w), 2: (h, w+1), 3: (h+1, w+1)) of ray r, importance.py:96-109
struct Corners {
    int64_t cell;            // (i, h, w) after the clamps
    float wh, ww;            // hf - h, wf - w with the unclamped h, w
};

__device__ __forceinline__ Corners corners(const int64_t *__restrict__ fidx, const float *__restrict__ xy, int64_t r, int res_y, int res_x) {
    const float wf = __fmul_rn(xy[2 * r], (float)res_x), hf = __fmul_rn(xy[2 * r + 1], (float)res_y);
    int64_t w = (int64_t)wf, h = (int64_t)hf;
    Corners c;
    c.ww = __fsub_rn(wf, (float)w);
    c.wh = __fsub_rn(hf, (float)h);
    w = w < 0 ? 0 : (w > res_x - 2 ? res_x - 2 : w);
    h = h < 0 ? 0 : (h > res_y - 2 ? res_y - 2 : h);
    c.cell = (fidx[r] * res_y + h) * res_x + w;
    return c;
}

__device__ __forceinline__ int64_t corner_cell(const Corners &c, int s, int res_x) {
    return c.cell + ((s & 1) ? res_x : 0) + ((s & 2) ? 1 : 0);
}

// ((1 - w_h) or w_h) * ((1 - w_w) or w_w) * val, left to right
__device__ __forceinline__ float corner_value(const Corners &c, int s, float val) {
    const float a = (s & 1) ? c.wh : __fsub_rn(1.f, c.wh);
    const float b = (s & 2) ? c.ww : __fsub_rn(1.f, c.ww);
    return __fmul_rn(__fmul_rn(a, b), val);
}

// the map, its marks and its cells: the arguments, or camera *cam's row of the sampling table
struct MapRef {
    float *map;
    int32_t *last;
    int64_t cells;
};

__device__ __forceinline__ MapRef map_ref(float *map, int32_t *last, int64_t n_images, int res_y, int res_x, const int64_t *table, const int64_t *cam) {
    if (table) {
        const int64_t *row = table + (*cam) * NSB_IMP_TABLE_WIDTH;
        map = (float *)row[9];
        last = (int32_t *)row[10];
        n_images = row[4];
    }
    return MapRef{map, last, n_images * res_y * res_x};
}

__global__ void __launch_bounds__(256)
k_err_mark(float *map_arg, int32_t *last_arg, int64_t n_images, const int64_t *__restrict__ table, const int64_t *__restrict__ cam,
           const int64_t *__restrict__ fidx, const float *__restrict__ xy, const float *__restrict__ val, int64_t n, int res_y, int res_x,
           int32_t *__restrict__ flag, const int64_t *__restrict__ skip) {
    if (skip && *skip) return;
    const MapRef m = map_ref(map_arg, last_arg, n_images, res_y, res_x, table, cam);
    int32_t *__restrict__ last = m.last;
    const int64_t cells = m.cells;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        if (val[r] < 0.f) atomicOr(flag, 1);
        const Corners c = corners(fidx, xy, r, res_y, res_x);
#pragma unroll
        for (int s = 0; s < 4; ++s) atomicMax(last + s * cells + corner_cell(c, s, res_x), (int32_t)r);
    }
}

__global__ void __launch_bounds__(256)
k_err_apply(float *map_arg, int32_t *last_arg, int64_t n_images, const int64_t *__restrict__ table, const int64_t *__restrict__ cam,
            const int64_t *__restrict__ fidx, const float *__restrict__ xy, const float *__restrict__ val, int res_y, int res_x,
            const int64_t *__restrict__ skip) {
    if (skip && *skip) return;
    const MapRef mr = map_ref(map_arg, last_arg, n_images, res_y, res_x, table, cam);
    float *__restrict__ map = mr.map;
    int32_t *__restrict__ last = mr.last;
    const int64_t cells = mr.cells;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < cells; q += (int64_t)gridDim.x * blockDim.x) {
        int32_t rs[4];
        bool any = false;
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            rs[s] = last[s * cells + q];
            any |= rs[s] >= 0;
        }
        if (!any) continue;
        float m = map[q];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            if (rs[s] < 0) continue;
            m = __fadd_rn(m, corner_value(corners(fidx, xy, rs[s], res_y, res_x), s, val[rs[s]]));
            last[s * cells + q] = -1;
        }
        map[q] = m;
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int nsb_imp_sample(const int64_t *table, const int64_t *cam, const int64_t *rng, int64_t n, int64_t n_uniform, int32_t res_y,
                              int32_t res_x, int32_t n_gt, const int64_t *gt_row_bytes, void *const *gt_out, const float *appear_table,
                              int32_t n_appear, float *h_appear, int64_t *fidx, float *xy, int64_t *pidx, float *dirs, int64_t *rng_next,
                              void *stream) {
    NSB_REQUIRE(n >= 1 && n_uniform >= 0 && n_uniform <= n && res_y >= 1 && res_x >= 1, "nsb_imp_sample: bad size");
    NSB_REQUIRE(2 * n < ((int64_t)1 << 31), "nsb_imp_sample: a draw of 2^31 or more values");
    NSB_REQUIRE(table && cam && rng && fidx && xy && (!dirs || pidx), "nsb_imp_sample: NULL argument");
    NSB_REQUIRE(n_gt >= 0 && n_gt <= NSB_IMP_MAX_GT && (n_gt == 0 || (gt_row_bytes && gt_out)), "nsb_imp_sample: 0 to %d ground-truth keys", NSB_IMP_MAX_GT);
    NSB_REQUIRE(!h_appear || (appear_table && n_appear >= 1), "nsb_imp_sample: h_appear without an appearance table");
    ImpGt gt;
    memset(&gt, 0, sizeof(gt));
    gt.n = n_gt;
    for (int k = 0; k < n_gt; ++k) {
        NSB_REQUIRE(gt_out[k] && gt_row_bytes[k] >= 1, "nsb_imp_sample: ground-truth key %d: NULL output or empty row", k);
        gt.row_bytes[k] = gt_row_bytes[k];
        gt.dst[k] = (uint8_t *)gt_out[k];
    }
    k_imp_sample<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(table, cam, rng, n, n_uniform, res_y, res_x, 1.0f / (float)res_y, 1.0f / (float)res_x,
                                                           torch_rand_grid_cap(), gt, appear_table, n_appear, h_appear, fidx, xy, pidx, dirs,
                                                           rng_next);
    return check_launch("nsb_imp_sample");
}

extern "C" int nsb_error_map_update(float *error_map, int32_t *last, int64_t n_images, const int64_t *table, const int64_t *cam, int32_t res_y,
                                    int32_t res_x, const int64_t *fidx, const float *xy, const float *val, int64_t n, int32_t *flag, const int64_t *skip,
                                    void *stream) {
    NSB_REQUIRE(n_images >= 1 && res_y >= 2 && res_x >= 2 && n >= 0 && n < ((int64_t)1 << 31), "nsb_error_map_update: bad size");
    NSB_REQUIRE(flag && (table ? cam != nullptr : (error_map && last)) && (n == 0 || (fidx && xy && val)), "nsb_error_map_update: NULL argument");
    if (n == 0) return 0;
    k_err_mark<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(error_map, last, n_images, table, cam, fidx, xy, val, n, res_y, res_x, flag, skip);
    if (check_launch("nsb_error_map_update")) return 1;
    k_err_apply<<<wave_grid(n_images * res_y * res_x, 256, 8), 256, 0, STREAM>>>(error_map, last, n_images, table, cam, fidx, xy, val, res_y, res_x,
                                                                                   skip);
    return check_launch("nsb_error_map_update");
}
