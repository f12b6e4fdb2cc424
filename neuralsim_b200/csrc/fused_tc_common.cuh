// Building blocks shared by the wgmma fused kernels (fused_tc.cu, color_tc.cu, ray_upsample.cu): tile constants, the per-thread
// LoTD gather that writes straight into a core-matrix A tile, point loading, decoder staging and the host-side argument checks.
#pragma once
#include "lotd_device.cuh"
#include "tc_util.cuh"

namespace nsb {

struct DecoderDevTC {
    const __half *W1, *b1, *W2, *b2;
    int width;
    int nh;                                // 2L: the decoder's input width = the row stride of W1 (L = PLMeta::n_pseudo, 1..24)
    float beta;
};

// accel.collect_samples fused into the query kernels (see nsb_occ_collect): xs is the point in [0,1]^3 table space (clamped: the
// voxel index is the same as for the unclamped point), sdf the fp16-valued result.
struct OccCollect {
    float *pcl;
    int rx, ry, rz;
    float inv_s;
};
inline OccCollect occ_collect_of(const nsb_occ_collect *c) {       // NULL or no grid: nothing is collected
    if (c && c->grid_pcl) return OccCollect{c->grid_pcl, c->res[0], c->res[1], c->res[2], c->inv_s};
    return OccCollect{nullptr, 1, 1, 1, 0.f};
}
__device__ __forceinline__ float r16(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ int occ_voxel(const OccCollect &oc, const float (&xs)[3]) {
    const int ix = min(max((int)__fmul_rn(xs[0], (float)oc.rx), 0), oc.rx - 1);
    const int iy = min(max((int)__fmul_rn(xs[1], (float)oc.ry), 0), oc.ry - 1);
    const int iz = min(max((int)__fmul_rn(xs[2], (float)oc.rz), 0), oc.rz - 1);
    return (ix * oc.ry + iy) * oc.rz + iz;
}
__device__ __forceinline__ void occ_collect_voxel(const OccCollect &oc, int voxel, float sdf) {
    // (1. / cosh((inv_s * x / 2.).clamp(-20, 20))) ** 2 on a half tensor: every op rounds to fp16 (maths/common.py:122-133)
    const float a = fminf(fmaxf(r16(r16(__fmul_rn(sdf, oc.inv_s)) * 0.5f), -20.f), 20.f);
    const float r = r16(__fdiv_rn(1.f, r16(coshf(a))));
    const float v = r16(__fmul_rn(r, r));
    if (v > 0.f) atomicMax(reinterpret_cast<int *>(oc.pcl) + voxel, __float_as_int(v));   // v >= 0: int order == float order
}
__device__ __forceinline__ void occ_collect_point(const OccCollect &oc, const float (&xs)[3], float sdf) {
    occ_collect_voxel(oc, occ_voxel(oc, xs), sdf);
}

constexpr int kTile = 128;
constexpr int HW = 64;                    // hidden width (zero padded to 64)
// Feature columns of the A tile (the template parameter NF of every wgmma kernel): 32 for tables of 1..16 two-feature levels, 48 for
// 17..24.  The width follows the table's L, not the active level count, so one instantiation serves every level bound of a schedule.
constexpr int kMaxNarrowLevels = 16, kMaxWideLevels = 24;
inline int feature_cols(uint32_t L) { return L <= (uint32_t)kMaxNarrowLevels ? 32 : 48; }

// The levels a launch uses: 0..max_level of the L = m.n_pseudo levels (make_decoder: pseudo level p is level p), i.e. the prefix of
// clamp(max_level + 1, 0, L) levels.  max_level is the host argument, or -- with a device level bound to the launch (ml_dev,
// nsb_bind_device_max_level) -- the value in device memory, read once at the start of the kernel and clamped to [-1, L-1].  Uniform across
// the CTA.
__device__ __forceinline__ uint32_t active_levels(int max_level, const int32_t *__restrict__ ml_dev, uint32_t L) {
    const int ml = ml_dev ? *ml_dev : max_level;
    return ml < 0 ? 0u : (ml >= (int)L - 1 ? L : (uint32_t)ml + 1u);
}

// the La active levels of one point -> row `r` of a chunk-major [R x >=NF] fp16 tile (4 bytes per level); the feature columns 2La..NF-1
// are written as zeros, so that nothing a previous tile left in shared memory reaches a wgmma (a stale fp16 Inf times a zero weight is
// NaN), and levels >= La are not read: a masked level costs its zero columns, not its 8 corner loads.
// U levels per loop trip: the 8 U corner loads of a trip are independent, so U = 2 doubles the loads in flight per thread (the
// latency-bound backward kernels run at 8-16 warps / SM; one level per trip thrashes L1 in the ray-major order of k_fused_sdf_tc);
// full unrolling is avoided on purpose (instruction cache, see fused_tc.cu).  An odd La ends with one level alone.  p_begin > 0 skips the
// first levels (written by the caller).
template <int R>
__device__ __forceinline__ void put_level_to_tile(uint8_t *tile, int r, uint32_t p, uint32_t v) {
    *reinterpret_cast<uint32_t *>(tile + (p >> 2) * (R * 16) + r * 16 + (p & 3) * 4) = v;
}
template <int R, int NF, int U = 2>
__device__ __forceinline__ void gather_row_to_tile(const PLMeta &m, const __half *__restrict__ grid, const float (&xs)[3],
                                                   uint32_t La, uint8_t *tile, int r, uint32_t p_begin = 0) {
    uint32_t p0 = p_begin;
#pragma unroll 1
    for (; p0 + U <= La; p0 += U) {
        uint32_t cell[U][8];
        float w[U][8];
        uint32_t packed[U];
#pragma unroll
        for (int u = 0; u < U; ++u) level_cells3(m, p0 + u, xs, cell[u], w[u]);
#pragma unroll
        for (int u = 0; u < U; ++u) packed[u] = level_feat2_cells(level_cells_ptr(m, p0 + u, grid), cell[u], w[u]);
#pragma unroll
        for (int u = 0; u < U; ++u) put_level_to_tile<R>(tile, r, p0 + u, packed[u]);
    }
#pragma unroll 1
    for (; p0 < La; ++p0) {
        uint32_t cell[8];
        float w[8];
        level_cells3(m, p0, xs, cell, w);
        put_level_to_tile<R>(tile, r, p0, level_feat2_cells(level_cells_ptr(m, p0, grid), cell, w));
    }
#pragma unroll 1
    for (; p0 < NF / 2; ++p0) put_level_to_tile<R>(tile, r, p0, 0u);
}

// d(y_f)/d(x_d) of one level (both features) from its 8 corner cells as loaded, exactly as k_lotd_fwd<3,2,true,true> computes dy_dx
__device__ __forceinline__ void jacobian_from_raw(const uint32_t (&raw)[8], const float (&fr)[3], const float (&scale)[3], float (&J0)[3],
                                                  float (&J1)[3]) {
    float2 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = __half22float2(*reinterpret_cast<const __half2 *>(&raw[c]));
#pragma unroll
    for (int gd = 0; gd < 3; ++gd) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float ww = scale[gd];
            int left = 0;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int d = k >= gd ? k + 1 : k;
                if (c & (1 << k)) { ww = __fmul_rn(ww, fr[d]); left += 1 << d; }
                else ww = __fmul_rn(ww, __fsub_rn(1.f, fr[d]));
            }
            const int right = left + (1 << gd);
            a0 = __fmaf_rn(ww, __fsub_rn(v[right].x, v[left].x), a0);
            a1 = __fmaf_rn(ww, __fsub_rn(v[right].y, v[left].y), a1);
        }
        J0[gd] = a0;
        J1[gd] = a1;
    }
}

// The input gradient of one level, first order (the encoding's input Hessian is not formed, as on the reference's hot path):
// gx += J0 h0 + J1 h1, with J from the level's 8 corners (loaded here) and (h0, h1) the cotangent of the level's two features.
__device__ __forceinline__ void level_input_grad(const PLMeta &m, uint32_t p, const __half *__restrict__ grid, const uint32_t (&cell)[8],
                                                 const float (&fr)[3], const float (&sc)[3], float h0, float h1, float (&gx)[3]) {
    uint32_t raw[8];
    const uint32_t *lp = level_cells_ptr(m, p, grid);
#pragma unroll
    for (int c = 0; c < 8; ++c) raw[c] = ld_nc_u32(lp + cell[c]);
    float J0[3], J1[3];
    jacobian_from_raw(raw, fr, sc, J0, J1);
#pragma unroll
    for (int d = 0; d < 3; ++d) gx[d] = __fmaf_rn(h1, J1[d], __fmaf_rn(h0, J0[d], gx[d]));
}

// table-space input gradient -> network space: the table sees x / 2 + 1/2.  The encoding clamps that to [1e-6, 1 - 1e-6] inside its op
// and returns the input gradient at the clamped point without masking it (LoTDFunction*, lotd.py), so neither is it masked here.
__device__ __forceinline__ float input_grad_to_net(float g) { return __fmul_rn(g, 0.5f); }

// Where the points of a kernel come from: x[i] (network space), or rays_o/rays_d[ray] + t[i] rays_d[ray] with ray = ridx[i] (or i).
struct PointSrc {
    const float *x, *rays_o, *rays_d, *t;
    const int64_t *ridx;
};

// point i: xn in network space, its ray, xs in table space; zeros for an invalid i
__device__ __forceinline__ void load_point(const PointSrc &ps, bool from_rays, int64_t i, bool valid, float (&xn)[3], float (&xs)[3],
                                           int64_t &ray) {
    xn[0] = xn[1] = xn[2] = 0.f;
    ray = 0;
    if (valid) {
        if (from_rays) {
            ray = ps.ridx ? ps.ridx[i] : i;
            const float tt = ps.t[i];
#pragma unroll
            for (int d = 0; d < 3; ++d) xn[d] = __fmaf_rn(ps.rays_d[ray * 3 + d], tt, ps.rays_o[ray * 3 + d]);
        } else {
#pragma unroll
            for (int d = 0; d < 3; ++d) xn[d] = ps.x[i * 3 + d];
            ray = ps.ridx ? ps.ridx[i] : i;
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) xs[d] = to_table_space(xn[d]);
}
__device__ __forceinline__ void load_point(const PointSrc &ps, bool from_rays, int64_t i, bool valid, float (&xs)[3]) {
    float xn[3];
    int64_t ray;
    load_point(ps, from_rays, i, valid, xn, xs, ray);
}

// Softplus(z; beta) with ATen's threshold (beta z > 20 -> identity) on the SFU: e = 2^(z beta log2 e), a = log2(1 + e) ln2 / beta.
// ex2.approx / lg2.approx are accurate to ~2^-22 relative; the result is rounded to fp16 (2^-11) right after, and the
// absolute error (< 1e-7 / beta) is far below the fp16 spacing at every magnitude, so the fp16 activation differs from the
// expf/log1pf evaluation only in rare round-to-nearest ties (tests: <= 1 fp16 ulp).  13 issue slots per hidden unit instead of ~50.
struct SoftplusK {
    float k, thr, out;                       // beta log2(e), 20 log2(e), ln2 / beta
    float beta;
    __device__ __forceinline__ explicit SoftplusK(float b) : k(b * 1.4426950408889634f), thr(20.f * 1.4426950408889634f), out(0.6931471805599453f / b), beta(b) {}
};
__device__ __forceinline__ float ex2_approx(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float lg2_approx(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

__device__ __forceinline__ float softplus_a(float zz, const SoftplusK &K) {
    const float t = zz * K.k;
    const float e = ex2_approx(t);
    const float a = lg2_approx(1.f + e) * K.out;
    return t > K.thr ? zz : a;
}
// a = softplus, s = its derivative sigmoid(beta z) (1 above the threshold, as ATen's backward)
__device__ __forceinline__ void softplus_as(float zz, const SoftplusK &K, float &a, float &s) {
    const float t = zz * K.k;
    const float e = ex2_approx(t);
    const float d = 1.f + e;
    const bool lin = t > K.thr;
    a = lin ? zz : lg2_approx(d) * K.out;
    s = lin ? 1.f : e * rcp_approx(d);
}

// W1 [width x 2L] (fp16, row-major) -> chunk-major [64 x NF] B tile, rows >= width and columns >= 2L zero
template <int NF>
__device__ __forceinline__ void stage_W1(const DecoderDevTC &dec, uint8_t *sB, int tid) {
    for (int e = tid; e < HW * (NF / 8); e += kTile) {
        const int j = e % HW, c = e / HW;
        __align__(16) __half q[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) q[k] = (j < dec.width && c * 8 + k < dec.nh) ? dec.W1[j * dec.nh + c * 8 + k] : __float2half_rn(0.f);
        *reinterpret_cast<uint4 *>(sB + c * (HW * 16) + j * 16) = *reinterpret_cast<const uint4 *>(q);
    }
}

// W1^T [NF x 64] -> chunk-major B tile (row = feature k, column = hidden j), columns >= width and rows >= 2L zero
template <int NF>
__device__ __forceinline__ void stage_W1T(const DecoderDevTC &dec, uint8_t *sBT, int tid) {
    for (int e = tid; e < NF * HW; e += kTile) {
        const int k = e % NF, j = e / NF;
        const __half v = (j < dec.width && k < dec.nh) ? dec.W1[j * dec.nh + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sBT + (j / 8) * (NF * 16) + k * 16 + (j % 8) * 2) = v;
    }
}

// b1 and W2 (zero past the decoder width) and b2 -> shared memory as fp32.  A kernel that does not read b1 or b2 passes nullptr for it;
// that is decided by the argument's type, because the compiler cannot prove a shared-memory address non-null.
template <typename B1, typename B2>
__device__ __forceinline__ void stage_decoder_vectors(const DecoderDevTC &dec, B1 sb1, float *sW2, B2 sb2, int tid) {
    constexpr bool kB1 = !std::is_same<B1, std::nullptr_t>::value, kB2 = !std::is_same<B2, std::nullptr_t>::value;
    if (tid < HW) {
        if constexpr (kB1) sb1[tid] = tid < dec.width ? __half2float(dec.b1[tid]) : 0.f;
        sW2[tid] = tid < dec.width ? __half2float(dec.W2[tid]) : 0.f;
    }
    if constexpr (kB2) {
        if (tid == 0) *sb2 = __half2float(dec.b2[0]);
    }
}

// Per-ray sum of per-point gradient rows (W floats each): the appearance-code rows of k_color_rad_bwd<true, .>, and the ray rows
// [dL/do | dL/dd | dL/dv | 0] of k_color_sdf_bwd<true> and k_sdf_bwd_tc<true, true>.  Row j belongs to ray ridx[keep[j]] (keep NULL:
// ridx[j]; ridx NULL: ray j).  The points of a ray are consecutive (packed samples), so a ray is a run of equal rays.  A warp looks at 32
// rows; for each run that starts among them, in order, the whole warp walks the run 32 rows at a time (lane l adds rows start + l,
// start + l + 32, ...; the run ends at the first row of another ray), reduces the lanes' sums by a fixed butterfly and adds column c < n_out
// once to out.p[c / out.k][ray_map[ray] * out.k + c % out.k] (ray_map NULL: row ray; a NULL output is not written).  One add per ray
// onto the caller's zeros in an order fixed by the run's position: the same bits on every run.  (A ray whose points form several runs --
// unsorted rays -- gets one atomic add per run.)
struct RowSumOut {
    float *p[3];
    int k;                                                     // columns per output
};
template <int W>
__global__ void __launch_bounds__(256)
k_ray_row_sum(const float *__restrict__ rows, const int64_t *__restrict__ ridx, const int64_t *__restrict__ keep, int64_t n, int n_out,
              const int64_t *__restrict__ ray_map, const RowSumOut out, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x / 32);
    auto ray_of = [&](int64_t j) { return ridx[keep ? keep[j] : j]; };
    for (int64_t w = blockIdx.x * (int64_t)(blockDim.x / 32) + threadIdx.x / 32; w * 32 < n; w += n_warps) {   // warp-uniform
        const int64_t i = w * 32 + lane;
        const int64_t ray = i < n ? (ridx ? ray_of(i) : i) : -1;
        uint32_t heads = __ballot_sync(~0u, i < n && (!ridx || i == 0 || ray_of(i - 1) != ray));
        while (heads) {
            const int src = __ffs(heads) - 1;
            heads &= heads - 1;
            const int64_t r = __shfl_sync(~0u, ray, src);
            float acc[W];
#pragma unroll
            for (int k = 0; k < W; ++k) acc[k] = 0.f;
            for (int64_t base = w * 32 + src;; base += 32) {
                const int64_t j = base + lane;
                const bool same = j < n && (ridx ? ray_of(j) == r : j == base);
                const uint32_t stop = ~__ballot_sync(~0u, same);
                const int end = stop ? __ffs(stop) - 1 : 32;        // the run continues in lanes [0, end) of this block
                if (lane < end) {
#pragma unroll
                    for (int q = 0; q < W / 4; ++q) {
                        const float4 a = *reinterpret_cast<const float4 *>(rows + j * W + 4 * q);
                        acc[4 * q] += a.x; acc[4 * q + 1] += a.y; acc[4 * q + 2] += a.z; acc[4 * q + 3] += a.w;
                    }
                }
                if (end < 32) break;
            }
#pragma unroll
            for (int k = 0; k < W; ++k)
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) acc[k] += __shfl_xor_sync(~0u, acc[k], off);
            if (lane < n_out) {
                float v = acc[0];
#pragma unroll
                for (int k = 1; k < W; ++k) v = lane == k ? acc[k] : v;
                const int which = lane / out.k;
                float *o = which == 0 ? out.p[0] : (which == 1 ? out.p[1] : out.p[2]);
                if (o) atomicAdd(o + (ray_map ? ray_map[r] : r) * out.k + (lane - which * out.k), v);
            }
        }
    }
}

// blocks of k_ray_row_sum over n rows: 8 warps of 32 rows per block, at most 2^20 blocks (the warps loop beyond)
inline unsigned row_sum_blocks(int64_t n) {
    const int64_t blocks = (n + 255) / 256;
    return (unsigned)(blocks < (1 << 20) ? blocks : (1 << 20));
}

// Host: the LoTD layout and decoder the wgmma kernels are built for -> their kernel arguments (0, or 2 with the error set).
// L = 1..24 levels of 2 features each in 3-D (feature_cols(L) picks the kernels' tile width); the decoder's W1 is [width x 2L].
inline int make_decoder(const nsb_lotd_meta *meta, const nsb_sdf_decoder *dec, PLMeta *m, DecoderDevTC *d, const char *who) {
    if (make_plmeta(meta, m)) return 2;
    NSB_REQUIRE(m->n_pseudo >= 1 && m->n_pseudo <= (uint32_t)kMaxWideLevels, "%s: built for 1 to %d LoTD levels (got %u)", who, kMaxWideLevels,
                m->n_pseudo);
    NSB_REQUIRE(m->F == 2 && m->D == 3 && m->n_out == 2 * m->n_pseudo && plmeta_two_feature_cells(*m), "%s: built for L x 2 LoTD features in 3-D", who);
    NSB_REQUIRE(plmeta_cell_key_fits(*m), "%s: a level resolution exceeds %u cells per axis (the backward's merge key)", who, 1u << kCellKeyBits);
    for (uint32_t p = 0; p < m->n_pseudo; ++p)        // 2-feature levels: the active levels are a prefix (active_levels)
        NSB_REQUIRE(m->level[p] == p, "%s: pseudo level %u is level %u, not itself", who, p, m->level[p]);
    NSB_REQUIRE(dec->width >= 1 && dec->width <= 64, "%s: decoder width must be <= 64", who);
    *d = DecoderDevTC{(const __half *)dec->W1, (const __half *)dec->b1, (const __half *)dec->W2, (const __half *)dec->b2, dec->width,
                      2 * (int)m->n_pseudo, dec->beta};
    return 0;
}

// ---- one 128-point tile of the fused SDF query: gather -> wgmma -> SFU epilogue (used by k_fused_sdf_tc and by the per-ray kernels)
struct SdfTile {
    const PLMeta &m;
    const __half *grid;
    uint32_t La;                           // active levels (active_levels)
    uint8_t *sA;
    uint32_t a_addr, b_addr;
    float *srow;                           // [kTile] shared: the sdf of each row, handed from the fragment owners to the row's thread
    const float *sb1, *sW2;
    float sb2;
    SoftplusK spk;
};

// The decoder's epilogue on the accumulator fragments Z = H . W1^T of a 128-row tile (warpgroup-collective): out[h][i] = the 64 -> 1
// layer of row 64h + tc::frag_row(i) without b2, in every lane of the row's quad.  Each lane folds its 16 of the row's 64 hidden units,
// the quad sums the four parts in a fixed order (the same for every row, so a point's sdf does not depend on where it sits in the tile).
__device__ __forceinline__ void sdf_rows_of_frags(const float (&z)[2][HW / 2], const float *sb1, const float *sW2, const SoftplusK &spk,
                                                  float (&out)[2][2]) {
    const int q = threadIdx.x & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float o = 0.f;
#pragma unroll
            for (int ch = 0; ch < HW / 8; ++ch)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int col = ch * 8 + 2 * q + j;
                    const float zz = r16(z[h][4 * ch + 2 * i + j] + sb1[col]);
                    o = fmaf(r16(softplus_a(zz, spk)), sW2[col], o);
                }
            o += __shfl_xor_sync(0xffffffffu, o, 1);
            o += __shfl_xor_sync(0xffffffffu, o, 2);
            out[h][i] = o;
        }
}

// all 128 threads: my point's table coordinates -> my sdf (fp16-rounded, as fp32).  Ends with the CTA barrier that frees the tile.
template <int NF>
__device__ __forceinline__ float sdf_of_tile(const SdfTile &c, const float (&xs)[3], int tid) {
    gather_row_to_tile<kTile, NF>(c.m, c.grid, xs, c.La, c.sA, tid);
    tc::fence_async_smem();                // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();
    float z[2][HW / 2];
    tc::mma_m128<HW, 0, 0, NF / 16>(z, tc::kmajor(c.a_addr, kTile), tc::kmajor(c.b_addr, HW), false);
    float out[2][2];
    sdf_rows_of_frags(z, c.sb1, c.sW2, c.spk, out);
    if ((tid & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 2; ++i) c.srow[h * 64 + tc::frag_row(i)] = out[h][i];
    }
    __syncthreads();
    return r16(c.srow[tid] + c.sb2);
}

}  // namespace nsb
