// Building blocks shared by the wgmma fused kernels (fused_tc.cu, color_tc.cu): tile constants, the per-thread
// LoTD gather that writes straight into a core-matrix A tile, point loading and W1 staging.
#pragma once
#include "lotd_device.cuh"
#include "tc_util.cuh"

namespace nsb {

struct DecoderDevTC {
    const __half *W1, *b1, *W2, *b2;
    int width;
    float beta;
};

// accel.collect_samples fused into the query kernels (see nsb_occ_collect): xs is the point in [0,1]^3 table space (clamped: the
// voxel index is the same as for the unclamped point), sdf the fp16-valued result.
struct OccCollect {
    float *pcl;
    int rx, ry, rz;
    float inv_s;
};
__device__ __forceinline__ float r16(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ void occ_collect_point(const OccCollect &oc, const float (&xs)[3], float sdf) {
    const int ix = min(max((int)__fmul_rn(xs[0], (float)oc.rx), 0), oc.rx - 1);
    const int iy = min(max((int)__fmul_rn(xs[1], (float)oc.ry), 0), oc.ry - 1);
    const int iz = min(max((int)__fmul_rn(xs[2], (float)oc.rz), 0), oc.rz - 1);
    // (1. / cosh((inv_s * x / 2.).clamp(-20, 20))) ** 2 on a half tensor: every op rounds to fp16 (maths/common.py:122-133)
    const float a = fminf(fmaxf(r16(r16(__fmul_rn(sdf, oc.inv_s)) * 0.5f), -20.f), 20.f);
    const float r = r16(__fdiv_rn(1.f, r16(coshf(a))));
    const float v = r16(__fmul_rn(r, r));
    if (v > 0.f) atomicMax(reinterpret_cast<int *>(oc.pcl) + ((ix * oc.ry + iy) * oc.rz + iz), __float_as_int(v));   // v >= 0: int order == float order
}

constexpr int kTile = 128;
constexpr int NF = 32, HW = 64;           // features, hidden width (zero padded to 64)

// the 16 levels of one point -> row `r` of a chunk-major [R x >=32] fp16 tile (4 bytes per level)
// U levels per loop trip: the 8 U corner loads of a trip are independent, so U = 2 doubles the loads in flight per thread (the
// latency-bound backward kernels run at 8-16 warps / SM); full unrolling is avoided on purpose (instruction cache, see fused_tc.cu).
template <int R, int U = 2, bool PAIRED = false>
__device__ __forceinline__ void gather_row_to_tile(const PLMeta &m, const __half *__restrict__ grid, const float (&xs)[3],
                                                   int max_level, uint8_t *tile, int r) {
#pragma unroll 1
    for (uint32_t p0 = 0; p0 < 16; p0 += U) {
        uint32_t cell[U][8];
        float w[U][8];
        uint32_t packed[U];
#pragma unroll
        for (int u = 0; u < U; ++u) level_cells3(m, p0 + u, xs, cell[u], w[u]);
#pragma unroll
        for (int u = 0; u < U; ++u)
            packed[u] = PAIRED ? level_feat2_cells_paired(level_cells_ptr(m, p0 + u, grid), cell[u], w[u], (m.is_hash >> (p0 + u)) & 1u)
                               : level_feat2_cells(level_cells_ptr(m, p0 + u, grid), cell[u], w[u]);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t p = p0 + u;
            *reinterpret_cast<uint32_t *>(tile + (p >> 2) * (R * 16) + r * 16 + (p & 3) * 4) = ((int)m.level[p] <= max_level) ? packed[u] : 0u;
        }
    }
}

__device__ __forceinline__ void load_point(bool from_rays, const float *__restrict__ x, const float *__restrict__ rays_o,
                                           const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
                                           const float *__restrict__ t, int64_t i, bool valid, float (&xs)[3]) {
    xs[0] = xs[1] = xs[2] = 0.f;
    if (valid) {
        if (from_rays) {
            const int64_t r = ridx ? ridx[i] : i;
            const float tt = t[i];
#pragma unroll
            for (int d = 0; d < 3; ++d) xs[d] = __fmaf_rn(rays_d[r * 3 + d], tt, rays_o[r * 3 + d]);
        } else {
#pragma unroll
            for (int d = 0; d < 3; ++d) xs[d] = x[i * 3 + d];
        }
    }
    // network space [-1,1] -> table space [0,1] (lotd_encoding.py:165), clamp (lotd.py:60)
#pragma unroll
    for (int d = 0; d < 3; ++d) xs[d] = fminf(fmaxf(__fmaf_rn(xs[d], 0.5f, 0.5f), 1.0e-6f), 1.f - 1.0e-6f);
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

// W1 [width x 32] (fp16, row-major) -> chunk-major [64 x 32] B tile, rows >= width zero
__device__ __forceinline__ void stage_W1(const DecoderDevTC &dec, uint8_t *sB, int tid) {
    for (int e = tid; e < HW * (NF / 8); e += kTile) {
        const int j = e % HW, c = e / HW;
        uint4 q = make_uint4(0, 0, 0, 0);
        if (j < dec.width) q = *reinterpret_cast<const uint4 *>(dec.W1 + j * NF + c * 8);
        *reinterpret_cast<uint4 *>(sB + c * (HW * 16) + j * 16) = q;
    }
}

// ---- one 128-point tile of the fused SDF query: gather -> wgmma -> SFU epilogue (used by k_fused_sdf_tc and by the per-ray kernels)
struct SdfTile {
    const PLMeta &m;
    const __half *grid;
    int max_level;
    uint8_t *sA;
    uint32_t a_addr, b_addr;
    float *srow;                           // [kTile] shared: the sdf of each row, handed from the fragment owners to the row's thread
    const float *sb1, *sW2;
    float sb2;
    SoftplusK spk;
};

// all 128 threads: my point's table coordinates -> my sdf (fp16-rounded, as fp32).  Ends with the CTA barrier that frees the tile.
// The epilogue runs on the accumulator fragments: each lane folds its 16 of a row's 64 hidden units, the quad sums the four parts
// in a fixed order (the same for every row, so a point's sdf does not depend on where it sits in the tile).
template <bool FAST_SP, int UNROLL, bool PAIRED>
__device__ __forceinline__ float sdf_of_tile(const SdfTile &c, const float (&xs)[3], int tid) {
    gather_row_to_tile<kTile, UNROLL, PAIRED>(c.m, c.grid, xs, c.max_level, c.sA, tid);
    tc::fence_async_smem();                // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();
    float z[2][HW / 2];
    tc::mma_m128<HW, 0, 0, NF / 16>(z, tc::kmajor(c.a_addr, kTile), tc::kmajor(c.b_addr, HW), false);
    const int lane = tid & 31, q = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float out = 0.f;
#pragma unroll
            for (int ch = 0; ch < HW / 8; ++ch)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int col = ch * 8 + 2 * q + j;
                    const float zz = __half2float(__float2half_rn(z[h][4 * ch + 2 * i + j] + c.sb1[col]));
                    float sp;
                    if (FAST_SP) sp = softplus_a(zz, c.spk);
                    else { const float zb = zz * c.spk.beta; sp = zb > 20.f ? zz : log1pf(expf(zb)) * (1.f / c.spk.beta); }
                    out = fmaf(__half2float(__float2half_rn(sp)), c.sW2[col], out);
                }
            out += __shfl_xor_sync(0xffffffffu, out, 1);
            out += __shfl_xor_sync(0xffffffffu, out, 2);
            if (q == 0) c.srow[h * 64 + (tid >> 5) * 16 + (lane >> 2) + 8 * i] = out;
        }
    __syncthreads();
    return __half2float(__float2half_rn(c.srow[tid] + c.sb2));
}

}  // namespace nsb
