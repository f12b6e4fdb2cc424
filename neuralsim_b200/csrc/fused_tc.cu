// Fused forward_sdf and its backward with the decoder GEMMs on the Hopper tensor cores (wgmma), sm_90a.
//
// One CTA = 128 threads = one warpgroup = one tile of 128 points; thread r owns point r for the gather and the scatter:
//   gather   thread r walks the 16 LoTD levels of its point (8 corner loads each); every level's two fp16 features go
//            straight into its row of the A tile in shared memory (core-matrix layout of tc_util.cuh)
//   MMA      the warpgroup issues wgmma (M=64, N=64, K=16) x2 per 64-row half: Z[128 x 64] (fp32, registers) = H[128 x 32] . W1^T
//   epilogue bias + Softplus(beta) with the autocast rounding points on the accumulator fragments, the 64 -> 1 layer as a
//            dot product per row (16 hidden units per lane, summed over the lane quad) -> sdf[r]
// The loop over levels is rolled on purpose (instruction cache: a fully unrolled gather is several thousand instructions).
// W1 is staged once per persistent CTA.  Numerics: the fp16 rounding points of the reference's autocast graph (DESIGN.md).
#include <stdlib.h>

#include "fused_tc_common.cuh"

namespace nsb {

// MODE 0: points x[n,3];  MODE 1: x = o[ridx[i]] + d[ridx[i]] t[i] in the given (ray-major) order;
// MODE 2: the same packed samples traversed RAY-TILED: a tile = 32 consecutive packs (rays) x 4 consecutive samples, lane = ray,
//         warp = sample ordinal.  For coherent rays (an image) the 32 lanes of a gather instruction then sit in neighbouring
//         cells -> few 128 B lines per request; the L1 tag stage is what bounds this kernel.  sdf is written to the packed slot, so
//         nothing downstream changes.  Incoherent rays (random training pixels) keep MODE 1: locality along the ray.
template <int MODE, bool FAST_SP = false, int UNROLL = 2, bool PAIRED = false>
__global__ void __launch_bounds__(kTile)
k_fused_sdf_tc(const PLMeta m, const __half *__restrict__ grid, const DecoderDevTC dec, const float *__restrict__ x,
               const float *__restrict__ rays_o, const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
               const float *__restrict__ t, int64_t n, int max_level, float *__restrict__ sdf, const int64_t *__restrict__ pack_infos,
               const int64_t *__restrict__ pack_ray, int64_t n_packs, const OccCollect oc, const int64_t *__restrict__ n_dev) {
    if (MODE == 2) n_packs = eff_n(n_packs, n_dev); else n = eff_n(n, n_dev);       // device-resident count (nsb_bind_device_counts)
    __shared__ __align__(128) uint8_t sA[kTile * NF * 2];    // 8 KB : features, chunk-major core-matrix layout
    __shared__ __align__(128) uint8_t sB[HW * NF * 2];       // 4 KB : W1 [64 x 32], same layout
    __shared__ float sb1[HW], sW2[HW], srow[kTile];
    __shared__ float sb2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    stage_W1(dec, sB, tid);
    if (tid < HW) {
        sb1[tid] = tid < dec.width ? __half2float(dec.b1[tid]) : 0.f;
        sW2[tid] = tid < dec.width ? __half2float(dec.W2[tid]) : 0.f;
    }
    if (tid == 0) sb2 = __half2float(dec.b2[0]);
    tc::fence_async_smem();
    __syncthreads();
    const SdfTile ctx{m, grid, max_level, sA, tc::smem_u32(sA), tc::smem_u32(sB), srow, sb1, sW2, sb2, SoftplusK(dec.beta)};

    if (MODE == 2) {
        const int64_t n_groups = (n_packs + 31) / 32;
        for (int64_t g = blockIdx.x; g < n_groups; g += gridDim.x) {
            const int64_t p = g * 32 + lane;
            int64_t first = 0, cnt = 0, ray = 0;
            if (p < n_packs) { first = pack_infos[2 * p]; cnt = pack_infos[2 * p + 1]; ray = pack_ray ? pack_ray[p] : p; }
            float o[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f};
            if (cnt > 0) {
#pragma unroll
                for (int q = 0; q < 3; ++q) { o[q] = rays_o[ray * 3 + q]; d[q] = rays_d[ray * 3 + q]; }
            }
            int max_n = (int)cnt;
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) max_n = max(max_n, __shfl_xor_sync(0xffffffffu, max_n, s));
            for (int k0 = 0; k0 < max_n; k0 += kTile / 32) {
                const int k = k0 + warp;
                const bool valid = k < cnt;
                float xs[3] = {0.f, 0.f, 0.f};
                if (valid) {
                    const float tt = t[first + k];
#pragma unroll
                    for (int q = 0; q < 3; ++q) xs[q] = __fmaf_rn(d[q], tt, o[q]);
                }
#pragma unroll
                for (int q = 0; q < 3; ++q) xs[q] = fminf(fmaxf(__fmaf_rn(xs[q], 0.5f, 0.5f), 1.0e-6f), 1.f - 1.0e-6f);
                const float v = sdf_of_tile<FAST_SP, UNROLL, PAIRED>(ctx, xs, tid);
                if (valid) {
                    sdf[first + k] = v;
                    if (oc.pcl) occ_collect_point(oc, xs, v);
                }
            }
        }
    } else {
        const int64_t n_tiles = (n + kTile - 1) / kTile;
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int64_t i = tile * kTile + tid;
            const bool valid = i < n;
            float xs[3];
            load_point(MODE == 1, x, rays_o, rays_d, ridx, t, i, valid, xs);
            const float v = sdf_of_tile<FAST_SP, UNROLL, PAIRED>(ctx, xs, tid);
            if (valid) {
                sdf[i] = v;
                if (oc.pcl) occ_collect_point(oc, xs, v);
            }
        }
    }
}

// =====================================================================================================================
// Backward of forward_sdf wrt. the LoTD table and the decoder weights, one kernel, nothing saved by the forward.
// Per tile of 128 points (thread r = point r = staged accumulator row r), d = dL/dsdf[r]:
//   recompute  gather -> A tile [H | 1 | 0..];  MMA1: Z = H.W1^T (staged cols 0..63);  z = fp16(Z + b1); s = sigmoid(beta z), a = fp16(softplus)
//   row r of the G tile [128 x 128] fp16 :=  [ dz_0..dz_63 | d*a_0..d*a_63 ],  dz_j = d * w2_j * s_j
//              (the reference rounds grad_z to fp16 at the same place, layers.py autocast backward)
//   MMA2: dH[128 x 32]  = dZ . W1                 A = G cols 0..63 (K-major), B = W1^T tile          -> staged cols 0..31
//   MMA3: X[128 x 40]  += G^T . [H | 1 | 0..]     both operands are the tiles above read MN-major, K = the 128 points;
//              rows 0..63 of X = [ dW1 | db1 ], rows 64..127, column 32 = dW2; accumulated over all tiles of the
//              persistent CTA in staged cols 64..103
//   scatter dH into the fp32 table gradient (8 corners x 16 levels, red.global.add.v2.f32);  db2 via a warp sum.
// =====================================================================================================================
template <bool FROM_RAYS>
__global__ void __launch_bounds__(kTile)
k_sdf_bwd_tc(const PLMeta m, const __half *__restrict__ grid, const DecoderDevTC dec, const float *__restrict__ x,
             const float *__restrict__ rays_o, const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
             const float *__restrict__ t, const float *__restrict__ d_sdf, int64_t n, int max_level, float *__restrict__ d_grid,
             float *__restrict__ d_W1, float *__restrict__ d_b1, float *__restrict__ d_W2, float *__restrict__ d_b2,
             const int64_t *__restrict__ keep, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    constexpr int NX = 40, GW = 128;                          // NX: features + [1,0,..] chunk; GW: dz | d*a
    constexpr int kCols = HW + NX, kS = tc::acc_stride(kCols);  // staged accumulators: Z / dH in cols 0..63, X in cols 64..103
    extern __shared__ uint8_t dyn_smem[];                     // 104 KB of tiles and staged accumulators (> the 48 KB static limit)
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 127) & ~uintptr_t(127));
    uint8_t *sA = tiles;                                      // 10 KB : [H | 1 | 0..]
    uint8_t *sG = sA + kTile * NX * 2;                        // 32 KB : [dz | d*a]
    uint8_t *sB = sG + kTile * GW * 2;                        //  4 KB : W1   [64 x 32]  (B of MMA1)
    uint8_t *sBT = sB + HW * NF * 2;                          //  4 KB : W1^T [32 x 64]  (B of MMA2)
    float *acc = reinterpret_cast<float *>(sBT + NF * HW * 2);   // 54 KB : [128 x kS] fp32
    __shared__ float sb1[HW], sW2[HW];
    __shared__ float sdb2;

    const int tid = threadIdx.x, lane = tid & 31;
    stage_W1(dec, sB, tid);
    for (int e = tid; e < NF * HW; e += kTile) {              // W1^T: row = feature k, col = hidden j
        const int k = e % NF, j = e / NF;
        const __half v = j < dec.width ? dec.W1[j * NF + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sBT + (j / 8) * (NF * 16) + k * 16 + (j % 8) * 2) = v;
    }
    if (tid < HW) {
        sb1[tid] = tid < dec.width ? __half2float(dec.b1[tid]) : 0.f;
        sW2[tid] = tid < dec.width ? __half2float(dec.W2[tid]) : 0.f;
    }
    *reinterpret_cast<uint4 *>(sA + 4 * (kTile * 16) + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);   // constant chunk: [1,0,..]
    for (int c = HW; c < kCols; ++c) acc[tid * kS + c] = 0.f;
    if (tid == 0) sdb2 = 0.f;
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t a_addr = tc::smem_u32(sA), g_addr = tc::smem_u32(sG), b_addr = tc::smem_u32(sB), bt_addr = tc::smem_u32(sBT);
    const SoftplusK spk(dec.beta);
    bool first_tile = true;

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i_ = tile * kTile + tid;
        const bool valid = i_ < n;
        const int64_t i = (valid && keep) ? keep[i_] : i_;        // optional index list: the samples with a non-zero cotangent
        float xs[3];
        load_point(FROM_RAYS, x, rays_o, rays_d, ridx, t, i, valid, xs);
        const float dd = valid ? d_sdf[i] : 0.f;
        gather_row_to_tile<kTile>(m, grid, xs, max_level, sA, tid);
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<HW, 0, 0, NF / 16>(acc, kS, 0, tc::kmajor(a_addr, kTile), tc::kmajor(b_addr, HW), false);   // Z = H . W1^T
        __syncthreads();
        // ---- my G row: dz (chunks 0..7) and d*a (chunks 8..15)
#pragma unroll 1
        for (int c = 0; c < HW / 8; ++c) {
            float z[8], dz[8], da[8];
            tc::acc_ld8(acc, kS, tid, c * 8, z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float zz = __half2float(__float2half_rn(z[j] + sb1[c * 8 + j]));
                float a, s;
                softplus_as(zz, spk, a, s);
                da[j] = dd * __half2float(__float2half_rn(a));
                dz[j] = dd * sW2[c * 8 + j] * s;
            }
            *reinterpret_cast<uint4 *>(sG + c * (kTile * 16) + tid * 16) = tc::pack8_f16(dz);
            *reinterpret_cast<uint4 *>(sG + (8 + c) * (kTile * 16) + tid * 16) = tc::pack8_f16(da);
        }
        tc::fence_async_smem();
        __syncthreads();                                         // every thread has read Z and written its G row
        tc::mma_to_rows<NF, 0, 0, HW / 16>(acc, kS, 0, tc::kmajor(g_addr, kTile), tc::kmajor(bt_addr, NF), false);          // dH = dZ . W1 : K = 64 hidden
        tc::mma_to_rows<NX, 1, 1, kTile / 16>(acc, kS, HW, tc::mnmajor(g_addr, kTile), tc::mnmajor(a_addr, kTile), true);   // X += G^T . [H|1] : K = 128 points
        first_tile = false;
        const float dsum = warp_sum(dd);
        if (lane == 0 && dsum != 0.f) atomicAdd(&sdb2, dsum);
        __syncthreads();
        // ---- my dH row -> scatter into the table gradient; only the reductions are predicated on "this point carries gradient".
        const bool active = valid && dd != 0.f;
        const bool warp_active = __any_sync(0xffffffffu, active);
#pragma unroll 1
        for (uint32_t g4 = 0; g4 < 4; ++g4) {
            float dh[8];
            tc::acc_ld8(acc, kS, tid, g4 * 8, dh);                  // 4 levels x 2 features
            if (!warp_active) continue;
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if ((int)m.level[p] > max_level) continue;               // uniform
                uint32_t cell[8];
                float w[8], a[8], b[8];
                level_cells3(m, p, xs, cell, w);
                const float g0 = active ? dh[2 * q] : 0.f, g1 = active ? dh[2 * q + 1] : 0.f;
#pragma unroll
                for (int c = 0; c < 8; ++c) { a[c] = g0 * w[c]; b[c] = g1 * w[c]; }
                bool issue = active;
                if (level_mergeable(m, p)) issue = warp_merge_updates(cell_key3(m, p, xs), active, a, b, lane);   // neighbouring samples, same cell
                if (issue) {
                    float2 *gp = level_grad_ptr(m, p, d_grid);
#pragma unroll
                    for (int c = 0; c < 8; ++c) red_add2(gp + cell[c], a[c], b[c]);
                }
            }
        }
        __syncthreads();                                         // tiles + staged rows free for the next iteration
    }
    // ---- flush the CTA's weight-gradient accumulators: X rows 0..63 = [dW1 | db1], rows 64..127 col 32 = dW2
    if (!first_tile) {                                           // uniform per CTA
#pragma unroll 1
        for (int c = 0; c < NF / 8; ++c) {
            float r[8];
            tc::acc_ld8(acc, kS, tid, HW + c * 8, r);
            if (tid < dec.width) {
#pragma unroll
                for (int k = 0; k < 8; ++k) atomicAdd(d_W1 + tid * NF + c * 8 + k, r[k]);
            }
        }
        float r1[8];
        tc::acc_ld8(acc, kS, tid, HW + 32, r1);
        if (tid < HW) { if (tid < dec.width) atomicAdd(d_b1 + tid, r1[0]); }
        else if (tid - HW < dec.width) atomicAdd(d_W2 + (tid - HW), r1[0]);
        if (tid == 0) atomicAdd(d_b2, sdb2);
    }
}

}  // namespace nsb

using namespace nsb;

// CTAs of k_fused_sdf_tc per SM in the persistent grid.  5 would fit (90-101 registers, ~13 KB of shared memory), but the gather
// is L1-bound and more warps gathering at once evict each other's lines: on an H100 (NVIDIA H100 80GB HBM3, 700 W) the boundary
// query of an 800x600 frame took 5.8 ms per launch at 4 CTAs / SM, 7.3-7.4 ms at 5 and 6.5 ms at 6 (bench.py, NSB_SDF_CTAS, alternated).
constexpr int kSdfCtasPerSM = 4;

static inline unsigned persistent_grid(int64_t n, int ctas_per_sm) {
    const int64_t n_tiles = (n + kTile - 1) / kTile;
    const int64_t wave = (int64_t)sm_count() * ctas_per_sm;
    return (unsigned)(n_tiles < wave ? n_tiles : wave);
}

template <int MODE>
static void launch_sdf(int variant, unsigned grid, cudaStream_t s, const PLMeta &m, const __half *g, const DecoderDevTC &d, const float *x, const float *ro,
                       const float *rd, const int64_t *ridx, const float *t, int64_t n, int ml, float *sdf, const int64_t *pi, const int64_t *pr, int64_t np,
                       const OccCollect &oc, const int64_t *nd) {
    // default (variant 1): SFU softplus, two levels per gather trip (one level per trip thrashes L1 in ray-major order).
    // variants: 0 libm / 2 levels per trip, 1 SFU / 2, 2 libm / 1, 3 SFU / 1, 4 SFU / 2 + paired corner loads (experiment, lotd_device.cuh)
    if (variant < 0) variant = 1;                      // SFU softplus, two levels per trip
    if (variant == 1) k_fused_sdf_tc<MODE, true, 2><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);
    else if (variant == 2) k_fused_sdf_tc<MODE, false, 1><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);
    else if (variant == 3) k_fused_sdf_tc<MODE, true, 1><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);
    else if (variant == 5) k_fused_sdf_tc<MODE, true, 4><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);   // experiment: four levels (32 loads) per trip
    else if (variant == 4 && plmeta_pairable(m, g)) k_fused_sdf_tc<MODE, true, 2, true><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);   // experiment: paired corner loads
    else k_fused_sdf_tc<MODE, false, 2><<<grid, kTile, 0, s>>>(m, g, d, x, ro, rd, ridx, t, n, ml, sdf, pi, pr, np, oc, nd);
}

// mode 0: x[n,3];  1: (rays_o, rays_d, ridx, t)[n];  2: ray-tiled packs (pack_infos[n_packs,2], pack_ray[n_packs] or NULL, t, sdf packed)
extern "C" int nsb_fused_sdf_tc_launch(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                       const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                                       int32_t max_level, float *sdf, void *stream, int mode, const int64_t *pack_infos,
                                       const int64_t *pack_ray, int64_t n_packs, const nsb_occ_collect *collect) {
    const DevCounts dn = take_counts();
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    NSB_REQUIRE(m.n_pseudo == 16 && m.F == 2 && m.D == 3 && plmeta_two_feature_cells(m), "nsb_fused_sdf (tensor-core): built for 16 x 2 LoTD features in 3-D");
    NSB_REQUIRE(dec->width >= 1 && dec->width <= 64, "nsb_fused_sdf (tensor-core): decoder width must be <= 64");
    DecoderDevTC d{(const __half *)dec->W1, (const __half *)dec->b1, (const __half *)dec->W2, (const __half *)dec->b2, dec->width,
                   dec->beta};
    // NSB_SDF_VARIANT / NSB_SDF_CTAS: profiling switches (profiles/ab_gather.py); see launch_sdf
    // read per call on purpose: profiles/ab_gather.py flips them between launches (two getenv of short names, ~50 ns)
    const char *ev = getenv("NSB_SDF_VARIANT"), *ec = getenv("NSB_SDF_CTAS");
    const int variant = ev ? atoi(ev) : -1;
    const int ctas = ec ? atoi(ec) : kSdfCtasPerSM;
    cudaStream_t s = (cudaStream_t)stream;
    const int ml = max_level < 0 ? -1 : max_level;
    const __half *g = (const __half *)params_half;
    OccCollect oc{nullptr, 1, 1, 1, 0.f};
    if (collect && collect->grid_pcl) oc = OccCollect{collect->grid_pcl, collect->res[0], collect->res[1], collect->res[2], collect->inv_s};
    if (mode == 2) {
        const int64_t groups = (n_packs + 31) / 32, wave = (int64_t)sm_count() * ctas;
        launch_sdf<2>(variant, (unsigned)(groups < wave ? groups : wave), s, m, g, d, nullptr, rays_o, rays_d, nullptr, t, n, ml, sdf, pack_infos, pack_ray, n_packs, oc, dn.a);
    } else if (mode == 1) launch_sdf<1>(variant, persistent_grid(n, ctas), s, m, g, d, nullptr, rays_o, rays_d, ridx, t, n, ml, sdf, nullptr, nullptr, 0, oc, dn.a);
    else launch_sdf<0>(variant, persistent_grid(n, ctas), s, m, g, d, x, nullptr, nullptr, nullptr, nullptr, n, ml, sdf, nullptr, nullptr, 0, oc, dn.a);
    return check_launch("nsb_fused_sdf(tc)");
}

extern "C" int nsb_fused_sdf_bwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                 const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf,
                                 int64_t n, int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2,
                                 void *stream) {
    return nsb_fused_sdf_bwd_indexed(meta, params_half, dec, x, rays_o, rays_d, ridx, t, d_sdf, nullptr, n, max_level, d_grid, d_W1, d_b1, d_W2, d_b2,
                                     stream);
}

extern "C" int nsb_fused_sdf_bwd_indexed(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                         const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf,
                                         const int64_t *keep, int64_t n, int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2,
                                         float *d_b2, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(meta && params_half && dec && d_sdf && d_grid && d_W1 && d_b1 && d_W2 && d_b2, "nsb_fused_sdf_bwd: NULL argument");
    NSB_REQUIRE(x || (rays_o && rays_d && t), "nsb_fused_sdf_bwd: need x or (rays_o, rays_d, t)");
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    NSB_REQUIRE(m.n_pseudo == 16 && m.F == 2 && m.D == 3 && plmeta_two_feature_cells(m), "nsb_fused_sdf_bwd: built for 16 x 2 LoTD features in 3-D");
    NSB_REQUIRE(dec->width >= 1 && dec->width <= 64, "nsb_fused_sdf_bwd: decoder width must be <= 64");
    DecoderDevTC d{(const __half *)dec->W1, (const __half *)dec->b1, (const __half *)dec->W2, (const __half *)dec->b2, dec->width,
                   dec->beta};
    constexpr int kBwdSmem = (128 * 40 + 128 * 128 + 64 * 32 + 32 * 64) * 2 + 128 * tc::acc_stride(64 + 40) * 4 + 128;
    opt_in_smem(k_sdf_bwd_tc<true>, kBwdSmem);
    opt_in_smem(k_sdf_bwd_tc<false>, kBwdSmem);
    const unsigned grid = persistent_grid(n, 2);           // shared memory: 2 x 104 KB per SM
    cudaStream_t s = (cudaStream_t)stream;
    const int ml = max_level < 0 ? -1 : max_level;
    if (x == nullptr) k_sdf_bwd_tc<true><<<grid, kTile, kBwdSmem, s>>>(m, (const __half *)params_half, d, nullptr, rays_o, rays_d, ridx, t, d_sdf, n, ml,
                                                                d_grid, d_W1, d_b1, d_W2, d_b2, keep, dn.a);
    else k_sdf_bwd_tc<false><<<grid, kTile, kBwdSmem, s>>>(m, (const __half *)params_half, d, x, nullptr, nullptr, nullptr, nullptr, d_sdf, n, ml,
                                                    d_grid, d_W1, d_b1, d_W2, d_b2, keep, dn.a);
    return check_launch("nsb_fused_sdf_bwd");
}
