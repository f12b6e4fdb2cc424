// Fused colour / normal query of the NeuS field and its backward (incl. the second-order path through nablas) on the
// Hopper tensor cores (wgmma), sm_90a.  One CTA = 128 threads = one warpgroup = one tile of 128 points, thread r owns
// point r (row r of the accumulators staged in shared memory, tc_util.cuh).  Replaces, for the packed samples that survive compression, the reference's chain
//   LoTDNeuS.forward (lotd_neus.py:141-167) = LoTDSDF.forward_sdf_nablas (lotd_sdf.py:201-257: LoTDFunctionFwdDydx ->
//   decoder -> autograd.grad -> LoTDFunctionBwdDydx) + RadianceNet.forward (mlp_nerf.py:267-289)
// and its autograd backward (LoTDFunctionBwdDydx.backward = lod_bwd_bwd_input, lotd.py:193-268; the autocast MLP
// double-backward) with three kernels:
//
//   k_color_fwd      one gather: h and the per-level Jacobian J from the same corner loads (J kept in registers, never stored)
//                    -> MMA Z=H.W1^T -> z,a,sdf,u=fp16(w2 s) -> MMA g=U.W1 (= dsdf/dh) -> nablas = J^T g -> radiance input row
//                    -> MMA -> relu -> MMA -> relu -> 64->3 -> sigmoid.   Saves the fp16 activation tiles Z, X, Y1, Y2 in core-matrix layout.
//   k_color_rad_bwd  radiance backward from the saved tiles: dZ2, dZ1 (MMA), dh (MMA), weight gradients accumulated in
//                    registers over all tiles of the persistent CTA (MN-major M64 MMAs contracting over the 128 points).
//   k_color_sdf_bwd  gather pass for dg = J.dn, MMA du = dG.W1^T, MMA g = U.W1, dz (softplus'' term + sdf term),
//                    MMA dh = dZ.W1, weight-gradient MMAs, one merged scatter (g (x) second-order weights + dh (x) trilinear
//                    weights) into the fp32 table gradient.
//
// Numerics: the fp16 rounding points of the reference's autocast graph (oracle/nets.py); J and nablas use the exact
// arithmetic of k_lotd_fwd<DYDX> / k_lotd_bwd_input, so nablas is bit-identical to the unfused kernels given the same g.
// Radiance input columns are kept in the internal order [h | x | SH(v) | n | h_appear | 0] (h first, so the h tile IS the
// first NF / 8 chunks of X); weights are permuted when staged / flushed.
// NF (a template parameter of every kernel here) is the width of the h tile: 32 for tables of 1..16 levels, 48 for 17..24
// (feature_cols); the X tile is then NF + 32 columns wide: 64, or 80.
#include "fused_tc_common.cuh"
#include "sh_device.cuh"

namespace nsb {

struct ColorNetDev {
    DecoderDevTC dec;                                   // sdf decoder: [width x 2L], [width], [width], [1]
    const __half *R1, *rb1, *R2, *rb2, *R3, *rb3;       // radiance net: [rw x rin], [rw], [rw x rw], [rw], [3 x rw], [3]
    int rw, rin, n_appear;
    float fac[3];                                       // sdf_scale / radius3d_original per axis
};

constexpr int XW = 64;                                  // padded hidden width of the radiance net
constexpr int kTileBytes = kTile * XW * 2;              // one saved activation tile (Z, Y1, Y2; X at NF = 32): 16 KB
constexpr int kChunk = kTile * 16;                      // bytes of one 8-column chunk of a 128-row tile
template <int NF>
constexpr int x_cols() { return NF + 32; }              // the radiance input tile [h(NF) | x sh n h_appear 0 (32)]
template <int NF>
constexpr int x_tile_bytes() { return kTile * x_cols<NF>() * 2; }   // one saved X tile: 16 KB, or 20 KB at NF = 48
constexpr int kXVCols = 32;                             // the ray-gradient columns [x | SH | 0] of k_color_rad_bwd<., true>: 19 used

// internal radiance-input column -> reference column (or -1 for padding); the reference input is [x(3), SH(16), n(3), h(nh), h_appear]
// with nh = 2L h columns, so rad_in = 22 + nh + n_appear, and the internal h columns nh..hc-1 are padding (hc = NF, the h tile's width;
// the columns after it sit hc - 32 further right than in the 32-column layout)
__host__ __device__ inline int ref_col(int k, int n_appear, int nh, int hc = 32) {
    if (k < hc) return k < nh ? 22 + k : -1;
    k -= hc - 32;
    if (k < 35) return k - 32;
    if (k < 51) return 3 + (k - 35);
    if (k < 54) return 19 + (k - 51);
    if (k < 54 + n_appear) return 22 + nh + (k - 54);
    return -1;
}


__device__ __forceinline__ void level_jacobian(const PLMeta &m, uint32_t p, const float (&xs)[3], const __half *__restrict__ grid,
                                               float (&J0)[3], float (&J1)[3]) {
    uint32_t cell[8], raw[8];
    float w[8], fr[3], scale[3];
    level_cells3(m, p, xs, cell, w, fr, scale);
    const uint32_t *lp = level_cells_ptr(m, p, grid);
#pragma unroll
    for (int c = 0; c < 8; ++c) raw[c] = ld_nc_u32(lp + cell[c]);
    jacobian_from_raw(raw, fr, scale, J0, J1);
}

__device__ __forceinline__ void unpack8(const uint4 &q, float (&v)[8]) {
    const __half2 *h = reinterpret_cast<const __half2 *>(&q);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}

// The colour kernels run at 1-2 CTAs per SM (shared-memory bound), i.e. 4-8 warps: their gathers live on loads in flight PER THREAD, and
// registers are plentiful -> four levels (32 corner loads) per gather trip instead of the two of k_fused_sdf_tc (which runs 24 warps per SM).
constexpr int kColorGatherU = 4;

// The one table gather of the colour forward: each level's 8 corners are loaded once and give both its fp16 feature pair (-> row r of the
// chunk-major X tile, zero from level La on, as gather_row_to_tile writes it) and its Jacobian J0[p], J1[p], which stay in registers until
// g = U.W1 is known.  Fully unrolled, unlike the rolled gathers of the 16-24-warp kernels, so that J (96 floats) is statically indexed:
// k_color_fwd runs 8 warps per SM and has no min-blocks bound, so it may use the registers.  The corner loads of kColorGatherU levels are
// issued before any of them is consumed.  Only the La active levels (active_levels) are loaded: levels p >= La load nothing and write zero
// columns; a trip that starts at or above La computes nothing, and in the trip that La cuts the levels >= La see zero corners (their J is
// zero and never read: nablas stops at La).
__device__ __forceinline__ void gather_row_and_jacobian(const PLMeta &m, const __half *__restrict__ grid, const float (&xs)[3], uint32_t La,
                                                        uint8_t *tile, int r, float (&J0)[16][3], float (&J1)[16][3]) {
#pragma unroll
    for (uint32_t p0 = 0; p0 < 16; p0 += kColorGatherU) {
        if (p0 >= La) {                                        // uniform
#pragma unroll
            for (int u = 0; u < kColorGatherU; ++u) put_level_to_tile<kTile>(tile, r, p0 + u, 0u);
            continue;
        }
        uint32_t cell[kColorGatherU][8], raw[kColorGatherU][8];
        float w[kColorGatherU][8], fr[kColorGatherU][3], sc[kColorGatherU][3];
#pragma unroll
        for (int u = 0; u < kColorGatherU; ++u) level_cells3(m, p0 + u, xs, cell[u], w[u], fr[u], sc[u]);
#pragma unroll
        for (int u = 0; u < kColorGatherU; ++u) {
            const uint32_t *lp = level_cells_ptr(m, p0 + u, grid);
#pragma unroll
            for (int c = 0; c < 8; ++c) raw[u][c] = p0 + u < La ? ld_nc_u32(lp + cell[u][c]) : 0u;
        }
#pragma unroll
        for (int u = 0; u < kColorGatherU; ++u) {
            const uint32_t p = p0 + u;
            const uint32_t packed = feat2_from_raw(raw[u], w[u]);
            put_level_to_tile<kTile>(tile, r, p, p < La ? packed : 0u);
            jacobian_from_raw(raw[u], fr[u], sc[u], J0[p], J1[p]);
        }
    }
}

// Resident CTAs per SM of the persistent grids of both colour backward kernels.  Their weight-gradient sums stay in registers (mma_m64)
// and only the tiles the MMAs read live in shared memory (about 101 and 97 KB per CTA), so two CTAs fit an SM and the gather, MMA and
// scatter phases of one overlap those of the other.  The launcher checks the occupancy calculator agrees (require_ctas_per_sm).
constexpr int kColorBwdCtasPerSM = 2;

// Resident CTAs per SM of the geometry-only forward (k_color_fwd<false>): without R1 / R2 and with the X tile cut to its h half it needs
// about 67 KB of shared memory instead of 91 KB, which would fit three CTAs on an SM.  The launcher asks for the shared-memory carve-out of
// exactly this many CTAs, because what is not carved out is L1, which the table gathers (ld.global.nc) hit: three CTAs leave about 28 KB of
// L1, two about 92 KB.  Three CTAs measured 2x slower (DESIGN.md §6), and with the Jacobian held in registers through the MMAs (about 250
// registers per thread) the register file holds two.
constexpr int kColorGeoCtasPerSM = 2;

// ===================================================================================================================== forward
// kRad = false is the geometry-only form (models without a radiance net, and rays that render no rgb): it stops after nablas, writes the
// Z tile and the h part of the X tile (at the X tile's stride, so k_color_sdf_bwd reads them unchanged) and never reads the
// radiance weights, view_dirs, h_appear, rgb_out, Y1t or Y2t.
// NF = 48: levels 0..15 are gathered with their Jacobian in registers (gather_row_and_jacobian), levels 16..La-1 by the plain gather;
// once g is known, their Jacobian is formed from a second load of the same 8 corners (L1 / L2 hits) and added in level order, so
// nablas keeps the arithmetic of k_lotd_bwd_input.
template <bool kRad, int NF>
__global__ void __launch_bounds__(kTile)
k_color_fwd(const PLMeta m, const __half *__restrict__ grid, const ColorNetDev net, const PointSrc ps, const float *__restrict__ view_dirs,
            const float *__restrict__ h_appear, int64_t n, int max_level, float *__restrict__ sdf_out, float *__restrict__ nab_out,
            float *__restrict__ rgb_out, float *__restrict__ x_out, uint8_t *__restrict__ Zt, uint8_t *__restrict__ Xt,
            uint8_t *__restrict__ Y1t, uint8_t *__restrict__ Y2t, const OccCollect oc, const int64_t *__restrict__ n_dev,
            const int32_t *__restrict__ ml_dev) {
    n = eff_n(n, n_dev);
    const uint32_t La = active_levels(max_level, ml_dev, m.n_pseudo);
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    constexpr int XC = x_cols<NF>();
    uint8_t *sX = tiles;                                       // 16 KB (NF = 48: 20 KB) [h | x sh n ha 0] (geometry-only: the h part)
    uint8_t *sU = sX + (kRad ? x_tile_bytes<NF>() : (NF / 8) * kChunk);   // 16 KB u, later relu(y1)
    uint8_t *sW1 = sU + kTileBytes;                            //  4 KB (6 KB) W1   [64 x NF]
    uint8_t *sW1T = sW1 + HW * NF * 2;                         //  4 KB (6 KB) W1^T [NF x 64]
    uint8_t *sR1 = sW1T + HW * NF * 2;                         //  8 KB (10 KB) R1 [64 x XC] (internal column order; radiance only)
    uint8_t *sR2 = sR1 + XW * XC * 2;                          //  8 KB R2 [64 x 64] (radiance only)
    constexpr int kS = tc::acc_stride(64);
    float *acc = reinterpret_cast<float *>(kRad ? sR2 + XW * XW * 2 : sR1);   // 34 KB staged accumulator rows (Z, g, Y1, Y2 in turn)
    __shared__ float sb1[HW], sW2[HW], srb1[XW], srb2[XW], sR3[3][XW];
    __shared__ float sb2, srb3[3];

    const int tid = threadIdx.x;
    stage_W1<NF>(net.dec, sW1, tid);
    stage_W1T<NF>(net.dec, sW1T, tid);
    if constexpr (kRad) {
        for (int e = tid; e < XW * XC; e += kTile) {
            const int j = e % XW, k = e / XW;                  // (out j, in k)
            const int rc = ref_col(k, net.n_appear, net.dec.nh, NF);
            const __half v1 = (j < net.rw && rc >= 0) ? net.R1[j * net.rin + rc] : __float2half_rn(0.f);
            *reinterpret_cast<__half *>(sR1 + (k / 8) * (XW * 16) + j * 16 + (k % 8) * 2) = v1;
            if (k < XW) {
                const __half v2 = (j < net.rw && k < net.rw) ? net.R2[j * net.rw + k] : __float2half_rn(0.f);
                *reinterpret_cast<__half *>(sR2 + (k / 8) * (XW * 16) + j * 16 + (k % 8) * 2) = v2;
            }
        }
    }
    stage_decoder_vectors(net.dec, sb1, sW2, &sb2, tid);
    if constexpr (kRad) {
        if (tid < XW) {
            srb1[tid] = tid < net.rw ? __half2float(net.rb1[tid]) : 0.f;
            srb2[tid] = tid < net.rw ? __half2float(net.rb2[tid]) : 0.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) sR3[k][tid] = tid < net.rw ? __half2float(net.R3[k * net.rw + tid]) : 0.f;
        }
        if (tid == 0) {
            for (int k = 0; k < 3; ++k) srb3[k] = __half2float(net.rb3[k]);
        }
    }
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t x_addr = tc::smem_u32(sX), u_addr = tc::smem_u32(sU), w1_addr = tc::smem_u32(sW1), w1t_addr = tc::smem_u32(sW1T);
    const uint32_t r1_addr = tc::smem_u32(sR1), r2_addr = tc::smem_u32(sR2);
    const SoftplusK spk(net.dec.beta);

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        float xn[3], xs[3];
        int64_t ray;
        load_point(ps, ps.x == nullptr, i, valid, xn, xs, ray);
        float J0[16][3], J1[16][3];
        gather_row_and_jacobian(m, grid, xs, La, sX, tid, J0, J1);                  // h -> chunks 0..3 of X, J -> registers
        if constexpr (NF > 32) gather_row_to_tile<kTile, NF, kColorGatherU>(m, grid, xs, La, sX, tid, 16);   // levels 16.. -> chunks 4..5
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<64, 0, 0, NF / 16>(acc, kS, 0, tc::kmajor(x_addr, kTile), tc::kmajor(w1_addr, HW), false);   // Z = H . W1^T
        __syncthreads();
        // ---- decoder epilogue: z, a -> sdf ; u = fp16(w2 * s) (first-order cotangent at z)
        float out = 0.f;
        // the saved tiles (512 B per point, written once and read once by the backward) are stored evict-first (st.global.cs), so that
        // the stream does not push the L2-resident table out of L2 while this kernel gathers from it
        uint8_t *zt = Zt ? Zt + tile * kTileBytes : nullptr;
#pragma unroll 1
        for (int c = 0; c < HW / 8; ++c) {
            float z[8], uu[8];
            tc::acc_ld8(acc, kS, tid, c * 8, z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                z[j] = r16(z[j] + sb1[c * 8 + j]);
                float a, s;
                softplus_as(z[j], spk, a, s);
                out = fmaf(r16(a), sW2[c * 8 + j], out);
                uu[j] = sW2[c * 8 + j] * s;
            }
            *reinterpret_cast<uint4 *>(sU + c * kChunk + tid * 16) = tc::pack8_f16(uu);
            if (zt) __stcs(reinterpret_cast<uint4 *>(zt + c * kChunk + tid * 16), tc::pack8_f16(z));
        }
        const float sdf = r16(out + sb2);
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<NF, 0, 0, HW / 16>(acc, kS, 0, tc::kmajor(u_addr, kTile), tc::kmajor(w1t_addr, NF), false);   // g = U . W1
        __syncthreads();
        // ---- nablas01 = J^T g, f ascending (k_lotd_bwd_input order), J from the gather (levels >= 16: from a second corner load)
        float nacc[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (uint32_t g4 = 0; g4 < NF / 8; ++g4) {
            float gg[8];
            tc::acc_ld8(acc, kS, tid, g4 * 8, gg);
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if (p < La) {
                    const float g0 = r16(gg[2 * q]), g1 = r16(gg[2 * q + 1]);
                    float Jr0[3], Jr1[3];
                    if (p >= 16) level_jacobian(m, p, xs, grid, Jr0, Jr1);
                    const uint32_t pj = p < 16 ? p : 15;       // p is a constant after unrolling: J stays statically indexed
#pragma unroll
                    for (int d = 0; d < 3; ++d) nacc[d] = __fmaf_rn(g0, p < 16 ? J0[pj][d] : Jr0[d], nacc[d]);
#pragma unroll
                    for (int d = 0; d < 3; ++d) nacc[d] = __fmaf_rn(g1, p < 16 ? J1[pj][d] : Jr1[d], nacc[d]);
                }
            }
        }
        float nab[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) nab[d] = __fmul_rn(__fmul_rn(nacc[d], 0.5f), net.fac[d]);
        float o3[3] = {0.f, 0.f, 0.f};
        if constexpr (kRad) {
            // ---- radiance input, columns NF..NF+31: [x | SH(v) | clamp(n) | h_appear | 0]
            {
                float xr[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) xr[k] = 0.f;
                xr[0] = xn[0]; xr[1] = xn[1]; xr[2] = xn[2];
                if (valid) {
                    sh_basis(view_dirs[ray * 3], view_dirs[ray * 3 + 1], view_dirs[ray * 3 + 2], 4, xr + 3);
                    if (h_appear) {
#pragma unroll
                        for (int k = 0; k < 8; ++k)
                            if (k < net.n_appear) xr[22 + k] = h_appear[ray * net.n_appear + k];
                    }
                }
#pragma unroll
                for (int d = 0; d < 3; ++d) xr[19 + d] = fminf(fmaxf(nab[d], -1.f), 1.f);
                uint8_t *xt = Xt ? Xt + tile * x_tile_bytes<NF>() : nullptr;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float v8[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) v8[k] = xr[c * 8 + k];
                    const uint4 q = tc::pack8_f16(v8);
                    *reinterpret_cast<uint4 *>(sX + (NF / 8 + c) * kChunk + tid * 16) = q;
                    if (xt) {
                        __stcs(reinterpret_cast<uint4 *>(xt + (NF / 8 + c) * kChunk + tid * 16), q);
                        __stcs(reinterpret_cast<uint4 *>(xt + c * kChunk + tid * 16), *reinterpret_cast<const uint4 *>(sX + c * kChunk + tid * 16));
                    }
                }
                if (xt) {
#pragma unroll
                    for (int c = 4; c < NF / 8; ++c)
                        __stcs(reinterpret_cast<uint4 *>(xt + c * kChunk + tid * 16), *reinterpret_cast<const uint4 *>(sX + c * kChunk + tid * 16));
                }
            }
            tc::fence_async_smem();
            __syncthreads();
            tc::mma_to_rows<64, 0, 0, XC / 16>(acc, kS, 0, tc::kmajor(x_addr, kTile), tc::kmajor(r1_addr, XW), false);   // Y1 = X . R1^T
            __syncthreads();
            uint8_t *y1t = Y1t ? Y1t + tile * kTileBytes : nullptr;
#pragma unroll 1
            for (int c = 0; c < XW / 8; ++c) {
                float y[8];
                tc::acc_ld8(acc, kS, tid, c * 8, y);
#pragma unroll
                for (int j = 0; j < 8; ++j) y[j] = fmaxf(r16(y[j] + srb1[c * 8 + j]), 0.f);
                const uint4 q = tc::pack8_f16(y);
                *reinterpret_cast<uint4 *>(sU + c * kChunk + tid * 16) = q;
                if (y1t) __stcs(reinterpret_cast<uint4 *>(y1t + c * kChunk + tid * 16), q);
            }
            tc::fence_async_smem();
            __syncthreads();
            tc::mma_to_rows<64, 0, 0, XW / 16>(acc, kS, 0, tc::kmajor(u_addr, kTile), tc::kmajor(r2_addr, XW), false);   // Y2 = relu(Y1) . R2^T
            __syncthreads();
            uint8_t *y2t = Y2t ? Y2t + tile * kTileBytes : nullptr;
#pragma unroll 1
            for (int c = 0; c < XW / 8; ++c) {
                float y[8];
                tc::acc_ld8(acc, kS, tid, c * 8, y);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    y[j] = fmaxf(r16(y[j] + srb2[c * 8 + j]), 0.f);
#pragma unroll
                    for (int k = 0; k < 3; ++k) o3[k] = fmaf(y[j], sR3[k][c * 8 + j], o3[k]);
                }
                if (y2t) __stcs(reinterpret_cast<uint4 *>(y2t + c * kChunk + tid * 16), tc::pack8_f16(y));
            }
        } else if (Xt) {                                       // the h part of the saved X tile (what k_color_sdf_bwd fetches)
            uint8_t *xt = Xt + tile * x_tile_bytes<NF>();
#pragma unroll
            for (int c = 0; c < NF / 8; ++c)
                __stcs(reinterpret_cast<uint4 *>(xt + c * kChunk + tid * 16), *reinterpret_cast<const uint4 *>(sX + c * kChunk + tid * 16));
        }
        if (valid) {
            sdf_out[i] = sdf;
            if (oc.pcl) occ_collect_point(oc, xs, sdf);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                nab_out[i * 3 + d] = nab[d];
                if constexpr (kRad) {
                    const float y3 = r16(o3[d] + srb3[d]);
                    rgb_out[i * 3 + d] = r16(1.f / (1.f + expf(-y3)));
                }
                if (x_out) x_out[i * 3 + d] = xn[d];
            }
        }
        __syncthreads();
    }
}

// ===================================================================================================================== radiance backward
// T = [dZ2 | dZ1 | y2] (128 points x 192, three 16 KB blocks).  MMAs per tile (NF = 32; at NF = 48 dh is N48 and XB N96):
//   dY1 = dZ2 . R2                 (M128 N64 K64)    A = T block 0 (K-major),           B = R2^T tile
//   dh  = dZ1 . R1[:, h columns]   (M128 NF  K64)    A = T block 1,                     B = R1h^T tile
//   XA += dZ2^T . [Y1 | 1 | 0]               (M64 N80 K128, MN-major) = [dR2 | drb2]
//   XB += dZ1^T . [X | 1 gy3 | 0]            (M64 N(NF+48) K128, MN-major) = [dR1 | drb1]
//   X3 += y2^T  . [1 gy3 0..]                (M64 N8  K128, MN-major): cols 1..3 = dR3^T
// XA, XB and X3 are register fragments carried over all tiles of the persistent CTA; the dY1 ReLU mask runs on the dY1 fragments, and
// dh goes from its fragments straight to global memory, so the kernel stages no fp32 rows (~104 KB of shared memory, 112 KB at NF = 48:
// 2 CTAs / SM).
// kAppear adds the appearance-code gradient of every point (the codes are the internal radiance input's columns NF+22..NF+22+n_appear):
//   da  = dZ1 . R1[:, h_appear]    (M128 N8 K64)     A = T block 1,                     B = R1a^T tile (1 KB more shared memory)
// written from its fragments like dh, as rows of 8 floats (zero beyond n_appear); k_ray_row_sum adds them up per ray.
// kRays adds the gradient of every point's position and SH view embedding (the reference's radiance input columns 0..18):
//   dxv = dZ1 . R1[:, 0:19]       (M128 N32 K64)     A = T block 1,                     B = R1x^T tile (4 KB more shared memory)
// written as rows of 24 floats [dL/dx (3) | dL/dSH (16) | 0]; k_color_sdf_bwd<true> adds dL/dx to the table's input gradient and maps
// dL/dSH to the view direction.
// The three saved activation tiles of a point tile (X, Y1, Y2: 3 x 16 KB (X: 20 KB at NF = 48), each contiguous in global memory and in shared memory) are
// fetched by the bulk async copy engine (cp.async.bulk -> mbarrier), issued by one thread; the fetch of the NEXT tile starts as soon
// as the last MMA that reads the current tiles has completed, so it overlaps the dh store and the next prologue.
template <bool kAppear, bool kRays, int NF>
__global__ void __launch_bounds__(kTile, kColorBwdCtasPerSM)
k_color_rad_bwd(const ColorNetDev net, const uint8_t *__restrict__ Xt, const uint8_t *__restrict__ Y1t, const uint8_t *__restrict__ Y2t,
                const float *__restrict__ rgb, const float *__restrict__ g_rgb, int64_t n, float *__restrict__ dh_out,
                float *__restrict__ dR1, float *__restrict__ drb1, float *__restrict__ dR2, float *__restrict__ drb2,
                float *__restrict__ dR3, float *__restrict__ drb3, const int64_t *__restrict__ n_dev, float *__restrict__ da_out,
                float *__restrict__ xv_out) {
    n = eff_n(n, n_dev);
    constexpr int NE = 80;                                     // 64 columns + the [1, gy3, 0..] chunk + a zero chunk (N % 16 == 0)
    constexpr int XC = x_cols<NF>(), NEX = XC + 16;            // the X tile, and the same with its two extra chunks (80, or 96)
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t *sT = tiles;                                       // 48 KB
    uint8_t *sY1 = sT + 3 * kTileBytes;                        // 20 KB [Y1 | 1 | 0]
    uint8_t *sXe = sY1 + kTile * NE * 2;                       // 20 KB (NF = 48: 24 KB) [X | 1 gy3 | 0]
    uint8_t *sR2T = sXe + kTile * NEX * 2;                     //  8 KB (N = in i, K = out j) = R2[j][i]
    uint8_t *sR1h = sR2T + XW * XW * 2;                        //  4 KB (6 KB) (N = h column k, K = out j) = R1[j][22 + k], zero for k >= 2L
    uint8_t *sR1a = sR1h + NF * XW * 2;                        //  1 KB (kAppear; N = code column k, K = out j) = R1[j][22 + 2L + k], zero for k >= n_appear
    uint8_t *sR1x = sR1a + 8 * XW * 2;                         //  4 KB (kRays; N = input column k, K = out j) = R1[j][k], zero for k >= 19
    __shared__ float sR3[3][XW];
    __shared__ float sdb3[3];
    __shared__ __align__(8) uint64_t mbar_ld;

    const int tid = threadIdx.x, lane = tid & 31;
    for (int e = tid; e < XW * XW; e += kTile) {
        const int i = e % XW, j = e / XW;
        const __half v = (j < net.rw && i < net.rw) ? net.R2[j * net.rw + i] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sR2T + (j / 8) * (XW * 16) + i * 16 + (j % 8) * 2) = v;
    }
    for (int e = tid; e < NF * XW; e += kTile) {
        const int k = e % NF, j = e / NF;
        const __half v = (j < net.rw && k < net.dec.nh) ? net.R1[j * net.rin + 22 + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sR1h + (j / 8) * (NF * 16) + k * 16 + (j % 8) * 2) = v;
    }
    if constexpr (kAppear) {
        for (int e = tid; e < 8 * XW; e += kTile) {
            const int k = e % 8, j = e / 8;
            const __half v = (j < net.rw && k < net.n_appear) ? net.R1[j * net.rin + 22 + net.dec.nh + k] : __float2half_rn(0.f);
            *reinterpret_cast<__half *>(sR1a + (j / 8) * (8 * 16) + k * 16 + (j % 8) * 2) = v;
        }
    }
    if constexpr (kRays) {
        for (int e = tid; e < kXVCols * XW; e += kTile) {
            const int k = e % kXVCols, j = e / kXVCols;
            const __half v = (j < net.rw && k < 19) ? net.R1[j * net.rin + k] : __float2half_rn(0.f);
            *reinterpret_cast<__half *>(sR1x + (j / 8) * (kXVCols * 16) + k * 16 + (j % 8) * 2) = v;
        }
    }
    if (tid < XW) {
#pragma unroll
        for (int k = 0; k < 3; ++k) sR3[k][tid] = tid < net.rw ? __half2float(net.R3[k * net.rw + tid]) : 0.f;
    }
    *reinterpret_cast<uint4 *>(sY1 + 8 * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);       // [1, 0, ...]
    *reinterpret_cast<uint4 *>(sY1 + 9 * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sXe + (XC / 8 + 1) * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    float xa[NE / 2], xb[NEX / 2], x3[4];
#pragma unroll
    for (int k = 0; k < NE / 2; ++k) xa[k] = 0.f;
#pragma unroll
    for (int k = 0; k < NEX / 2; ++k) xb[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) x3[k] = 0.f;
    if (tid == 0) {
        sdb3[0] = sdb3[1] = sdb3[2] = 0.f;
        tc::mbar_init(&mbar_ld, 1);
        tc::fence_mbar_init();
    }
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t t_addr = tc::smem_u32(sT), y1_addr = tc::smem_u32(sY1), xe_addr = tc::smem_u32(sXe);
    const uint32_t r2t_addr = tc::smem_u32(sR2T), r1h_addr = tc::smem_u32(sR1h);
    uint32_t ld_phase = 0;
    bool first_tile = true;

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    auto fetch = [&](int64_t tile) {                          // one thread: 48 KB (52 KB) of saved activations -> the three shared-memory tiles
        tc::mbar_arrive_expect_tx(&mbar_ld, 2 * kTileBytes + x_tile_bytes<NF>());
        tc::tma_load_bulk(sT + 2 * kTileBytes, Y2t + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sY1, Y1t + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sXe, Xt + tile * x_tile_bytes<NF>(), x_tile_bytes<NF>(), &mbar_ld);
    };
    if (tid == 0 && (int64_t)blockIdx.x < n_tiles) fetch(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        tc::mbar_wait(&mbar_ld, ld_phase);                    // the tiles of this iteration have landed
        ld_phase ^= 1;
        float gy[3] = {0.f, 0.f, 0.f};
        if (valid && g_rgb) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float y = rgb[i * 3 + k];
                gy[k] = r16(r16(g_rgb[i * 3 + k]) * ((1.f - y) * y));          // sigmoid backward on the fp16 output
            }
        }
        {
            float e8[8] = {1.f, gy[0], gy[1], gy[2], 0.f, 0.f, 0.f, 0.f};
            *reinterpret_cast<uint4 *>(sXe + (XC / 8) * kChunk + tid * 16) = tc::pack8_f16(e8);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float sgy = warp_sum(gy[k]);
            if (lane == 0 && sgy != 0.f) atomicAdd(&sdb3[k], sgy);
        }
#pragma unroll 1
        for (int c = 0; c < 8; ++c) {
            float y2[8], d[8];
            unpack8(*reinterpret_cast<const uint4 *>(sT + 2 * kTileBytes + c * kChunk + tid * 16), y2);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v = gy[0] * sR3[0][c * 8 + j] + gy[1] * sR3[1][c * 8 + j] + gy[2] * sR3[2][c * 8 + j];
                d[j] = y2[j] > 0.f ? v : 0.f;
            }
            *reinterpret_cast<uint4 *>(sT + c * kChunk + tid * 16) = tc::pack8_f16(d);
        }
        tc::fence_async_smem();
        __syncthreads();
        {
            float dy[2][XW / 2];
            tc::mma_m128<64, 0, 0, XW / 16>(dy, tc::kmajor(t_addr, kTile), tc::kmajor(r2t_addr, XW), false);   // dY1 = dZ2 . R2
            // dZ1 = dY1 masked by Y1 > 0, on the fragments: T block 1 is read by no MMA in flight
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < XW / 8; ++c)
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const uint32_t off = tc::pair_off<kTile>(h * 64 + tc::frag_row(r), tc::frag_col(c));
                        const float2 y1 = tc::ld_pair_f16(sY1, off);
                        tc::st_pair_f16(sT + kTileBytes, off, y1.x > 0.f ? dy[h][4 * c + 2 * r] : 0.f, y1.y > 0.f ? dy[h][4 * c + 2 * r + 1] : 0.f);
                    }
        }
        tc::fence_async_smem();
        __syncthreads();
        float dh[2][NF / 2];
        tc::mma_m128<NF, 0, 0, XW / 16>(dh, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(r1h_addr, NF), false);   // dh = dZ1 . R1[:, h]
        float da[2][4];
        if constexpr (kAppear)
            tc::mma_m128<8, 0, 0, XW / 16>(da, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(tc::smem_u32(sR1a), 8), false);   // da = dZ1 . R1[:, h_appear]
        float dxv[2][kXVCols / 2];
        if constexpr (kRays)
            tc::mma_m128<kXVCols, 0, 0, XW / 16>(dxv, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(tc::smem_u32(sR1x), kXVCols), false);   // dxv = dZ1 . R1[:, 0:19]
        // weight gradients: contract over the 128 points
        tc::mma_m64<NE, 1, 1, kTile / 16>(xa, tc::mnmajor(t_addr, kTile), tc::mnmajor(y1_addr, kTile), true);
        tc::mma_m64<NEX, 1, 1, kTile / 16>(xb, tc::mnmajor(t_addr + kTileBytes, kTile), tc::mnmajor(xe_addr, kTile), true);
        tc::mma_m64<8, 1, 1, kTile / 16>(x3, tc::mnmajor(t_addr + 2 * kTileBytes, kTile), tc::mnmajor(xe_addr + (XC / 8) * kChunk, kTile), true);
        first_tile = false;
        __syncthreads();
        if (tid == 0 && tile + gridDim.x < n_tiles) {
            // every reader of the three tiles is done: the threads' own reads precede the __syncthreads before the MMAs above, and those MMAs
            // (the last readers) have completed before the barrier above -> the next tile's activations may overwrite them while this tile is finished
            tc::fence_async_smem();
            fetch(tile + gridDim.x);
        }
        // dh from the fragments: the four lanes of a row write its 32 contiguous bytes of a chunk.  No shared memory is read after the
        // barrier above, so the next iteration may overwrite T right away.
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int64_t row = tile * kTile + h * 64 + tc::frag_row(r);
                if (row < n) {
#pragma unroll
                    for (int c = 0; c < NF / 8; ++c)
                        *reinterpret_cast<float2 *>(dh_out + row * NF + tc::frag_col(c)) = make_float2(dh[h][4 * c + 2 * r], dh[h][4 * c + 2 * r + 1]);
                    if constexpr (kAppear) *reinterpret_cast<float2 *>(da_out + row * 8 + tc::frag_col(0)) = make_float2(da[h][2 * r], da[h][2 * r + 1]);
                    if constexpr (kRays) {
#pragma unroll
                        for (int c = 0; c < 3; ++c)
                            *reinterpret_cast<float2 *>(xv_out + row * 24 + tc::frag_col(c)) = make_float2(dxv[h][4 * c + 2 * r], dxv[h][4 * c + 2 * r + 1]);
                    }
                }
            }
    }
    if (!first_tile) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = tc::frag_row(r);
            if (row >= net.rw) continue;
#pragma unroll
            for (int c = 0; c < NEX / 8; ++c)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int col = tc::frag_col(c) + j;
                    const float b = xb[4 * c + 2 * r + j];
                    if (c < NE / 8) {
                        const float a = xa[(4 * c + 2 * r + j) % (NE / 2)];   // (the modulo only keeps the index in range for c >= NE / 8)
                        if (col < XW) {
                            if (col < net.rw) atomicAdd(dR2 + row * net.rw + col, a);
                        } else if (col == XW)
                            atomicAdd(drb2 + row, a);
                    }
                    if (col < XC) {
                        const int rc = ref_col(col, net.n_appear, net.dec.nh, NF);
                        if (rc >= 0) atomicAdd(dR1 + row * net.rin + rc, b);
                    } else if (col == XC)
                        atomicAdd(drb1 + row, b);
                }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int col = tc::frag_col(0) + j;
                if (col >= 1 && col <= 3) atomicAdd(dR3 + (col - 1) * net.rw + row, x3[2 * r + j]);
            }
        }
        if (tid < 3) atomicAdd(drb3 + tid, sdb3[tid]);
    }
}

// ===================================================================================================================== sdf / nablas backward
// T = [dz | u | v] (128 x 192).  gin = dL/dnablas * fac * 0.5 (cotangent of nablas01), dsdf optional, dh_r = dL/dh from the radiance net.
//   dg_f = sum_d gin_d J[f][d]  (k_lotd_ddLdy)                                   -> fp16 tile Ge = [dG | 1 0..]
//   du = dG . W1^T (M128 N64 K=NF);  g = U . W1 (M128 N=NF K64)
//   dz_j = fp16(du_j) w2_j beta s_j (1 - s_j) + dsdf w2_j s_j ;  v_j = fp16(du_j) s_j + dsdf a16_j
//   dhz = dZ . W1 (M128 N=NF K64)
//   W  += dz^T . [H | 1 | 0]     (M64 N=NF+16 K128, MN-major) = [dW1 (z part) | db1]
//   W[:, 0..NF-1] += u^T . dG    (M64 N=NF K128, MN-major): dW1 (second-order part); N = NF keeps sum(u) out of db1
//   V  += v^T . [1 0..]          (M64 N8  K128, MN-major): col 0 = dW2
//   scatter per level / corner:  g_f * wsum_c(gin) + (dhz_f + dh_r_f) * w_c
// W and V are register fragments carried over all tiles of the persistent CTA, dz and v are computed on the du fragments, and only g and
// dhz -- the scatter needs a point's whole row of them -- are staged as fp32 rows, in T once its last MMA has completed (~97 KB of
// shared memory, 109 KB at NF = 48: 2 CTAs / SM; at NF = 48 the rows also take the head of Ge, which follows T and is free then).
// The saved Z tile (16 KB) and the H part of the saved X tile (8 KB, 12 KB at NF = 48) are fetched by the bulk async copy engine into shared memory, and
// the NEXT tile's fetch is issued right after the last MMA of the current tile -- it runs behind the whole scatter phase.  (Reading Z
// straight from global memory in the two epilogue loops costs 16 dependent round trips per tile at 8 warps per SM.)
// kXGrad adds the gradient of every point's ray (the depths t are constants): the scatter loop loads the corners of each level it scatters
// to once more and adds J^T (dhz + dh_r) to the point's table-space input gradient (first order: the table-Hessian term of the scatter does
// not reach x), which is mapped to network space and added to dL/dx of the radiance input (xv rows of k_color_rad_bwd<., true>, NULL
// without rgb); dL/dSH of those rows is mapped to the view direction through the SH Jacobian.  Each point writes a row of 12 floats
// [g_x | t g_x | g_v | 0 0 0], which k_ray_row_sum adds up per ray.
template <bool kXGrad, int NF>
__global__ void __launch_bounds__(kTile, kColorBwdCtasPerSM)
k_color_sdf_bwd(const PLMeta m, const __half *__restrict__ grid, const ColorNetDev net, const PointSrc ps, const uint8_t *__restrict__ Zt,
                const uint8_t *__restrict__ Xt, const float *__restrict__ g_nab, const float *__restrict__ g_sdf, const float *__restrict__ dh_r,
                int64_t n, int max_level, float *__restrict__ d_grid, float *__restrict__ d_W1, float *__restrict__ d_b1, float *__restrict__ d_W2,
                float *__restrict__ d_b2, const int64_t *__restrict__ n_dev, const float *__restrict__ xv_rows,
                const float *__restrict__ view_dirs, float *__restrict__ gx_out, const int32_t *__restrict__ ml_dev) {
    n = eff_n(n, n_dev);
    const uint32_t La = active_levels(max_level, ml_dev, m.n_pseudo);
    constexpr int NX = NF + 16;                                // NF + the [1 0..] chunk + a zero chunk (N % 16 == 0)
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t *sT = tiles;                                       // 48 KB [dz | u | v]
    uint8_t *sGe = sT + 3 * kTileBytes;                        // 12 KB (NF = 48: 16 KB) [dG | 1 | 0]
    uint8_t *sHe = sGe + kTile * NX * 2;                       // 12 KB (16 KB) [H | 1 | 0]
    uint8_t *sW1 = sHe + kTile * NX * 2;                       //  4 KB (6 KB)
    uint8_t *sW1T = sW1 + HW * NF * 2;                         //  4 KB (6 KB)
    uint8_t *sZ = sW1T + NF * HW * 2;                          // 16 KB saved pre-activations
    constexpr int kS = tc::acc_stride(2 * NF);                 // staged rows [g | dhz] for the scatter: 34 KB (50 KB), aliasing T (and Ge)
    float *stage = reinterpret_cast<float *>(sT);
    // the rows may run into Ge's feature chunks (free after the MMAs), never into its constant [1 0..] and zero chunks at NF / 8 and
    // NF / 8 + 1, which are written once before the tile loop
    static_assert(kTile * kS * 4 <= 3 * kTileBytes + (NF / 8) * kChunk, "the staged rows must end before Ge's constant chunks");
    __shared__ float sW2[HW], sdsdf[kTile];
    __shared__ float sdb2;
    __shared__ __align__(8) uint64_t mbar_ld;

    const int tid = threadIdx.x, lane = tid & 31;
    stage_W1<NF>(net.dec, sW1, tid);
    stage_W1T<NF>(net.dec, sW1T, tid);
    stage_decoder_vectors(net.dec, nullptr, sW2, nullptr, tid);
    *reinterpret_cast<uint4 *>(sHe + (NF / 8) * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sGe + (NF / 8) * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sHe + (NF / 8 + 1) * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sGe + (NF / 8 + 1) * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    float wacc[NX / 2], vacc[4];
#pragma unroll
    for (int k = 0; k < NX / 2; ++k) wacc[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) vacc[k] = 0.f;
    if (tid == 0) {
        sdb2 = 0.f;
        tc::mbar_init(&mbar_ld, 1);
        tc::fence_mbar_init();
    }
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t t_addr = tc::smem_u32(sT), he_addr = tc::smem_u32(sHe), ge_addr = tc::smem_u32(sGe), w1_addr = tc::smem_u32(sW1),
                   w1t_addr = tc::smem_u32(sW1T);
    const SoftplusK spk(net.dec.beta);
    uint32_t ld_phase = 0;
    bool first_tile = true;

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    auto fetch = [&](int64_t tile) {                          // one thread: Z tile + the H chunks of the X tile -> shared memory
        tc::mbar_arrive_expect_tx(&mbar_ld, kTileBytes + (NF / 8) * kChunk);
        tc::tma_load_bulk(sZ, Zt + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sHe, Xt + tile * x_tile_bytes<NF>(), (NF / 8) * kChunk, &mbar_ld);
    };
    if (tid == 0 && (int64_t)blockIdx.x < n_tiles) fetch(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        float xn[3], xs[3];
        int64_t ray;
        load_point(ps, ps.x == nullptr, i, valid, xn, xs, ray);
        float gin[3] = {0.f, 0.f, 0.f};
        if (valid && g_nab) {
#pragma unroll
            for (int d = 0; d < 3; ++d) gin[d] = g_nab[i * 3 + d] * net.fac[d] * 0.5f;
        }
        const float dsdf = (valid && g_sdf) ? g_sdf[i] : 0.f;
        sdsdf[tid] = dsdf;                                    // read by the fragment owners of my row
        tc::mbar_wait(&mbar_ld, ld_phase);                    // this tile's Z and H have landed
        ld_phase ^= 1;
        // u = fp16(w2 s)
#pragma unroll 1
        for (int c = 0; c < 8; ++c) {
            float z[8], uu[8];
            unpack8(*reinterpret_cast<const uint4 *>(sZ + c * kChunk + tid * 16), z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a, s;
                softplus_as(z[j], spk, a, s);
                uu[j] = sW2[c * 8 + j] * s;
            }
            *reinterpret_cast<uint4 *>(sT + kTileBytes + c * kChunk + tid * 16) = tc::pack8_f16(uu);
        }
        // dg = J gin (fp16), level by level, into my row of Ge; zero for the levels >= La (columns 2La..NF-1)
#pragma unroll 4
        for (uint32_t p = 0; p < NF / 2; ++p) {               // four levels per trip: 32 independent corner loads in flight (2 CTAs / SM: registers are free)
            uint32_t packed = 0;
            if (p < La) {
                float J0[3], J1[3];
                level_jacobian(m, p, xs, grid, J0, J1);
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int d = 0; d < 3; ++d) { a0 = __fmaf_rn(gin[d], J0[d], a0); a1 = __fmaf_rn(gin[d], J1[d], a1); }
                const __half2 h = __floats2half2_rn(a0, a1);
                packed = *reinterpret_cast<const uint32_t *>(&h);
            }
            *reinterpret_cast<uint32_t *>(sGe + (p >> 2) * kChunk + tid * 16 + (p & 3) * 4) = packed;
        }
        tc::fence_async_smem();
        __syncthreads();
        float gfr[2][NF / 2];
        {
            float du[2][HW / 2];
            tc::mma_m128<64, 0, 0, NF / 16>(du, tc::kmajor(ge_addr, kTile), tc::kmajor(w1_addr, HW), false);                  // du = dG . W1^T
            tc::mma_m128<NF, 0, 0, HW / 16>(gfr, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(w1t_addr, NF), false);   // g = U . W1
            // dz -> T block 0, v -> T block 2, on the du fragments (no MMA in flight reads those blocks)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = h * 64 + tc::frag_row(r);
                    const float ds = sdsdf[row];
#pragma unroll
                    for (int c = 0; c < HW / 8; ++c) {
                        const int col = tc::frag_col(c);
                        const uint32_t off = tc::pair_off<kTile>(row, col);
                        const float2 z2 = tc::ld_pair_f16(sZ, off);
                        float dz[2], vv[2];
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const float z = j ? z2.y : z2.x;
                            float a, s;
                            softplus_as(z, spk, a, s);
                            const float w2 = sW2[col + j], d = r16(du[h][4 * c + 2 * r + j]);
                            const float curv = (z * spk.k > spk.thr) ? 0.f : spk.beta * s * (1.f - s);
                            dz[j] = d * w2 * curv + ds * w2 * s;
                            vv[j] = d * s + ds * r16(a);
                        }
                        tc::st_pair_f16(sT, off, dz[0], dz[1]);
                        tc::st_pair_f16(sT + 2 * kTileBytes, off, vv[0], vv[1]);
                    }
                }
        }
        tc::fence_async_smem();
        __syncthreads();
        float dhz[2][NF / 2];
        tc::mma_m128<NF, 0, 0, HW / 16>(dhz, tc::kmajor(t_addr, kTile), tc::kmajor(w1t_addr, NF), false);                        // dhz = dZ . W1
        tc::mma_m64<NX, 1, 1, kTile / 16>(wacc, tc::mnmajor(t_addr, kTile), tc::mnmajor(he_addr, kTile), true);
        tc::mma_m64<NF, 1, 1, kTile / 16>(*reinterpret_cast<float(*)[NF / 2]>(wacc), tc::mnmajor(t_addr + kTileBytes, kTile), tc::mnmajor(ge_addr, kTile), true);
        tc::mma_m64<8, 1, 1, kTile / 16>(vacc, tc::mnmajor(t_addr + 2 * kTileBytes, kTile), tc::mnmajor(ge_addr + (NF / 8) * kChunk, kTile), true);
        first_tile = false;
        const float dsum = warp_sum(dsdf);
        if (lane == 0 && dsum != 0.f) atomicAdd(&sdb2, dsum);
        __syncthreads();
        if (tid == 0 && tile + gridDim.x < n_tiles) {
            // sZ was last read by the threads before the __syncthreads that precedes the MMAs above, sHe by those MMAs, which have completed
            // (the staged rows below overlap Ge, never He)
            tc::fence_async_smem();
            fetch(tile + gridDim.x);
        }
        // T is free (its MMAs have completed before the barrier above): stage the rows of g and dhz there for the scatter
        tc::frag_store<NF>(gfr, stage, kS, 0);
        tc::frag_store<NF>(dhz, stage, kS, NF);
        __syncthreads();
        // ---- merged scatter
        float gx[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (uint32_t g4 = 0; g4 * 4 < La; ++g4) {
            float gg[8], hz[8];
            tc::acc_ld8(stage, kS, tid, g4 * 8, gg);
            tc::acc_ld8(stage, kS, tid, NF + g4 * 8, hz);
            if (valid && dh_r) {
                const float4 r0 = *reinterpret_cast<const float4 *>(dh_r + i * NF + g4 * 8), r1 = *reinterpret_cast<const float4 *>(dh_r + i * NF + g4 * 8 + 4);
                hz[0] += r0.x; hz[1] += r0.y; hz[2] += r0.z; hz[3] += r0.w; hz[4] += r1.x; hz[5] += r1.y; hz[6] += r1.z; hz[7] += r1.w;
            }
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if (p >= La) continue;                                                       // uniform
                uint32_t cell[8];
                float w[8], fr[3], sc[3], ua[8], ub[8];
                level_cells3(m, p, xs, cell, w, fr, sc);
                const float g0 = valid ? r16(gg[2 * q]) : 0.f, g1 = valid ? r16(gg[2 * q + 1]) : 0.f;
                const float h0 = valid ? hz[2 * q] : 0.f, h1 = valid ? hz[2 * q + 1] : 0.f;
                if constexpr (kXGrad) level_input_grad(m, p, grid, cell, fr, sc, h0, h1, gx);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    float wsum = 0.f;
#pragma unroll
                    for (int gd = 0; gd < 3; ++gd) {
                        float ww = __fmul_rn(sc[gd], gin[gd]);
#pragma unroll
                        for (int d = 0; d < 3; ++d) {
                            if (d == gd) continue;
                            ww = __fmul_rn(ww, (c & (1 << d)) ? fr[d] : __fsub_rn(1.f, fr[d]));
                        }
                        wsum += (c & (1 << gd)) ? ww : -ww;
                    }
                    ua[c] = g0 * wsum + h0 * w[c];
                    ub[c] = g1 * wsum + h1 * w[c];
                }
                if (warp_merge_updates(cell_key3(m, p, xs), valid, ua, ub, lane)) {   // neighbouring samples, same cell
                    float2 *gp = level_grad_ptr(m, p, d_grid);
#pragma unroll
                    for (int c = 0; c < 8; ++c) red_add2(gp + cell[c], ua[c], ub[c]);
                }
            }
        }
        if constexpr (kXGrad) {
            if (valid) {
                float g[3], gv[3] = {0.f, 0.f, 0.f};
#pragma unroll
                for (int d = 0; d < 3; ++d) g[d] = input_grad_to_net(gx[d]);
                if (xv_rows) {
                    const float *xr = xv_rows + i * 24;
#pragma unroll
                    for (int d = 0; d < 3; ++d) g[d] = __fadd_rn(g[d], xr[d]);
                    float jx[16], jy[16], jz[16];
                    sh_jacobian(view_dirs[ray * 3], view_dirs[ray * 3 + 1], view_dirs[ray * 3 + 2], 4, jx, jy, jz);
#pragma unroll
                    for (int c = 0; c < 16; ++c) {
                        const float dsh = xr[3 + c];
                        gv[0] = fmaf(dsh, jx[c], gv[0]); gv[1] = fmaf(dsh, jy[c], gv[1]); gv[2] = fmaf(dsh, jz[c], gv[2]);
                    }
                }
                const float tt = ps.t[i];
                float4 *o = reinterpret_cast<float4 *>(gx_out + i * 12);
                o[0] = make_float4(g[0], g[1], g[2], __fmul_rn(tt, g[0]));
                o[1] = make_float4(__fmul_rn(tt, g[1]), __fmul_rn(tt, g[2]), gv[0], gv[1]);
                o[2] = make_float4(gv[2], 0.f, 0.f, 0.f);
            }
        }
        __syncthreads();
    }
    if (!first_tile) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = tc::frag_row(r);
            if (row >= net.dec.width) continue;
#pragma unroll
            for (int c = 0; c <= NF / 8; ++c)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int col = tc::frag_col(c) + j;
                    if (col < net.dec.nh) atomicAdd(d_W1 + row * net.dec.nh + col, wacc[4 * c + 2 * r + j]);
                    else if (col == NF) atomicAdd(d_b1 + row, wacc[4 * c + 2 * r + j]);
                }
            if (tc::frag_col(0) == 0) atomicAdd(d_W2 + row, vacc[2 * r]);
        }
        if (tid == 0) atomicAdd(d_b2, sdb2);
    }
}

}  // namespace nsb

using namespace nsb;

namespace {
// radiance: the launch runs the radiance net (rgb asked for).  Otherwise rad_width == 0 with NULL radiance pointers (a geometry-only
// model) is accepted as well as a whole radiance net, which is then not read.
int make_net(const nsb_color_net *c, const nsb_lotd_meta *meta, PLMeta *m, ColorNetDev *d, const char *who, bool radiance) {
    const nsb_sdf_decoder dec{c->W1, c->b1, c->W2, c->b2, c->width, c->beta};
    if (int rc = make_decoder(meta, &dec, m, &d->dec, who)) return rc;
    if (radiance || c->rad_width != 0) {
        NSB_REQUIRE(c->rad_width >= 1 && c->rad_width <= 64, "%s: radiance width must be <= 64", who);
        NSB_REQUIRE(c->n_appear >= 0 && c->n_appear <= 8 && c->rad_in == 22 + d->dec.nh + c->n_appear,
                    "%s: radiance input must be [x(3), SH deg 4 (16), n(3), h(2L = %d), h_appear(<=8)]", who, d->dec.nh);
    } else {
        NSB_REQUIRE(!c->R1 && !c->rb1 && !c->R2 && !c->rb2 && !c->R3 && !c->rb3, "%s: rad_width 0 (no radiance net) needs NULL radiance pointers", who);
    }
    d->R1 = (const __half *)c->R1; d->rb1 = (const __half *)c->rb1; d->R2 = (const __half *)c->R2; d->rb2 = (const __half *)c->rb2;
    d->R3 = (const __half *)c->R3; d->rb3 = (const __half *)c->rb3;
    d->rw = c->rad_width; d->rin = c->rad_in; d->n_appear = c->n_appear;
    for (int k = 0; k < 3; ++k) d->fac[k] = c->nablas_scale[k];
    return 0;
}
}  // namespace

static int64_t n_tiles(int64_t n) { return (n + kTile - 1) / kTile; }

extern "C" int64_t nsb_color_tile_bytes(int64_t n) { return n_tiles(n) * (int64_t)kTileBytes; }

extern "C" int64_t nsb_color_act_bytes(int64_t n, int32_t n_levels) {
    return n_tiles(n) * (int64_t)(n_levels <= kMaxNarrowLevels ? x_tile_bytes<32>() : x_tile_bytes<48>());
}

// dynamic shared memory of the colour kernels at tile width NF (the 1 KB is the alignment slack of the tiles)
template <int NF>       // k_color_fwd<false>: the h part of X, U, W1, W1^T, the staged rows (67 KB; 75 KB at NF = 48)
constexpr int color_geo_smem() { return (NF / 8) * kChunk + kTileBytes + 2 * HW * NF * 2 + kTile * tc::acc_stride(64) * 4 + 1024; }
template <int NF>       // k_color_fwd<true>: X, U, W1, W1^T, R1, R2, the staged rows (91 KB; 101 KB at NF = 48)
constexpr int color_fwd_smem() {
    return x_tile_bytes<NF>() + kTileBytes + 2 * HW * NF * 2 + XW * x_cols<NF>() * 2 + XW * XW * 2 + kTile * tc::acc_stride(64) * 4 + 1024;
}
template <int NF, bool kAppear, bool kRays>   // k_color_rad_bwd: T, [Y1 | 1 | 0], [X | 1 gy3 | 0], R2^T, R1h, R1a, R1x (101-106 KB; 107-112 KB)
constexpr int color_rad_bwd_smem() {
    return 3 * kTileBytes + kTile * 80 * 2 + kTile * (x_cols<NF>() + 16) * 2 + XW * XW * 2 + NF * XW * 2 + (kAppear || kRays ? 8 * XW * 2 : 0) +
           (kRays ? kXVCols * XW * 2 : 0) + 1024;
}
template <int NF>       // k_color_sdf_bwd: T, Ge, He, W1, W1^T, Z (97 KB; 109 KB at NF = 48)
constexpr int color_sdf_bwd_smem() { return 3 * kTileBytes + 2 * kTile * (NF + 16) * 2 + 2 * HW * NF * 2 + kTileBytes + 1024; }
static_assert(color_geo_smem<32>() == 4 * kChunk + kTileBytes + 2 * HW * 32 * 2 + kTile * tc::acc_stride(64) * 4 + 1024, "32-column budget");
static_assert(color_fwd_smem<32>() == 2 * kTileBytes + 2 * HW * 32 * 2 + 2 * XW * XW * 2 + kTile * tc::acc_stride(64) * 4 + 1024, "32-column budget");
static_assert(color_rad_bwd_smem<32, true, true>() == 3 * kTileBytes + 2 * kTile * 80 * 2 + XW * XW * 2 + 32 * XW * 2 + 8 * XW * 2 + 32 * XW * 2 + 1024,
              "32-column budget");
static_assert(color_sdf_bwd_smem<32>() == 3 * kTileBytes + 2 * kTile * 48 * 2 + 2 * HW * 32 * 2 + kTileBytes + 1024, "32-column budget");

// calls f(std::integral_constant<int, NF>{}) with the tile width of an L-level table
template <typename F>
static int with_feature_cols(uint32_t L, F &&f) {
    return feature_cols(L) == 32 ? f(std::integral_constant<int, 32>{}) : f(std::integral_constant<int, 48>{});
}

extern "C" int nsb_fused_color_fwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x, const float *rays_o,
                                   const float *rays_d, const int64_t *ridx, const float *t, const float *view_dirs, const float *h_appear,
                                   int64_t n, int32_t max_level, float *sdf, float *nablas, float *rgb, float *x_out, void *act_z, void *act_x,
                                   void *act_y1, void *act_y2, const nsb_occ_collect *collect, void *stream) {
    const DevCounts dn = take_counts();
    const int32_t *ml_dev = take_max_level();
    if (n == 0) return 0;
    const bool rad = rgb != nullptr;
    NSB_REQUIRE(meta && params_half && net && sdf && nablas && (view_dirs || !rad), "nsb_fused_color_fwd: NULL argument");
    NSB_REQUIRE(x || (rays_o && rays_d && t), "nsb_fused_color_fwd: need x or (rays_o, rays_d, t)");
    if (rad)
        NSB_REQUIRE((act_z && act_x && act_y1 && act_y2) || (!act_z && !act_x && !act_y1 && !act_y2), "nsb_fused_color_fwd: pass all four activation buffers or none");
    else
        NSB_REQUIRE((act_z && act_x) || (!act_z && !act_x), "nsb_fused_color_fwd: without rgb, pass act_z and act_x or neither");
    PLMeta m;
    ColorNetDev d;
    if (int rc = make_net(net, meta, &m, &d, "nsb_fused_color_fwd", rad)) return rc;
    const PointSrc ps{x, rays_o, rays_d, t, ridx};
    const int ml = max_level < 0 ? -1 : max_level;
    if (!rad) {                                                // geometry only: sdf, nablas, x, Z and the h part of X
        return with_feature_cols(m.n_pseudo, [&](auto nf) -> int {
            constexpr int NF = decltype(nf)::value, kSmemG = color_geo_smem<NF>();
            // carve-out for kColorGeoCtasPerSM CTAs (dynamic + static shared memory + the 1 KB the hardware reserves per CTA), in % of 228 KB;
            // the driver rounds it up to the next configuration it supports
            constexpr int kCarveout = (100 * kColorGeoCtasPerSM * (kSmemG + 2 * 1024) + 228 * 1024 - 1) / (228 * 1024);
            if (smem_opt_in_needed(reinterpret_cast<const void *>(k_color_fwd<false, NF>), current_device(), kSmemG)) {
                cudaFuncSetAttribute(k_color_fwd<false, NF>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemG);
                cudaFuncSetAttribute(k_color_fwd<false, NF>, cudaFuncAttributePreferredSharedMemoryCarveout, kCarveout);
            }
            if (int rc = require_ctas_per_sm(k_color_fwd<false, NF>, kTile, kSmemG, kColorGeoCtasPerSM, "nsb_fused_color_fwd(geometry)")) return rc;
            k_color_fwd<false, NF><<<persistent_grid(n_tiles(n), kColorGeoCtasPerSM), kTile, kSmemG, (cudaStream_t)stream>>>(
                m, (const __half *)params_half, d, ps, nullptr, nullptr, n, ml, sdf, nablas, nullptr, x_out, (uint8_t *)act_z, (uint8_t *)act_x,
                nullptr, nullptr, occ_collect_of(collect), dn.a, ml_dev);
            return check_launch("nsb_fused_color_fwd");
        });
    }
    NSB_REQUIRE(d.n_appear == 0 || h_appear, "nsb_fused_color_fwd: h_appear is NULL but the net has %d appearance channels", d.n_appear);
    return with_feature_cols(m.n_pseudo, [&](auto nf) -> int {
        constexpr int NF = decltype(nf)::value, kSmem = color_fwd_smem<NF>();   // 91 KB (101 KB): 2 CTAs / SM
        opt_in_smem(k_color_fwd<true, NF>, kSmem);
        k_color_fwd<true, NF><<<persistent_grid(n_tiles(n), 2), kTile, kSmem, (cudaStream_t)stream>>>(
            m, (const __half *)params_half, d, ps, view_dirs, h_appear, n, ml, sdf, nablas, rgb, x_out, (uint8_t *)act_z, (uint8_t *)act_x,
            (uint8_t *)act_y1, (uint8_t *)act_y2, occ_collect_of(collect), dn.a, ml_dev);
        return check_launch("nsb_fused_color_fwd");
    });
}

// the two backward kernels (k_color_rad_bwd only with g_rgb), then with kAppear the per-ray sum of the code gradients and with kRays the
// per-ray sum of the ray gradients
template <bool kAppear, bool kRays>
static int color_bwd(const char *who, const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x, const float *rays_o,
                     const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level, const void *act_z, const void *act_x,
                     const void *act_y1, const void *act_y2, const float *rgb, const float *g_sdf, const float *g_nablas, const float *g_rgb,
                     float *dh_scratch, float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2,
                     float *d_rb2, float *d_R3, float *d_rb3, const float *view_dirs, float *ha_scratch, const int64_t *ray_map, float *d_h_appear,
                     float *ray_scratch, float *d_rays_o, float *d_rays_d, float *d_view_dirs, void *stream) {
    const DevCounts dn = take_counts();
    const int32_t *ml_dev = take_max_level();
    if (n == 0) return 0;
    NSB_REQUIRE(meta && params_half && net && act_z && act_x, "%s: NULL argument", who);
    NSB_REQUIRE(d_grid && d_W1 && d_b1 && d_W2 && d_b2, "%s: NULL gradient buffer", who);
    if (g_rgb) {                                               // the radiance backward's inputs and outputs
        NSB_REQUIRE(act_y1 && act_y2 && rgb && dh_scratch, "%s: NULL argument (g_rgb given)", who);
        NSB_REQUIRE(d_R1 && d_rb1 && d_R2 && d_rb2 && d_R3 && d_rb3, "%s: NULL radiance gradient buffer (g_rgb given)", who);
    }
    if (kAppear) NSB_REQUIRE(g_rgb && ha_scratch && d_h_appear, "%s: needs g_rgb, ha_scratch and d_h_appear", who);
    if (kRays) {
        NSB_REQUIRE(!x && rays_o && rays_d && t && ray_scratch, "%s: ray gradients need the points as rays (x NULL, rays_o, rays_d, t) and ray_scratch", who);
        NSB_REQUIRE(!g_rgb || view_dirs, "%s: ray gradients with g_rgb need view_dirs", who);
    }
    NSB_REQUIRE(x || (rays_o && rays_d && t), "%s: need x or (rays_o, rays_d, t)", who);
    PLMeta m;
    ColorNetDev d;
    if (int rc = make_net(net, meta, &m, &d, who, g_rgb != nullptr)) return rc;
    if (kAppear) NSB_REQUIRE(d.n_appear >= 1, "%s: the net has no appearance channels", who);
    cudaStream_t s = (cudaStream_t)stream;
    const float *dh = nullptr;
    float *xv_rows = (kRays && g_rgb) ? ray_scratch + n * 12 : nullptr;   // [n, 24] after the [n, 12] ray rows
    if (g_rgb) {
        const int rc = with_feature_cols(m.n_pseudo, [&](auto nf) -> int {
            constexpr int NF = decltype(nf)::value, kSmemR = color_rad_bwd_smem<NF, kAppear, kRays>();
            opt_in_smem(k_color_rad_bwd<kAppear, kRays, NF>, kSmemR);
            if (int rc = require_ctas_per_sm(k_color_rad_bwd<kAppear, kRays, NF>, kTile, kSmemR, kColorBwdCtasPerSM, "nsb_fused_color_bwd(radiance)")) return rc;
            k_color_rad_bwd<kAppear, kRays, NF><<<persistent_grid(n_tiles(n), kColorBwdCtasPerSM), kTile, kSmemR, s>>>(
                d, (const uint8_t *)act_x, (const uint8_t *)act_y1, (const uint8_t *)act_y2, rgb, g_rgb, n, dh_scratch, d_R1, d_rb1, d_R2, d_rb2, d_R3,
                d_rb3, dn.a, ha_scratch, xv_rows);
            return check_launch("nsb_fused_color_bwd(radiance)");
        });
        if (rc) return rc;
        dh = dh_scratch;
        if (kAppear) {
            k_ray_row_sum<8><<<row_sum_blocks(n), 256, 0, s>>>(ha_scratch, ridx, nullptr, n, d.n_appear, ray_map,
                                                                RowSumOut{{d_h_appear, nullptr, nullptr}, d.n_appear}, dn.a);
            if (int rc = check_launch("nsb_fused_color_bwd(code sum)")) return rc;
        }
    }
    const PointSrc ps{x, rays_o, rays_d, t, ridx};
    const int rc = with_feature_cols(m.n_pseudo, [&](auto nf) -> int {
        constexpr int NF = decltype(nf)::value, kSmemS = color_sdf_bwd_smem<NF>();
        opt_in_smem(k_color_sdf_bwd<kRays, NF>, kSmemS);
        if (int rc = require_ctas_per_sm(k_color_sdf_bwd<kRays, NF>, kTile, kSmemS, kColorBwdCtasPerSM, "nsb_fused_color_bwd(sdf)")) return rc;
        k_color_sdf_bwd<kRays, NF><<<persistent_grid(n_tiles(n), kColorBwdCtasPerSM), kTile, kSmemS, s>>>(
            m, (const __half *)params_half, d, ps, (const uint8_t *)act_z, (const uint8_t *)act_x, g_nablas, g_sdf, dh, n, max_level < 0 ? -1 : max_level,
            d_grid, d_W1, d_b1, d_W2, d_b2, dn.a, xv_rows, view_dirs, ray_scratch, ml_dev);
        return check_launch("nsb_fused_color_bwd(sdf)");
    });
    if (rc) return rc;
    if (kRays) {
        k_ray_row_sum<12><<<row_sum_blocks(n), 256, 0, s>>>(ray_scratch, ridx, nullptr, n, 9, ray_map, RowSumOut{{d_rays_o, d_rays_d, d_view_dirs}, 3},
                                                             dn.a);
        return check_launch("nsb_fused_color_bwd(ray sum)");
    }
    return 0;
}

extern "C" int nsb_fused_color_bwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x, const float *rays_o,
                                   const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level, const void *act_z,
                                   const void *act_x, const void *act_y1, const void *act_y2, const float *rgb, const float *g_sdf,
                                   const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1, float *d_b1,
                                   float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3, float *d_rb3,
                                   void *stream) {
    return color_bwd<false, false>("nsb_fused_color_bwd", meta, params_half, net, x, rays_o, rays_d, ridx, t, n, max_level, act_z, act_x, act_y1, act_y2,
                                   rgb, g_sdf, g_nablas, g_rgb, dh_scratch, d_grid, d_W1, d_b1, d_W2, d_b2, d_R1, d_rb1, d_R2, d_rb2, d_R3, d_rb3, nullptr,
                                   nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int nsb_fused_color_bwd_appear(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x,
                                          const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                                          const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                                          const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid,
                                          float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2,
                                          float *d_R3, float *d_rb3, float *ha_scratch, const int64_t *ray_map, float *d_h_appear, void *stream) {
    return color_bwd<true, false>("nsb_fused_color_bwd_appear", meta, params_half, net, x, rays_o, rays_d, ridx, t, n, max_level, act_z, act_x, act_y1,
                                  act_y2, rgb, g_sdf, g_nablas, g_rgb, dh_scratch, d_grid, d_W1, d_b1, d_W2, d_b2, d_R1, d_rb1, d_R2, d_rb2, d_R3, d_rb3,
                                  nullptr, ha_scratch, ray_map, d_h_appear, nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int nsb_fused_color_bwd_grads(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x,
                                         const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                                         const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                                         const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid,
                                         float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2,
                                         float *d_R3, float *d_rb3, const float *view_dirs, float *ha_scratch, const int64_t *ray_map,
                                         float *d_h_appear, float *ray_scratch, float *d_rays_o, float *d_rays_d, float *d_view_dirs, void *stream) {
    const char *who = "nsb_fused_color_bwd_grads";
    const bool appear = d_h_appear != nullptr, rays = d_rays_o || d_rays_d || d_view_dirs;
#define NSB_COLOR_BWD(A, R)                                                                                                                       \
    color_bwd<A, R>(who, meta, params_half, net, x, rays_o, rays_d, ridx, t, n, max_level, act_z, act_x, act_y1, act_y2, rgb, g_sdf, g_nablas, g_rgb, \
                    dh_scratch, d_grid, d_W1, d_b1, d_W2, d_b2, d_R1, d_rb1, d_R2, d_rb2, d_R3, d_rb3, view_dirs, ha_scratch, ray_map, d_h_appear,    \
                    ray_scratch, d_rays_o, d_rays_d, d_view_dirs, stream)
    const int rc = appear ? (rays ? NSB_COLOR_BWD(true, true) : NSB_COLOR_BWD(true, false))
                          : (rays ? NSB_COLOR_BWD(false, true) : NSB_COLOR_BWD(false, false));
#undef NSB_COLOR_BWD
    return rc;
}
