// Fused colour / normal query of the NeuS field and its backward (incl. the second-order path through nablas) on the
// Hopper tensor cores (wgmma), sm_90a.  One CTA = 128 threads = one warpgroup = one tile of 128 points, thread r owns
// point r (row r of the accumulators staged in shared memory, tc_util.cuh).  Replaces, for the packed samples that survive compression, the reference's chain
//   LoTDNeuS.forward (lotd_neus.py:141-167) = LoTDSDF.forward_sdf_nablas (lotd_sdf.py:201-257: LoTDFunctionFwdDydx ->
//   decoder -> autograd.grad -> LoTDFunctionBwdDydx) + RadianceNet.forward (mlp_nerf.py:267-289)
// and its autograd backward (LoTDFunctionBwdDydx.backward = lod_bwd_bwd_input, lotd.py:193-268; the autocast MLP
// double-backward) with three kernels:
//
//   k_color_fwd      gather h -> MMA Z=H.W1^T -> z,a,sdf,u=fp16(w2 s) -> MMA g=U.W1 (= dsdf/dh) -> second gather pass
//                    nablas = J^T g (J recomputed per level, never stored) -> radiance input row -> MMA -> relu -> MMA ->
//                    relu -> 64->3 -> sigmoid.   Saves the fp16 activation tiles Z, X, Y1, Y2 in core-matrix layout.
//   k_color_rad_bwd  radiance backward from the saved tiles: dZ2, dZ1 (MMA), dh (MMA), weight gradients accumulated in
//                    shared memory over all tiles of the persistent CTA (MN-major MMAs contracting over the 128 points).
//   k_color_sdf_bwd  gather pass for dg = J.dn, MMA du = dG.W1^T, MMA g = U.W1, dz (softplus'' term + sdf term),
//                    MMA dh = dZ.W1, weight-gradient MMAs, one merged scatter (g (x) second-order weights + dh (x) trilinear
//                    weights) into the fp32 table gradient.
//
// Numerics: the fp16 rounding points of the reference's autocast graph (oracle/nets.py); J and nablas use the exact
// arithmetic of k_lotd_fwd<DYDX> / k_lotd_bwd_input, so nablas is bit-identical to the unfused kernels given the same g.
// Radiance input columns are kept in the internal order [h | x | SH(v) | n | h_appear | 0] (h first, so the h tile IS the
// first four chunks of X); weights are permuted when staged / flushed.
#include "fused_tc_common.cuh"
#include "sh_device.cuh"

namespace nsb {

struct ColorNetDev {
    const __half *W1, *b1, *W2, *b2;                    // sdf decoder: [width x 32], [width], [width], [1]
    const __half *R1, *rb1, *R2, *rb2, *R3, *rb3;       // radiance net: [rw x rin], [rw], [rw x rw], [rw], [3 x rw], [3]
    int width, rw, rin, n_appear;
    float beta;
    float fac[3];                                       // sdf_scale / radius3d_original per axis
};

constexpr int XW = 64;                                  // padded radiance input width / hidden width
constexpr int kTileBytes = kTile * XW * 2;              // one saved activation tile: 16 KB
constexpr int kChunk = kTile * 16;                      // bytes of one 8-column chunk of a 128-row tile

// internal radiance-input column -> reference column (or -1 for padding)
__host__ __device__ inline int ref_col(int k, int n_appear) {
    if (k < 32) return 22 + k;
    if (k < 35) return k - 32;
    if (k < 51) return 3 + (k - 35);
    if (k < 54) return 19 + (k - 51);
    if (k < 54 + n_appear) return k;
    return -1;
}


// d(y_f)/d(x_d) of one level (both features), exactly as k_lotd_fwd<3,2,true,true> computes dy_dx
__device__ __forceinline__ void level_jacobian(const PLMeta &m, uint32_t p, const float (&xs)[3], const __half *__restrict__ grid,
                                               float (&J0)[3], float (&J1)[3]) {
    uint32_t cell[8];
    float w[8], fr[3], scale[3];
    level_cells3(m, p, xs, cell, w, fr, scale);
    const uint32_t *lp = level_cells_ptr(m, p, grid);
    float2 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const uint32_t raw = ld_nc_u32(lp + cell[c]);
        v[c] = __half22float2(*reinterpret_cast<const __half2 *>(&raw));
    }
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

__device__ __forceinline__ float r16f(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ void unpack8(const uint4 &q, float (&v)[8]) {
    const __half2 *h = reinterpret_cast<const __half2 *>(&q);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}

__device__ __forceinline__ void stage_W1T(const __half *W1, int width, uint8_t *sBT, int tid) {
    for (int e = tid; e < NF * HW; e += kTile) {              // W1^T: row = feature k, col = hidden j
        const int k = e % NF, j = e / NF;
        const __half v = j < width ? W1[j * NF + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sBT + (j / 8) * (NF * 16) + k * 16 + (j % 8) * 2) = v;
    }
}

struct PointSrc {
    const float *x, *rays_o, *rays_d, *t;
    const int64_t *ridx;
};

__device__ __forceinline__ void load_point_net(const PointSrc &ps, int64_t i, bool valid, float (&xn)[3], float (&xs)[3], int64_t &ray) {
    xn[0] = xn[1] = xn[2] = 0.f;
    ray = 0;
    if (valid) {
        if (ps.x) {
#pragma unroll
            for (int d = 0; d < 3; ++d) xn[d] = ps.x[i * 3 + d];
            ray = ps.ridx ? ps.ridx[i] : i;
        } else {
            ray = ps.ridx ? ps.ridx[i] : i;
            const float tt = ps.t[i];
#pragma unroll
            for (int d = 0; d < 3; ++d) xn[d] = __fmaf_rn(ps.rays_d[ray * 3 + d], tt, ps.rays_o[ray * 3 + d]);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) xs[d] = fminf(fmaxf(__fmaf_rn(xn[d], 0.5f, 0.5f), 1.0e-6f), 1.f - 1.0e-6f);
}

// The colour kernels run at 1-2 CTAs per SM (shared-memory bound), i.e. 4-8 warps: their gathers live on loads in flight PER THREAD, and
// registers are plentiful -> four levels (32 corner loads) per gather trip instead of the two of k_fused_sdf_tc (which runs 24 warps per SM).
constexpr int kColorGatherU = 4;

// ===================================================================================================================== forward
__global__ void __launch_bounds__(kTile)
k_color_fwd(const PLMeta m, const __half *__restrict__ grid, const ColorNetDev net, const PointSrc ps, const float *__restrict__ view_dirs,
            const float *__restrict__ h_appear, int64_t n, int max_level, float *__restrict__ sdf_out, float *__restrict__ nab_out,
            float *__restrict__ rgb_out, float *__restrict__ x_out, uint8_t *__restrict__ Zt, uint8_t *__restrict__ Xt,
            uint8_t *__restrict__ Y1t, uint8_t *__restrict__ Y2t, const OccCollect oc, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t *sX = tiles;                                       // 16 KB [h | x sh n ha 0]
    uint8_t *sU = sX + kTileBytes;                             // 16 KB u, later relu(y1)
    uint8_t *sW1 = sU + kTileBytes;                            //  4 KB W1   [64 x 32]
    uint8_t *sW1T = sW1 + HW * NF * 2;                         //  4 KB W1^T [32 x 64]
    uint8_t *sR1 = sW1T + HW * NF * 2;                         //  8 KB R1 [64 x 64] (internal column order)
    uint8_t *sR2 = sR1 + XW * XW * 2;                          //  8 KB R2 [64 x 64]
    constexpr int kS = tc::acc_stride(64);
    float *acc = reinterpret_cast<float *>(sR2 + XW * XW * 2); // 34 KB staged accumulator rows (Z, g, Y1, Y2 in turn)
    __shared__ float sb1[HW], sW2[HW], srb1[XW], srb2[XW], sR3[3][XW];
    __shared__ float sb2, srb3[3];

    const int tid = threadIdx.x;
    {
        DecoderDevTC dec{net.W1, net.b1, net.W2, net.b2, net.width, net.beta};
        stage_W1(dec, sW1, tid);
        stage_W1T(net.W1, net.width, sW1T, tid);
    }
    for (int e = tid; e < XW * XW; e += kTile) {
        const int j = e % XW, k = e / XW;                      // (out j, in k)
        const int rc = ref_col(k, net.n_appear);
        const __half v1 = (j < net.rw && rc >= 0) ? net.R1[j * net.rin + rc] : __float2half_rn(0.f);
        const __half v2 = (j < net.rw && k < net.rw) ? net.R2[j * net.rw + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sR1 + (k / 8) * (XW * 16) + j * 16 + (k % 8) * 2) = v1;
        *reinterpret_cast<__half *>(sR2 + (k / 8) * (XW * 16) + j * 16 + (k % 8) * 2) = v2;
    }
    if (tid < HW) {
        sb1[tid] = tid < net.width ? __half2float(net.b1[tid]) : 0.f;
        sW2[tid] = tid < net.width ? __half2float(net.W2[tid]) : 0.f;
        srb1[tid] = tid < net.rw ? __half2float(net.rb1[tid]) : 0.f;
        srb2[tid] = tid < net.rw ? __half2float(net.rb2[tid]) : 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) sR3[k][tid] = tid < net.rw ? __half2float(net.R3[k * net.rw + tid]) : 0.f;
    }
    if (tid == 0) {
        sb2 = __half2float(net.b2[0]);
        for (int k = 0; k < 3; ++k) srb3[k] = __half2float(net.rb3[k]);
    }
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t x_addr = tc::smem_u32(sX), u_addr = tc::smem_u32(sU), w1_addr = tc::smem_u32(sW1), w1t_addr = tc::smem_u32(sW1T);
    const uint32_t r1_addr = tc::smem_u32(sR1), r2_addr = tc::smem_u32(sR2);
    const SoftplusK spk(net.beta);

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        float xn[3], xs[3];
        int64_t ray;
        load_point_net(ps, i, valid, xn, xs, ray);
        gather_row_to_tile<kTile, kColorGatherU>(m, grid, xs, max_level, sX, tid);          // h -> chunks 0..3 of X
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<64, 0, 0, NF / 16>(acc, kS, 0, tc::kmajor(x_addr, kTile), tc::kmajor(w1_addr, HW), false);   // Z = H . W1^T
        __syncthreads();
        // ---- decoder epilogue: z, a -> sdf ; u = fp16(w2 * s) (first-order cotangent at z)
        float out = 0.f;
        uint8_t *zt = Zt ? Zt + tile * kTileBytes : nullptr;
#pragma unroll 1
        for (int c = 0; c < HW / 8; ++c) {
            float z[8], uu[8];
            tc::acc_ld8(acc, kS, tid, c * 8, z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                z[j] = r16f(z[j] + sb1[c * 8 + j]);
                float a, s;
                softplus_as(z[j], spk, a, s);
                out = fmaf(r16f(a), sW2[c * 8 + j], out);
                uu[j] = sW2[c * 8 + j] * s;
            }
            *reinterpret_cast<uint4 *>(sU + c * kChunk + tid * 16) = tc::pack8_f16(uu);
            if (zt) *reinterpret_cast<uint4 *>(zt + c * kChunk + tid * 16) = tc::pack8_f16(z);
        }
        const float sdf = r16f(out + sb2);
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<32, 0, 0, HW / 16>(acc, kS, 0, tc::kmajor(u_addr, kTile), tc::kmajor(w1t_addr, NF), false);   // g = U . W1
        __syncthreads();
        // ---- second gather pass: nablas01 = J^T g, f ascending (k_lotd_bwd_input order)
        float nacc[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (uint32_t g4 = 0; g4 < 4; ++g4) {
            float gg[8];
            tc::acc_ld8(acc, kS, tid, g4 * 8, gg);
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if ((int)m.level[p] <= max_level) {
                    float J0[3], J1[3];
                    level_jacobian(m, p, xs, grid, J0, J1);
                    const float g0 = r16f(gg[2 * q]), g1 = r16f(gg[2 * q + 1]);
#pragma unroll
                    for (int d = 0; d < 3; ++d) nacc[d] = __fmaf_rn(g0, J0[d], nacc[d]);
#pragma unroll
                    for (int d = 0; d < 3; ++d) nacc[d] = __fmaf_rn(g1, J1[d], nacc[d]);
                }
            }
        }
        float nab[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) nab[d] = __fmul_rn(__fmul_rn(nacc[d], 0.5f), net.fac[d]);
        // ---- radiance input, columns 32..63: [x | SH(v) | clamp(n) | h_appear | 0]
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
            uint8_t *xt = Xt ? Xt + tile * kTileBytes : nullptr;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float v8[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) v8[k] = xr[c * 8 + k];
                const uint4 q = tc::pack8_f16(v8);
                *reinterpret_cast<uint4 *>(sX + (4 + c) * kChunk + tid * 16) = q;
                if (xt) {
                    *reinterpret_cast<uint4 *>(xt + (4 + c) * kChunk + tid * 16) = q;
                    *reinterpret_cast<uint4 *>(xt + c * kChunk + tid * 16) = *reinterpret_cast<const uint4 *>(sX + c * kChunk + tid * 16);
                }
            }
        }
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<64, 0, 0, XW / 16>(acc, kS, 0, tc::kmajor(x_addr, kTile), tc::kmajor(r1_addr, XW), false);   // Y1 = X . R1^T
        __syncthreads();
        uint8_t *y1t = Y1t ? Y1t + tile * kTileBytes : nullptr;
#pragma unroll 1
        for (int c = 0; c < XW / 8; ++c) {
            float y[8];
            tc::acc_ld8(acc, kS, tid, c * 8, y);
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = fmaxf(r16f(y[j] + srb1[c * 8 + j]), 0.f);
            const uint4 q = tc::pack8_f16(y);
            *reinterpret_cast<uint4 *>(sU + c * kChunk + tid * 16) = q;
            if (y1t) *reinterpret_cast<uint4 *>(y1t + c * kChunk + tid * 16) = q;
        }
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<64, 0, 0, XW / 16>(acc, kS, 0, tc::kmajor(u_addr, kTile), tc::kmajor(r2_addr, XW), false);   // Y2 = relu(Y1) . R2^T
        __syncthreads();
        float o3[3] = {0.f, 0.f, 0.f};
        uint8_t *y2t = Y2t ? Y2t + tile * kTileBytes : nullptr;
#pragma unroll 1
        for (int c = 0; c < XW / 8; ++c) {
            float y[8];
            tc::acc_ld8(acc, kS, tid, c * 8, y);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                y[j] = fmaxf(r16f(y[j] + srb2[c * 8 + j]), 0.f);
#pragma unroll
                for (int k = 0; k < 3; ++k) o3[k] = fmaf(y[j], sR3[k][c * 8 + j], o3[k]);
            }
            if (y2t) *reinterpret_cast<uint4 *>(y2t + c * kChunk + tid * 16) = tc::pack8_f16(y);
        }
        if (valid) {
            sdf_out[i] = sdf;
            if (oc.pcl) occ_collect_point(oc, xs, sdf);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                nab_out[i * 3 + d] = nab[d];
                const float y3 = r16f(o3[d] + srb3[d]);
                rgb_out[i * 3 + d] = r16f(1.f / (1.f + expf(-y3)));
                if (x_out) x_out[i * 3 + d] = xn[d];
            }
        }
        __syncthreads();
    }
}

// ===================================================================================================================== radiance backward
// T = [dZ2 | dZ1 | y2] (128 points x 192, three 16 KB blocks).  MMAs per tile:
//   dY1 = dZ2 . R2                 (M128 N64 K64)    A = T block 0 (K-major),           B = R2^T tile
//   dh  = dZ1 . R1[:, h columns]   (M128 N32 K64)    A = T block 1,                     B = R1h^T tile
//   XA += [dZ2 | dZ1]^T . [Y1 | 1]           (M128 N72 K128, MN-major): rows 0..63  = [dR2 | drb2]
//   XB += [dZ1 | y2 ]^T . [X | 1 gy3 0..]    (M128 N72 K128, MN-major): rows 0..63  = [dR1 | drb1], rows 64..127, cols 65..67 = dR3^T
// TMA = true: the three saved activation tiles of a point tile (X, Y1, Y2: 3 x 16 KB, each contiguous in global memory and in shared
// memory) are fetched by the bulk async copy engine (cp.async.bulk -> mbarrier), issued by one thread; the fetch of the NEXT tile starts as soon
// as the last MMA that reads the current tiles has completed, so it overlaps the epilogue, the dh store and the next prologue.
template <bool TMA>
__global__ void __launch_bounds__(kTile)
k_color_rad_bwd(const ColorNetDev net, const uint8_t *__restrict__ Xt, const uint8_t *__restrict__ Y1t, const uint8_t *__restrict__ Y2t,
                const float *__restrict__ rgb, const float *__restrict__ g_rgb, int64_t n, float *__restrict__ dh_out,
                float *__restrict__ dR1, float *__restrict__ drb1, float *__restrict__ dR2, float *__restrict__ drb2,
                float *__restrict__ dR3, float *__restrict__ drb3, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    constexpr int NE = 80;                                     // 64 columns + the [1, gy3, 0..] chunk + a zero chunk (N % 16 == 0)
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t *sT = tiles;                                       // 48 KB
    uint8_t *sY1 = sT + 3 * kTileBytes;                        // 20 KB [Y1 | 1 | 0]
    uint8_t *sXe = sY1 + kTile * NE * 2;                       // 20 KB [X | 1 gy3 | 0]
    uint8_t *sR2T = sXe + kTile * NE * 2;                      //  8 KB (N = in i, K = out j) = R2[j][i]
    uint8_t *sR1h = sR2T + XW * XW * 2;                        //  4 KB (N = h column k, K = out j) = R1[j][22 + k]
    constexpr uint32_t cDY1 = 0, cDH = 0, cXA = 64, cXB = 64 + NE;   // staged accumulator columns (dY1, then dh; XA, XB persist)
    constexpr int kS = tc::acc_stride(64 + 2 * NE);
    float *acc = reinterpret_cast<float *>(sR1h + NF * XW * 2); // 114 KB
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
        const __half v = j < net.rw ? net.R1[j * net.rin + 22 + k] : __float2half_rn(0.f);
        *reinterpret_cast<__half *>(sR1h + (j / 8) * (NF * 16) + k * 16 + (j % 8) * 2) = v;
    }
    if (tid < XW) {
#pragma unroll
        for (int k = 0; k < 3; ++k) sR3[k][tid] = tid < net.rw ? __half2float(net.R3[k * net.rw + tid]) : 0.f;
    }
    *reinterpret_cast<uint4 *>(sY1 + 8 * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);       // [1, 0, ...]
    *reinterpret_cast<uint4 *>(sY1 + 9 * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sXe + 9 * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    for (int c = cXA; c < cXB + NE; ++c) acc[tid * kS + c] = 0.f;
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
    auto fetch = [&](int64_t tile) {                          // one thread: 48 KB of saved activations -> the three shared-memory tiles
        tc::mbar_arrive_expect_tx(&mbar_ld, 3 * kTileBytes);
        tc::tma_load_bulk(sT + 2 * kTileBytes, Y2t + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sY1, Y1t + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sXe, Xt + tile * kTileBytes, kTileBytes, &mbar_ld);
    };
    if (TMA && tid == 0 && (int64_t)blockIdx.x < n_tiles) fetch(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        if (TMA) {
            tc::mbar_wait(&mbar_ld, ld_phase);                // the tiles of this iteration have landed
            ld_phase ^= 1;
        } else {
            const uint8_t *xt = Xt + tile * kTileBytes, *y1t = Y1t + tile * kTileBytes, *y2t = Y2t + tile * kTileBytes;
#pragma unroll 1
            for (int c = 0; c < 8; ++c) {
                *reinterpret_cast<uint4 *>(sT + 2 * kTileBytes + c * kChunk + tid * 16) = *reinterpret_cast<const uint4 *>(y2t + c * kChunk + tid * 16);
                *reinterpret_cast<uint4 *>(sY1 + c * kChunk + tid * 16) = *reinterpret_cast<const uint4 *>(y1t + c * kChunk + tid * 16);
                *reinterpret_cast<uint4 *>(sXe + c * kChunk + tid * 16) = *reinterpret_cast<const uint4 *>(xt + c * kChunk + tid * 16);
            }
        }
        float gy[3] = {0.f, 0.f, 0.f};
        if (valid && g_rgb) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float y = rgb[i * 3 + k];
                gy[k] = r16f(r16f(g_rgb[i * 3 + k]) * ((1.f - y) * y));          // sigmoid backward on the fp16 output
            }
        }
        {
            float e8[8] = {1.f, gy[0], gy[1], gy[2], 0.f, 0.f, 0.f, 0.f};
            *reinterpret_cast<uint4 *>(sXe + 8 * kChunk + tid * 16) = tc::pack8_f16(e8);
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
        tc::mma_to_rows<64, 0, 0, XW / 16>(acc, kS, cDY1, tc::kmajor(t_addr, kTile), tc::kmajor(r2t_addr, XW), false);   // dY1 = dZ2 . R2
        __syncthreads();
#pragma unroll 1
        for (int c = 0; c < 8; ++c) {
            float dy[8], y1[8];
            tc::acc_ld8(acc, kS, tid, cDY1 + c * 8, dy);
            unpack8(*reinterpret_cast<const uint4 *>(sY1 + c * kChunk + tid * 16), y1);
#pragma unroll
            for (int j = 0; j < 8; ++j) dy[j] = y1[j] > 0.f ? dy[j] : 0.f;
            *reinterpret_cast<uint4 *>(sT + kTileBytes + c * kChunk + tid * 16) = tc::pack8_f16(dy);
        }
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<32, 0, 0, XW / 16>(acc, kS, cDH, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(r1h_addr, NF), false);   // dh = dZ1 . R1[:, h]
        // weight gradients: contract over the 128 points
        tc::mma_to_rows<NE, 1, 1, kTile / 16>(acc, kS, cXA, tc::mnmajor(t_addr, kTile), tc::mnmajor(y1_addr, kTile), true);
        tc::mma_to_rows<NE, 1, 1, kTile / 16>(acc, kS, cXB, tc::mnmajor(t_addr + kTileBytes, kTile), tc::mnmajor(xe_addr, kTile), true);
        first_tile = false;
        __syncthreads();
        if (TMA && tid == 0 && tile + gridDim.x < n_tiles) {
            // every reader of the three tiles is done: the threads' own reads precede the __syncthreads before the MMAs above, and those MMAs
            // (the last readers) have completed before the barrier above -> the next tile's activations may overwrite them while this tile is finished
            tc::fence_async_smem();
            fetch(tile + gridDim.x);
        }
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
            float dh[8];
            tc::acc_ld8(acc, kS, tid, cDH + c * 8, dh);
            if (valid) {
                *reinterpret_cast<float4 *>(dh_out + i * NF + c * 8) = make_float4(dh[0], dh[1], dh[2], dh[3]);
                *reinterpret_cast<float4 *>(dh_out + i * NF + c * 8 + 4) = make_float4(dh[4], dh[5], dh[6], dh[7]);
            }
        }
        __syncthreads();
    }
    if (!first_tile) {
#pragma unroll 1
        for (int c = 0; c < 9; ++c) {
            float a[8], b[8];
            tc::acc_ld8(acc, kS, tid, cXA + c * 8, a);
            tc::acc_ld8(acc, kS, tid, cXB + c * 8, b);
            if (tid < net.rw) {
                if (c < 8) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const int col = c * 8 + k;
                        if (col < net.rw) atomicAdd(dR2 + tid * net.rw + col, a[k]);
                        const int rc = ref_col(col, net.n_appear);
                        if (rc >= 0) atomicAdd(dR1 + tid * net.rin + rc, b[k]);
                    }
                } else {
                    atomicAdd(drb2 + tid, a[0]);
                    atomicAdd(drb1 + tid, b[0]);
                }
            } else if (tid >= XW && tid - XW < net.rw && c == 8) {
#pragma unroll
                for (int k = 0; k < 3; ++k) atomicAdd(dR3 + k * net.rw + (tid - XW), b[1 + k]);
            }
        }
        if (tid < 3) atomicAdd(drb3 + tid, sdb3[tid]);
    }
}

// ===================================================================================================================== sdf / nablas backward
// T = [dz | u | v] (128 x 192).  gin = dL/dnablas * fac * 0.5 (cotangent of nablas01), dsdf optional, dh_r = dL/dh from the radiance net.
//   dg_f = sum_d gin_d J[f][d]  (k_lotd_ddLdy)                                   -> fp16 tile Ge = [dG | 1 0..]
//   du = dG . W1^T (M128 N64 K32);  g = U . W1 (M128 N32 K64)
//   dz_j = fp16(du_j) w2_j beta s_j (1 - s_j) + dsdf w2_j s_j ;  v_j = fp16(du_j) s_j + dsdf a16_j
//   dhz = dZ . W1 (M128 N32 K64)
//   X1 += [dz | u]^T . [H | 1]   rows 0..63 = [dW1 (z part) | db1]
//   X2 += [u | v]^T . [dG | 1]   rows 0..63, cols 0..31 = dW1 (second-order part);  rows 64..127, col 32 = dW2
//   scatter per level / corner:  g_f * wsum_c(gin) + (dhz_f + dh_r_f) * w_c
// TMA = true: the saved Z tile (16 KB) and the H half of the saved X tile (8 KB) are fetched by the bulk async copy engine into shared memory, and
// the NEXT tile's fetch is issued right after the last MMA of the current tile -- it runs behind the whole scatter phase.  (Without it the two
// epilogue loops read Z straight from global memory, 16 dependent round trips per tile at 8 warps per SM.)
template <bool TMA>
__global__ void __launch_bounds__(kTile)
k_color_sdf_bwd(const PLMeta m, const __half *__restrict__ grid, const ColorNetDev net, const PointSrc ps, const uint8_t *__restrict__ Zt,
                const uint8_t *__restrict__ Xt, const float *__restrict__ g_nab, const float *__restrict__ g_sdf, const float *__restrict__ dh_r,
                int64_t n, int max_level, float *__restrict__ d_grid, float *__restrict__ d_W1, float *__restrict__ d_b1, float *__restrict__ d_W2,
                float *__restrict__ d_b2, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    constexpr int NX = 48;                                     // 32 + the [1 0..] chunk + a zero chunk (N % 16 == 0)
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t *sT = tiles;                                       // 48 KB [dz | u | v]
    uint8_t *sHe = sT + 3 * kTileBytes;                        // 12 KB [H | 1 | 0]
    uint8_t *sGe = sHe + kTile * NX * 2;                       // 12 KB [dG | 1 | 0]
    uint8_t *sW1 = sGe + kTile * NX * 2;                       //  4 KB
    uint8_t *sW1T = sW1 + HW * NF * 2;                         //  4 KB
    uint8_t *sZ = sW1T + NF * HW * 2;                          // 16 KB saved pre-activations (TMA only)
    constexpr uint32_t cDU = 0, cDHZ = 0, cG = 64, cX1 = 96, cX2 = 96 + NX;   // staged accumulator columns (du, then dhz; X1, X2 persist)
    constexpr int kS = tc::acc_stride(96 + 2 * NX);
    float *acc = reinterpret_cast<float *>(sZ + kTileBytes);   // 98 KB
    __shared__ float sW2[HW];
    __shared__ float sdb2;
    __shared__ __align__(8) uint64_t mbar_ld;

    const int tid = threadIdx.x, lane = tid & 31;
    {
        DecoderDevTC dec{net.W1, net.b1, net.W2, net.b2, net.width, net.beta};
        stage_W1(dec, sW1, tid);
        stage_W1T(net.W1, net.width, sW1T, tid);
    }
    if (tid < HW) sW2[tid] = tid < net.width ? __half2float(net.W2[tid]) : 0.f;
    *reinterpret_cast<uint4 *>(sHe + 4 * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sGe + 4 * kChunk + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sHe + 5 * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(sGe + 5 * kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    for (int c = cX1; c < cX2 + NX; ++c) acc[tid * kS + c] = 0.f;
    if (tid == 0) {
        sdb2 = 0.f;
        tc::mbar_init(&mbar_ld, 1);
        tc::fence_mbar_init();
    }
    tc::fence_async_smem();
    __syncthreads();
    const uint32_t t_addr = tc::smem_u32(sT), he_addr = tc::smem_u32(sHe), ge_addr = tc::smem_u32(sGe), w1_addr = tc::smem_u32(sW1),
                   w1t_addr = tc::smem_u32(sW1T);
    const SoftplusK spk(net.beta);
    uint32_t ld_phase = 0;
    bool first_tile = true;

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    auto fetch = [&](int64_t tile) {                          // one thread: Z tile + the H chunks of the X tile -> shared memory
        tc::mbar_arrive_expect_tx(&mbar_ld, kTileBytes + 4 * kChunk);
        tc::tma_load_bulk(sZ, Zt + tile * kTileBytes, kTileBytes, &mbar_ld);
        tc::tma_load_bulk(sHe, Xt + tile * kTileBytes, 4 * kChunk, &mbar_ld);
    };
    if (TMA && tid == 0 && (int64_t)blockIdx.x < n_tiles) fetch(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i = tile * kTile + tid;
        const bool valid = i < n;
        float xn[3], xs[3];
        int64_t ray;
        load_point_net(ps, i, valid, xn, xs, ray);
        float gin[3] = {0.f, 0.f, 0.f};
        if (valid && g_nab) {
#pragma unroll
            for (int d = 0; d < 3; ++d) gin[d] = g_nab[i * 3 + d] * net.fac[d] * 0.5f;
        }
        const float dsdf = (valid && g_sdf) ? g_sdf[i] : 0.f;
        const uint8_t *zt = TMA ? sZ : Zt + tile * kTileBytes;
        if (TMA) {
            tc::mbar_wait(&mbar_ld, ld_phase);                // this tile's Z and H have landed
            ld_phase ^= 1;
        } else {
            const uint8_t *xt = Xt + tile * kTileBytes;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                *reinterpret_cast<uint4 *>(sHe + c * kChunk + tid * 16) = *reinterpret_cast<const uint4 *>(xt + c * kChunk + tid * 16);
        }
        // u = fp16(w2 s)
#pragma unroll 1
        for (int c = 0; c < 8; ++c) {
            float z[8], uu[8];
            unpack8(*reinterpret_cast<const uint4 *>(zt + c * kChunk + tid * 16), z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a, s;
                softplus_as(z[j], spk, a, s);
                uu[j] = sW2[c * 8 + j] * s;
            }
            *reinterpret_cast<uint4 *>(sT + kTileBytes + c * kChunk + tid * 16) = tc::pack8_f16(uu);
        }
        // dg = J gin (fp16), level by level, into my row of Ge
#pragma unroll 4
        for (uint32_t p = 0; p < 16; ++p) {               // four levels per trip: 32 independent corner loads in flight (2 CTAs / SM: registers are free)
            uint32_t packed = 0;
            if ((int)m.level[p] <= max_level) {
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
        tc::mma_to_rows<64, 0, 0, NF / 16>(acc, kS, cDU, tc::kmajor(ge_addr, kTile), tc::kmajor(w1_addr, HW), false);                // du = dG . W1^T
        tc::mma_to_rows<32, 0, 0, HW / 16>(acc, kS, cG, tc::kmajor(t_addr + kTileBytes, kTile), tc::kmajor(w1t_addr, NF), false);    // g = U . W1
        __syncthreads();
#pragma unroll 1
        for (int c = 0; c < 8; ++c) {
            float du[8], z[8], dz[8], vv[8];
            tc::acc_ld8(acc, kS, tid, cDU + c * 8, du);
            unpack8(*reinterpret_cast<const uint4 *>(zt + c * kChunk + tid * 16), z);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a, s;
                softplus_as(z[j], spk, a, s);
                const float w2 = sW2[c * 8 + j], d = r16f(du[j]);
                const float curv = (z[j] * spk.k > spk.thr) ? 0.f : spk.beta * s * (1.f - s);
                dz[j] = d * w2 * curv + dsdf * w2 * s;
                vv[j] = d * s + dsdf * r16f(a);
            }
            *reinterpret_cast<uint4 *>(sT + c * kChunk + tid * 16) = tc::pack8_f16(dz);
            *reinterpret_cast<uint4 *>(sT + 2 * kTileBytes + c * kChunk + tid * 16) = tc::pack8_f16(vv);
        }
        tc::fence_async_smem();
        __syncthreads();
        tc::mma_to_rows<32, 0, 0, HW / 16>(acc, kS, cDHZ, tc::kmajor(t_addr, kTile), tc::kmajor(w1t_addr, NF), false);               // dhz = dZ . W1
        tc::mma_to_rows<NX, 1, 1, kTile / 16>(acc, kS, cX1, tc::mnmajor(t_addr, kTile), tc::mnmajor(he_addr, kTile), true);
        tc::mma_to_rows<NX, 1, 1, kTile / 16>(acc, kS, cX2, tc::mnmajor(t_addr + kTileBytes, kTile), tc::mnmajor(ge_addr, kTile), true);
        first_tile = false;
        const float dsum = warp_sum(dsdf);
        if (lane == 0 && dsum != 0.f) atomicAdd(&sdb2, dsum);
        __syncthreads();
        if (TMA && tid == 0 && tile + gridDim.x < n_tiles) {
            // sZ was last read by the threads before the __syncthreads that precedes the MMAs above, sHe by those MMAs, which have completed
            tc::fence_async_smem();
            fetch(tile + gridDim.x);
        }
        // ---- merged scatter
#pragma unroll 1
        for (uint32_t g4 = 0; g4 < 4; ++g4) {
            float gg[8], hz[8];
            tc::acc_ld8(acc, kS, tid, cG + g4 * 8, gg);
            tc::acc_ld8(acc, kS, tid, cDHZ + g4 * 8, hz);
            if (valid && dh_r) {
                const float4 r0 = *reinterpret_cast<const float4 *>(dh_r + i * NF + g4 * 8), r1 = *reinterpret_cast<const float4 *>(dh_r + i * NF + g4 * 8 + 4);
                hz[0] += r0.x; hz[1] += r0.y; hz[2] += r0.z; hz[3] += r0.w; hz[4] += r1.x; hz[5] += r1.y; hz[6] += r1.z; hz[7] += r1.w;
            }
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if ((int)m.level[p] > max_level) continue;               // uniform
                uint32_t cell[8];
                float w[8], fr[3], sc[3], ua[8], ub[8];
                level_cells3(m, p, xs, cell, w, fr, sc);
                const float g0 = valid ? r16f(gg[2 * q]) : 0.f, g1 = valid ? r16f(gg[2 * q + 1]) : 0.f;
                const float h0 = valid ? hz[2 * q] : 0.f, h1 = valid ? hz[2 * q + 1] : 0.f;
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
                bool issue = valid;
                if (level_mergeable(m, p)) issue = warp_merge_updates(cell_key3(m, p, xs), valid, ua, ub, lane);   // neighbouring samples, same cell
                if (issue) {
                    float2 *gp = level_grad_ptr(m, p, d_grid);
#pragma unroll
                    for (int c = 0; c < 8; ++c) red_add2(gp + cell[c], ua[c], ub[c]);
                }
            }
        }
        __syncthreads();
    }
    if (!first_tile) {
#pragma unroll 1
        for (int c = 0; c < NF / 8; ++c) {
            float a[8], b[8];
            tc::acc_ld8(acc, kS, tid, cX1 + c * 8, a);
            tc::acc_ld8(acc, kS, tid, cX2 + c * 8, b);
            if (tid < net.width) {
#pragma unroll
                for (int k = 0; k < 8; ++k) atomicAdd(d_W1 + tid * NF + c * 8 + k, a[k] + b[k]);
            }
        }
        float a1[8], b1[8];
        tc::acc_ld8(acc, kS, tid, cX1 + 32, a1);
        tc::acc_ld8(acc, kS, tid, cX2 + 32, b1);
        if (tid < HW) { if (tid < net.width) atomicAdd(d_b1 + tid, a1[0]); }
        else if (tid - HW < net.width) atomicAdd(d_W2 + (tid - HW), b1[0]);
        if (tid == 0) atomicAdd(d_b2, sdb2);
    }
}

}  // namespace nsb

using namespace nsb;

namespace {
int make_net(const nsb_color_net *c, const nsb_lotd_meta *meta, PLMeta *m, ColorNetDev *d, const char *who) {
    if (make_plmeta(meta, m)) return 2;
    NSB_REQUIRE(m->n_pseudo == 16 && m->F == 2 && m->D == 3 && plmeta_two_feature_cells(*m), "%s: built for 16 x 2 LoTD features in 3-D", who);
    NSB_REQUIRE(c->width >= 1 && c->width <= 64 && c->rad_width >= 1 && c->rad_width <= 64, "%s: hidden widths must be <= 64", who);
    NSB_REQUIRE(c->n_appear >= 0 && c->n_appear <= 8 && c->rad_in == 54 + c->n_appear,
                "%s: radiance input must be [x(3), SH deg 4 (16), n(3), h(32), h_appear(<=8)]", who);
    *d = ColorNetDev{(const __half *)c->W1, (const __half *)c->b1, (const __half *)c->W2, (const __half *)c->b2, (const __half *)c->R1,
                     (const __half *)c->rb1, (const __half *)c->R2, (const __half *)c->rb2, (const __half *)c->R3, (const __half *)c->rb3,
                     c->width, c->rad_width, c->rad_in, c->n_appear, c->beta, {c->nablas_scale[0], c->nablas_scale[1], c->nablas_scale[2]}};
    return 0;
}
inline unsigned tiles_grid(int64_t n, int ctas_per_sm) {
    const int64_t n_tiles = (n + kTile - 1) / kTile, wave = (int64_t)sm_count() * ctas_per_sm;
    return (unsigned)(n_tiles < wave ? n_tiles : wave);
}
}  // namespace

namespace nsb { extern std::atomic<int> g_opt_color_tma; }

extern "C" int64_t nsb_color_tile_bytes(int64_t n) { return ((n + kTile - 1) / kTile) * (int64_t)kTileBytes; }

extern "C" int nsb_fused_color_fwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x, const float *rays_o,
                                   const float *rays_d, const int64_t *ridx, const float *t, const float *view_dirs, const float *h_appear,
                                   int64_t n, int32_t max_level, float *sdf, float *nablas, float *rgb, float *x_out, void *act_z, void *act_x,
                                   void *act_y1, void *act_y2, const nsb_occ_collect *collect, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(meta && params_half && net && sdf && nablas && rgb && view_dirs, "nsb_fused_color_fwd: NULL argument");
    NSB_REQUIRE(x || (rays_o && rays_d && t), "nsb_fused_color_fwd: need x or (rays_o, rays_d, t)");
    NSB_REQUIRE((act_z && act_x && act_y1 && act_y2) || (!act_z && !act_x && !act_y1 && !act_y2), "nsb_fused_color_fwd: pass all four activation buffers or none");
    PLMeta m;
    ColorNetDev d;
    if (int rc = make_net(net, meta, &m, &d, "nsb_fused_color_fwd")) return rc;
    NSB_REQUIRE(d.n_appear == 0 || h_appear, "nsb_fused_color_fwd: h_appear is NULL but the net has %d appearance channels", d.n_appear);
    constexpr int kSmem = 2 * kTileBytes + 2 * HW * NF * 2 + 2 * XW * XW * 2 + kTile * tc::acc_stride(64) * 4 + 1024;
    opt_in_smem(k_color_fwd, kSmem);
    PointSrc ps{x, rays_o, rays_d, t, ridx};
    OccCollect oc{nullptr, 1, 1, 1, 0.f};
    if (collect && collect->grid_pcl) oc = OccCollect{collect->grid_pcl, collect->res[0], collect->res[1], collect->res[2], collect->inv_s};
    k_color_fwd<<<tiles_grid(n, 2), kTile, kSmem, (cudaStream_t)stream>>>(m, (const __half *)params_half, d, ps, view_dirs, h_appear, n,
                                                                          max_level < 0 ? -1 : max_level, sdf, nablas, rgb, x_out, (uint8_t *)act_z,
                                                                          (uint8_t *)act_x, (uint8_t *)act_y1, (uint8_t *)act_y2, oc, dn.a);
    return check_launch("nsb_fused_color_fwd");
}

extern "C" int nsb_fused_color_bwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_color_net *net, const float *x, const float *rays_o,
                                   const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level, const void *act_z,
                                   const void *act_x, const void *act_y1, const void *act_y2, const float *rgb, const float *g_sdf,
                                   const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1, float *d_b1,
                                   float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3, float *d_rb3,
                                   void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(meta && params_half && net && act_z && act_x && act_y1 && act_y2 && rgb && dh_scratch, "nsb_fused_color_bwd: NULL argument");
    NSB_REQUIRE(d_grid && d_W1 && d_b1 && d_W2 && d_b2 && d_R1 && d_rb1 && d_R2 && d_rb2 && d_R3 && d_rb3, "nsb_fused_color_bwd: NULL gradient buffer");
    NSB_REQUIRE(x || (rays_o && rays_d && t), "nsb_fused_color_bwd: need x or (rays_o, rays_d, t)");
    PLMeta m;
    ColorNetDev d;
    if (int rc = make_net(net, meta, &m, &d, "nsb_fused_color_bwd")) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const float *dh = nullptr;
    if (g_rgb) {
        constexpr int kSmemR = 3 * kTileBytes + 2 * kTile * 80 * 2 + XW * XW * 2 + NF * XW * 2 + kTile * tc::acc_stride(64 + 2 * 80) * 4 + 1024;   // 1 CTA / SM
        opt_in_smem(k_color_rad_bwd<true>, kSmemR);
        opt_in_smem(k_color_rad_bwd<false>, kSmemR);
        if (g_opt_color_tma.load())
            k_color_rad_bwd<true><<<tiles_grid(n, 1), kTile, kSmemR, s>>>(d, (const uint8_t *)act_x, (const uint8_t *)act_y1, (const uint8_t *)act_y2, rgb, g_rgb, n,
                                                                          dh_scratch, d_R1, d_rb1, d_R2, d_rb2, d_R3, d_rb3, dn.a);
        else
            k_color_rad_bwd<false><<<tiles_grid(n, 1), kTile, kSmemR, s>>>(d, (const uint8_t *)act_x, (const uint8_t *)act_y1, (const uint8_t *)act_y2, rgb, g_rgb, n,
                                                                           dh_scratch, d_R1, d_rb1, d_R2, d_rb2, d_R3, d_rb3, dn.a);
        if (int rc = check_launch("nsb_fused_color_bwd(radiance)")) return rc;
        dh = dh_scratch;
    }
    constexpr int kSmemS = 3 * kTileBytes + 2 * kTile * 48 * 2 + 2 * HW * NF * 2 + kTileBytes + kTile * tc::acc_stride(96 + 2 * 48) * 4 + 1024;   // 1 CTA / SM
    opt_in_smem(k_color_sdf_bwd<true>, kSmemS);
    opt_in_smem(k_color_sdf_bwd<false>, kSmemS);
    PointSrc ps{x, rays_o, rays_d, t, ridx};
    if (g_opt_color_tma.load() >= 2)
        k_color_sdf_bwd<true><<<tiles_grid(n, 1), kTile, kSmemS, s>>>(m, (const __half *)params_half, d, ps, (const uint8_t *)act_z, (const uint8_t *)act_x,
                                                                      g_nablas, g_sdf, dh, n, max_level < 0 ? -1 : max_level, d_grid, d_W1, d_b1, d_W2, d_b2, dn.a);
    else
        k_color_sdf_bwd<false><<<tiles_grid(n, 1), kTile, kSmemS, s>>>(m, (const __half *)params_half, d, ps, (const uint8_t *)act_z, (const uint8_t *)act_x,
                                                                       g_nablas, g_sdf, dh, n, max_level < 0 ? -1 : max_level, d_grid, d_W1, d_b1, d_W2, d_b2, dn.a);
    return check_launch("nsb_fused_color_bwd(sdf)");
}
