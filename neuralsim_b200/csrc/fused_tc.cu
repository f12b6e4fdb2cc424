// Fused forward_sdf and its backward with the decoder GEMMs on the Hopper tensor cores (wgmma), sm_90a.
//
// One CTA = 128 threads = one warpgroup = one tile of 128 points; thread r owns point r for the gather and the scatter (the ray-tiled
// query, MODE 2 below, gives the gather and the MMA + epilogue to different warps of a larger CTA, with the same per-row arithmetic):
//   gather   thread r walks the L (1..24) LoTD levels of its point (8 corner loads each); every level's two fp16 features go
//            straight into its row of the A tile in shared memory (core-matrix layout of tc_util.cuh), columns 2L..NF-1 are zero
//   MMA      the warpgroup issues wgmma (M=64, N=64, K=16) x NF/16 per 64-row half: Z[128 x 64] (fp32, registers) = H[128 x NF] . W1^T
//            (NF = 32 feature columns for tables of 1..16 levels, 48 for 17..24: feature_cols, fused_tc_common.cuh)
//   epilogue bias + Softplus(beta) with the autocast rounding points on the accumulator fragments, the 64 -> 1 layer as a
//            dot product per row (16 hidden units per lane, summed over the lane quad) -> sdf[r]
// The loop over levels is rolled on purpose (instruction cache: a fully unrolled gather is several thousand instructions).
// W1 is staged once per persistent CTA.  Numerics: the fp16 rounding points of the reference's autocast graph (DESIGN.md).
#include "fused_tc_common.cuh"

namespace nsb {

// MODE 0: points x[n,3];  MODE 1: x = o[ridx[i]] + d[ridx[i]] t[i] in the given (ray-major) order;
// MODE 2: the same packed samples traversed RAY-TILED: a tile = 32 packs (rays) x 4 consecutive samples, lane = ray, warp = sample
//         ordinal.  The 32 packs of group g are order[32 g .. 32 g + 32) -- nsb_ray_block_order puts an 8 x 4 pixel block of an image
//         there -- or, with order == NULL, packs 32 g .. 32 g + 32 (a 32 x 1 strip of one image row).  For coherent rays the 32 lanes
//         of a gather instruction then sit in neighbouring cells -> few 128 B lines per request, and a block touches fewer lines than
//         a strip (DESIGN.md §5).  sdf is written to the packed slot, so nothing downstream changes.  Incoherent rays (random training
//         pixels) keep MODE 1: locality along the ray.
// CTAs of k_fused_sdf_tc per SM in the persistent grid of modes 0 and 1 (points / rays).  5 would fit (90 registers, ~13 KB of shared
// memory), but their gather is L1-bound and more warps gathering at once evict each other's lines: on an H100 (NVIDIA H100 80GB HBM3,
// 700 W) the boundary query of an 800x600 frame, then walked in 32 x 1 strips, took 5.8 ms per launch at 4 CTAs / SM, 7.3-7.4 ms at 5
// and 6.5 ms at 6 (bench.py, alternated).
constexpr int kSdfCtasPerSM = 4;

// MODE 2 is warp-specialised: a CTA = one consumer warpgroup (warps 0..3: MMA + epilogue + store) and kPackSets sets of 4 producer warps
// (the gather), which hand 128-row A tiles over a ring of kPackSlots shared-memory slots guarded by "full" / "empty" mbarriers.  Tile j of
// a CTA (its groups in grid-stride order, each group's sample ordinals 4 at a time) is gathered by set j % kPackSets into slot
// j % kPackSlots; the consumer takes the tiles in order.  The gather warps thus never wait on a CTA barrier, the MMA or the SFU epilogue,
// and the consumer's epilogue of one tile overlaps the gather of the next ones.  One CTA of 5 sets (20 gather warps) per SM, launched at
// 80 registers and split by setmaxnreg, 72 for the gather and 120 for the 64 accumulators of the epilogue; 7 slots (~71 KB).  On an H100
// (NVIDIA H100 80GB HBM3, 700 W) the boundary query of an 800x600 frame took 4.31-4.36 ms per step at this size, 4.62-4.65 ms with 4 sets
// (16 gather warps, 96 registers, no split) and 5.14-5.19 ms before the split into roles (5 CTAs of 128 threads per SM) (bench.py,
// alternated, DESIGN.md §6).  2 CTAs of 2 sets per SM would cap every thread at 80 registers: the epilogue spills.
constexpr int kPackSets = 5, kPackSlots = 7, kPackCtasPerSM = 1;
// registers per thread after the split (setmaxnreg): 20 producer warps x 72 + 4 consumer warps x 120 = the 768 x 80 the CTA is launched with
constexpr int kPackProducerRegs = 72, kPackConsumerRegs = 120;
static_assert(kPackSets * kTile * kPackProducerRegs + kTile * kPackConsumerRegs <= kTile * (1 + kPackSets) * 80, "register split");
constexpr int kPackThreads = kTile * (1 + kPackSets);
// ~71 KB at NF = 32, ~98 KB at NF = 48: one CTA per SM either way
template <int NF>
constexpr int pack_smem() { return kPackSlots * (kTile * NF * 2 + kTile * 12) + HW * NF * 2 + 2 * HW * 4 + kPackSlots * 20 + 16 + 128; }

// one slot of the ring: the A tile (8 KB, 12 KB at NF = 48) and, per row, the output index (-1: no sample) and the occupancy voxel of the sample
struct PackSlots {
    uint8_t *a;                            // [kPackSlots][kTile * NF * 2 bytes]
    int64_t *out;                          // [kPackSlots][kTile]
    int *voxel;                            // [kPackSlots][kTile]
    uint64_t *full, *empty;                // [kPackSlots]: 128 producer arrivals / 128 consumer arrivals per phase
    int *end;                              // [kPackSlots]: 1 = no tile, the CTA's work is done
};

// the producer side of MODE 2: set `set` walks every group of this CTA, gathers its tiles j (j % kPackSets == set) into the ring and,
// when it owns the index past the last tile, posts the end marker there.  Lane = pack (ray), warp w of the set = sample ordinal k0 + w.
template <int NF>
__device__ __forceinline__ void sdf_packs_produce(const PLMeta &m, const __half *__restrict__ grid, uint32_t La, const float *__restrict__ rays_o,
                                                  const float *__restrict__ rays_d, const float *__restrict__ t, const int64_t *__restrict__ pack_infos,
                                                  const int64_t *__restrict__ pack_ray, const int64_t *__restrict__ order, int64_t n_packs,
                                                  const OccCollect &oc, const PackSlots &ring, int set, int w, int lane) {
    const int row = w * 32 + lane;
    const int64_t n_groups = (n_packs + 31) / 32;
    uint32_t j = 0;                                            // the CTA's tile counter
    for (int64_t g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const int64_t slot = g * 32 + lane;
        int64_t first = 0, cnt = 0, ray = 0;
        if (slot < n_packs) {
            const int64_t p = order ? order[slot] : slot;
            first = pack_infos[2 * p]; cnt = pack_infos[2 * p + 1]; ray = pack_ray ? pack_ray[p] : p;
        }
        int max_n = (int)cnt;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) max_n = max(max_n, __shfl_xor_sync(0xffffffffu, max_n, s));
        const uint32_t tiles = (uint32_t)(max_n + 3) / 4;
        uint32_t mine = j + (uint32_t)((set - (int)(j % kPackSets) + kPackSets) % kPackSets);   // my first tile index >= j
        if (mine < j + tiles) {
            float o[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f};
            if (cnt > 0) {
#pragma unroll
                for (int q = 0; q < 3; ++q) { o[q] = rays_o[ray * 3 + q]; d[q] = rays_d[ray * 3 + q]; }
            }
            for (; mine < j + tiles; mine += kPackSets) {
                const int k = (int)(mine - j) * 4 + w;
                const bool valid = k < cnt;
                float xs[3] = {0.f, 0.f, 0.f};
                if (valid) {
                    const float tt = t[first + k];
#pragma unroll
                    for (int q = 0; q < 3; ++q) xs[q] = __fmaf_rn(d[q], tt, o[q]);
                }
#pragma unroll
                for (int q = 0; q < 3; ++q) xs[q] = to_table_space(xs[q]);
                const uint32_t s = mine % kPackSlots;
                tc::mbar_wait(&ring.empty[s], ((mine / kPackSlots) & 1u) ^ 1u);
                gather_row_to_tile<kTile, NF>(m, grid, xs, La, ring.a + s * (kTile * NF * 2), row);
                ring.out[s * kTile + row] = valid ? first + k : -1;
                ring.voxel[s * kTile + row] = (valid && oc.pcl) ? occ_voxel(oc, xs) : 0;
                tc::fence_async_smem();                        // the tile's generic-proxy writes -> visible to the wgmma (async proxy)
                tc::mbar_arrive(&ring.full[s]);
            }
        }
        j += tiles;
    }
    if ((int)(j % kPackSets) == set) {                         // the end marker, in tile j's place
        const uint32_t s = j % kPackSlots;
        tc::mbar_wait(&ring.empty[s], ((j / kPackSlots) & 1u) ^ 1u);
        if (row == 0) ring.end[s] = 1;
        tc::mbar_arrive(&ring.full[s]);
    }
}

template <int MODE, int NF>
__global__ void __launch_bounds__(MODE == 2 ? kPackThreads : kTile, MODE == 2 ? kPackCtasPerSM : 0)
k_fused_sdf_tc(const PLMeta m, const __half *__restrict__ grid, const DecoderDevTC dec, const float *__restrict__ x,
               const float *__restrict__ rays_o, const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
               const float *__restrict__ t, int64_t n, int max_level, float *__restrict__ sdf, const int64_t *__restrict__ pack_infos,
               const int64_t *__restrict__ pack_ray, const int64_t *__restrict__ order, int64_t n_packs, const OccCollect oc,
               const int64_t *__restrict__ n_dev, const int32_t *__restrict__ ml_dev) {
    const int tid = threadIdx.x;
    const uint32_t La = active_levels(max_level, ml_dev, m.n_pseudo);
    if constexpr (MODE == 2) {
        const int warp = tid >> 5, lane = tid & 31;
        n_packs = eff_n(n_packs, n_dev);                       // device-resident count (nsb_bind_device_counts)
        extern __shared__ uint8_t dyn_smem[];
        uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 127) & ~uintptr_t(127));
        PackSlots ring;
        ring.a = base;                                                            // kPackSlots x 8 KB : the A tiles
        uint8_t *sB = ring.a + kPackSlots * (kTile * NF * 2);                     //  4 KB : W1 [64 x NF]
        ring.out = reinterpret_cast<int64_t *>(sB + HW * NF * 2);
        ring.voxel = reinterpret_cast<int *>(ring.out + kPackSlots * kTile);
        float *sb1 = reinterpret_cast<float *>(ring.voxel + kPackSlots * kTile), *sW2 = sb1 + HW;
        ring.full = reinterpret_cast<uint64_t *>(sW2 + HW);
        ring.empty = ring.full + kPackSlots;
        ring.end = reinterpret_cast<int *>(ring.empty + kPackSlots);
        float *sb2 = reinterpret_cast<float *>(ring.end + kPackSlots);
        if (tid < kTile) {
            stage_W1<NF>(dec, sB, tid);
            stage_decoder_vectors(dec, sb1, sW2, sb2, tid);
        }
        if (tid < kPackSlots) {
            tc::mbar_init(&ring.full[tid], kTile);
            tc::mbar_init(&ring.empty[tid], kTile);
            ring.end[tid] = 0;
        }
        tc::fence_mbar_init();
        tc::fence_async_smem();
        __syncthreads();
        if (warp >= 4) {                                       // producers
            tc::setmaxnreg_dec<kPackProducerRegs>();
            sdf_packs_produce<NF>(m, grid, La, rays_o, rays_d, t, pack_infos, pack_ray, order, n_packs, oc, ring, (warp - 4) >> 2, warp & 3, lane);
            return;
        }
        tc::setmaxnreg_inc<kPackConsumerRegs>();
        // consumer warpgroup: tile j from slot j % kPackSlots -> MMA -> slot free -> epilogue -> sdf of each row from its quad's lane 0
        const uint32_t b_addr = tc::smem_u32(sB);
        const SoftplusK spk(dec.beta);
        const float b2 = *sb2;
        for (uint32_t j = 0;; ++j) {
            const uint32_t s = j % kPackSlots;
            tc::mbar_wait(&ring.full[s], (j / kPackSlots) & 1u);
            if (ring.end[s]) break;
            float z[2][HW / 2];
            tc::mma_m128<HW, 0, 0, NF / 16>(z, tc::kmajor(tc::smem_u32(ring.a + s * (kTile * NF * 2)), kTile), tc::kmajor(b_addr, HW), false);
            int64_t out_i[2][2];
            int vox[2][2];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int row = h * 64 + tc::frag_row(i);
                    out_i[h][i] = ring.out[s * kTile + row];
                    vox[h][i] = ring.voxel[s * kTile + row];
                }
            tc::mbar_arrive(&ring.empty[s]);                   // the MMA has read the tile, the row data are in registers
            float v[2][2];
            sdf_rows_of_frags(z, sb1, sW2, spk, v);
            if ((lane & 3) == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        if (out_i[h][i] < 0) continue;
                        const float r = r16(v[h][i] + b2);
                        sdf[out_i[h][i]] = r;
                        if (oc.pcl) occ_collect_voxel(oc, vox[h][i], r);
                    }
            }
        }
    } else {
        n = eff_n(n, n_dev);                                   // device-resident count (nsb_bind_device_counts)
        __shared__ __align__(128) uint8_t sA[kTile * NF * 2];    // 8 KB (NF = 48: 12 KB) : features, chunk-major core-matrix layout
        __shared__ __align__(128) uint8_t sB[HW * NF * 2];       // 4 KB (6 KB) : W1 [64 x NF], same layout
        __shared__ float sb1[HW], sW2[HW], srow[kTile];
        __shared__ float sb2;
        stage_W1<NF>(dec, sB, tid);
        stage_decoder_vectors(dec, sb1, sW2, &sb2, tid);
        tc::fence_async_smem();
        __syncthreads();
        const SdfTile ctx{m, grid, La, sA, tc::smem_u32(sA), tc::smem_u32(sB), srow, sb1, sW2, sb2, SoftplusK(dec.beta)};
        const int64_t n_tiles = (n + kTile - 1) / kTile;
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int64_t i = tile * kTile + tid;
            const bool valid = i < n;
            float xs[3];
            load_point(PointSrc{x, rays_o, rays_d, t, ridx}, MODE == 1, i, valid, xs);
            const float v = sdf_of_tile<NF>(ctx, xs, tid);
            if (valid) {
                sdf[i] = v;
                if (oc.pcl) occ_collect_point(oc, xs, v);
            }
        }
    }
}

// =====================================================================================================================
// Backward of forward_sdf wrt. the LoTD table and the decoder weights, one kernel, nothing saved by the forward.
// Per tile of 128 points (thread r = point r for the gather and the scatter), d = dL/dsdf[r]:
//   recompute  gather -> A tile [H | 1 | 0..];  MMA1: Z = H.W1^T (registers);  z = fp16(Z + b1); s = sigmoid(beta z), a = fp16(softplus)
//   G tile [128 x 128] fp16 :=  [ dz_0..dz_63 | d*a_0..d*a_63 ],  dz_j = d * w2_j * s_j, written from the Z fragments
//              (the reference rounds grad_z to fp16 at the same place, layers.py autocast backward)
//   MMA2: dH[128 x NF]  = dZ . W1                 A = G cols 0..63 (K-major), B = W1^T tile          -> registers
//   MMA3: X[64 x NF+8] += dZ^T . [H | 1 | 0..]    both operands are the tiles above read MN-major, K = the 128 points: [ dW1 | db1 ]
//   MMA4: V[64 x 8]    += (d*a)^T . [1 0..]       column 0 = dW2
//              X and V are register fragments carried over all tiles of the persistent CTA
//   dH staged as fp32 rows in G (free once the MMAs have completed) -> scatter into the fp32 table gradient (8 corners x L levels,
//   red.global.add.v2.f32);  db2 via a warp sum.  Columns 2L..NF-1 of H and dH are zero and neither scattered nor flushed.
// =====================================================================================================================
// Resident CTAs per SM of the persistent grid of k_sdf_bwd_tc: 51 KB of shared memory and 120 registers fit four.  On an H100
// (NVIDIA H100 80GB HBM3, 400 W power limit) the kernel took 2.43 / 2.43 ms per bench step at 2 CTAs / SM, 2.24 / 2.19 ms at 3 and
// 2.16 / 2.13 ms at 4 (profiles/bwd_kernels.py, the three builds alternated in one run; 2.48 ms before its sums moved to registers).
constexpr int kSdfBwdCtasPerSM = 4;
// The 48-column form (tables of 17..24 levels) needs 58 KB of shared memory per CTA (wider H tile, W1 and W1^T): three fit an SM.
constexpr int kSdfBwdWideCtasPerSM = 3;
template <int NF>
constexpr int sdf_bwd_ctas() { return NF == 32 ? kSdfBwdCtasPerSM : kSdfBwdWideCtasPerSM; }
// dynamic shared memory of k_sdf_bwd_tc: [H | 1 | 0..], G, W1, W1^T and the 128 B alignment slack (50 KB at NF = 32, 58 KB at 48)
template <int NF>
constexpr int sdf_bwd_smem() { return (kTile * (NF + 8) + kTile * 128 + HW * NF + NF * HW) * 2 + 128; }
static_assert(sdf_bwd_smem<32>() == (128 * 40 + 128 * 128 + 64 * 32 + 32 * 64) * 2 + 128, "the 32-column budget is unchanged");

// kXGrad (points from rays only) adds the gradient of every point's ray, the depths t being constants: the scatter loads the corners of
// each level it scatters to once more and adds J^T dH to the point's table-space input gradient g, which is mapped to network space and
// written as row i_ (the kernel's row, not keep[i_]) of gx_out [n, 8] = [g | t g | 0 0]; k_ray_row_sum adds the rows up per ray.
template <bool FROM_RAYS, bool kXGrad, int NF>
__global__ void __launch_bounds__(kTile, sdf_bwd_ctas<NF>())
k_sdf_bwd_tc(const PLMeta m, const __half *__restrict__ grid, const DecoderDevTC dec, const float *__restrict__ x,
             const float *__restrict__ rays_o, const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
             const float *__restrict__ t, const float *__restrict__ d_sdf, int64_t n, int max_level, float *__restrict__ d_grid,
             float *__restrict__ d_W1, float *__restrict__ d_b1, float *__restrict__ d_W2, float *__restrict__ d_b2,
             const int64_t *__restrict__ keep, const int64_t *__restrict__ n_dev, float *__restrict__ gx_out, const int32_t *__restrict__ ml_dev) {
    n = eff_n(n, n_dev);
    const uint32_t La = active_levels(max_level, ml_dev, m.n_pseudo);
    constexpr int NX = NF + 8, GW = 128;                      // NX: features + [1,0,..] chunk; GW: dz | d*a
    constexpr int kS = tc::acc_stride(NF);                    // staged dH rows for the scatter: 18 KB (26 KB), aliasing G
    extern __shared__ uint8_t dyn_smem[];                     // 50 KB (NF = 48: 58 KB) of tiles (> the 48 KB static limit)
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dyn_smem) + 127) & ~uintptr_t(127));
    uint8_t *sA = tiles;                                      // 10 KB (14 KB) : [H | 1 | 0..]
    uint8_t *sG = sA + kTile * NX * 2;                        // 32 KB : [dz | d*a]
    uint8_t *sB = sG + kTile * GW * 2;                        //  4 KB (6 KB) : W1   [64 x NF]  (B of MMA1)
    uint8_t *sBT = sB + HW * NF * 2;                          //  4 KB (6 KB) : W1^T [NF x 64]  (B of MMA2)
    float *stage = reinterpret_cast<float *>(sG);
    static_assert(kTile * kS * 4 <= kTile * GW * 2, "the staged dH rows must fit in G");
    __shared__ float sb1[HW], sW2[HW], sdd[kTile];
    __shared__ float sdb2;

    const int tid = threadIdx.x, lane = tid & 31;
    stage_W1<NF>(dec, sB, tid);
    stage_W1T<NF>(dec, sBT, tid);
    stage_decoder_vectors(dec, sb1, sW2, nullptr, tid);
    *reinterpret_cast<uint4 *>(sA + (NF / 8) * (kTile * 16) + tid * 16) = make_uint4(0x00003C00u, 0, 0, 0);   // constant chunk: [1,0,..]
    float xacc[NX / 2], vacc[4];
#pragma unroll
    for (int k = 0; k < NX / 2; ++k) xacc[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) vacc[k] = 0.f;
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
        load_point(PointSrc{x, rays_o, rays_d, t, ridx}, FROM_RAYS, i, valid, xs);
        const float dd = valid ? d_sdf[i] : 0.f;
        sdd[tid] = dd;                                           // read by the fragment owners of my row
        gather_row_to_tile<kTile, NF>(m, grid, xs, La, sA, tid);
        tc::fence_async_smem();
        __syncthreads();
        {
            float z[2][HW / 2];
            tc::mma_m128<HW, 0, 0, NF / 16>(z, tc::kmajor(a_addr, kTile), tc::kmajor(b_addr, HW), false);   // Z = H . W1^T
            // ---- G on the Z fragments: dz (chunks 0..7) and d*a (chunks 8..15); G is read by no MMA in flight
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = h * 64 + tc::frag_row(r);
                    const float d = sdd[row];
#pragma unroll
                    for (int c = 0; c < HW / 8; ++c) {
                        const int col = tc::frag_col(c);
                        float dz[2], da[2];
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const float zz = r16(z[h][4 * c + 2 * r + j] + sb1[col + j]);
                            float a, s;
                            softplus_as(zz, spk, a, s);
                            da[j] = d * r16(a);
                            dz[j] = d * sW2[col + j] * s;
                        }
                        tc::st_pair_f16(sG, tc::pair_off<kTile>(row, col), dz[0], dz[1]);
                        tc::st_pair_f16(sG, tc::pair_off<kTile>(row, HW + col), da[0], da[1]);
                    }
                }
        }
        tc::fence_async_smem();
        __syncthreads();                                         // G is complete
        float dh_fr[2][NF / 2];
        tc::mma_m128<NF, 0, 0, HW / 16>(dh_fr, tc::kmajor(g_addr, kTile), tc::kmajor(bt_addr, NF), false);                          // dH = dZ . W1 : K = 64 hidden
        tc::mma_m64<NX, 1, 1, kTile / 16>(xacc, tc::mnmajor(g_addr, kTile), tc::mnmajor(a_addr, kTile), true);                      // X += dZ^T . [H|1] : K = 128 points
        tc::mma_m64<8, 1, 1, kTile / 16>(vacc, tc::mnmajor(g_addr + 8 * (kTile * 16), kTile), tc::mnmajor(a_addr + (NF / 8) * (kTile * 16), kTile), true);   // V += (d*a)^T . 1
        first_tile = false;
        const float dsum = warp_sum(dd);
        if (lane == 0 && dsum != 0.f) atomicAdd(&sdb2, dsum);
        __syncthreads();                                         // the MMAs reading G have completed
        tc::frag_store<NF>(dh_fr, stage, kS, 0);
        __syncthreads();
        // ---- my dH row -> scatter into the table gradient; only the reductions are predicated on "this point carries gradient".
        const bool active = valid && dd != 0.f;
        const bool warp_active = __any_sync(0xffffffffu, active);
        float gx[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (uint32_t g4 = 0; g4 * 4 < La; ++g4) {
            float dh[8];
            tc::acc_ld8(stage, kS, tid, g4 * 8, dh);                // 4 levels x 2 features
            if (!warp_active) continue;
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q) {
                const uint32_t p = g4 * 4 + q;
                if (p >= La) continue;                                                       // uniform
                uint32_t cell[8];
                float w[8], a[8], b[8], fr[3], sc[3];
                if constexpr (kXGrad) level_cells3(m, p, xs, cell, w, fr, sc);
                else level_cells3(m, p, xs, cell, w);
                const float g0 = active ? dh[2 * q] : 0.f, g1 = active ? dh[2 * q + 1] : 0.f;
                if constexpr (kXGrad) level_input_grad(m, p, grid, cell, fr, sc, g0, g1, gx);
#pragma unroll
                for (int c = 0; c < 8; ++c) { a[c] = g0 * w[c]; b[c] = g1 * w[c]; }
                if (warp_merge_updates(cell_key3(m, p, xs), active, a, b, lane)) {   // neighbouring samples, same cell
                    float2 *gp = level_grad_ptr(m, p, d_grid);
#pragma unroll
                    for (int c = 0; c < 8; ++c) red_add2(gp + cell[c], a[c], b[c]);
                }
            }
        }
        if constexpr (kXGrad) {
            if (valid) {
                float g[3];
#pragma unroll
                for (int d = 0; d < 3; ++d) g[d] = input_grad_to_net(gx[d]);
                const float tt = t[i];
                float4 *o = reinterpret_cast<float4 *>(gx_out + i_ * 8);
                o[0] = make_float4(g[0], g[1], g[2], __fmul_rn(tt, g[0]));
                o[1] = make_float4(__fmul_rn(tt, g[1]), __fmul_rn(tt, g[2]), 0.f, 0.f);
            }
        }
        __syncthreads();                                         // tiles + staged rows free for the next iteration
    }
    // ---- flush the CTA's weight-gradient accumulators: X = [dW1 | db1], V column 0 = dW2
    if (!first_tile) {                                           // uniform per CTA
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = tc::frag_row(r);
            if (row >= dec.width) continue;
#pragma unroll
            for (int c = 0; c <= NF / 8; ++c)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int col = tc::frag_col(c) + j;
                    if (col < dec.nh) atomicAdd(d_W1 + row * dec.nh + col, xacc[4 * c + 2 * r + j]);
                    else if (col == NF) atomicAdd(d_b1 + row, xacc[4 * c + 2 * r + j]);
                }
            if (tc::frag_col(0) == 0) atomicAdd(d_W2 + row, vacc[2 * r]);
        }
        if (tid == 0) atomicAdd(d_b2, sdb2);
    }
}

}  // namespace nsb

using namespace nsb;

// mode 0: x[n,3];  1: (rays_o, rays_d, ridx, t)[n];  2: ray-tiled packs (pack_infos[n_packs,2], pack_ray[n_packs] or NULL,
// pack_order[n_packs] or NULL, t, sdf packed)
extern "C" int nsb_fused_sdf_tc_launch(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                       const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                                       int32_t max_level, float *sdf, void *stream, int mode, const int64_t *pack_infos,
                                       const int64_t *pack_ray, const int64_t *pack_order, int64_t n_packs, const nsb_occ_collect *collect) {
    const DevCounts dn = take_counts();
    const int32_t *ml_dev = take_max_level();
    PLMeta m;
    DecoderDevTC d;
    if (int rc = make_decoder(meta, dec, &m, &d, "nsb_fused_sdf (tensor-core)")) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int ml = max_level < 0 ? -1 : max_level;
    const __half *g = (const __half *)params_half;
    const OccCollect oc = occ_collect_of(collect);
    const unsigned tiles = persistent_grid((n + kTile - 1) / kTile, kSdfCtasPerSM);
    auto launch = [&](auto nf) -> int {
        constexpr int NF = decltype(nf)::value;
        if (mode == 2) {      // a work unit of mode 2 is a group of 32 packs
            constexpr int kPackSmem = pack_smem<NF>();
            opt_in_smem(k_fused_sdf_tc<2, NF>, kPackSmem);
            if (int rc = require_ctas_per_sm(k_fused_sdf_tc<2, NF>, kPackThreads, kPackSmem, kPackCtasPerSM, "nsb_fused_sdf (packs)")) return rc;
            k_fused_sdf_tc<2, NF><<<persistent_grid((n_packs + 31) / 32, kPackCtasPerSM), kPackThreads, kPackSmem, s>>>(
                m, g, d, nullptr, rays_o, rays_d, nullptr, t, n, ml, sdf, pack_infos, pack_ray, pack_order, n_packs, oc, dn.a, ml_dev);
        } else if (mode == 1)
            k_fused_sdf_tc<1, NF><<<tiles, kTile, 0, s>>>(m, g, d, nullptr, rays_o, rays_d, ridx, t, n, ml, sdf, nullptr, nullptr, nullptr, 0, oc, dn.a, ml_dev);
        else
            k_fused_sdf_tc<0, NF><<<tiles, kTile, 0, s>>>(m, g, d, x, nullptr, nullptr, nullptr, nullptr, n, ml, sdf, nullptr, nullptr, nullptr, 0, oc, dn.a, ml_dev);
        return check_launch("nsb_fused_sdf(tc)");
    };
    return feature_cols(m.n_pseudo) == 32 ? launch(std::integral_constant<int, 32>{}) : launch(std::integral_constant<int, 48>{});
}

extern "C" int nsb_fused_sdf_bwd(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                 const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf,
                                 int64_t n, int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2,
                                 void *stream) {
    return nsb_fused_sdf_bwd_indexed(meta, params_half, dec, x, rays_o, rays_d, ridx, t, d_sdf, nullptr, n, max_level, d_grid, d_W1, d_b1, d_W2, d_b2,
                                     stream);
}

// the backward of the fused SDF query, with kXGrad the per-point ray rows and their per-ray sums (k_ray_row_sum, color_tc.cu)
template <bool kXGrad>
static int sdf_bwd(const char *who, const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x, const float *rays_o,
                   const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf, const int64_t *keep, int64_t n, int32_t max_level,
                   float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *gx_scratch, const int64_t *ray_map, float *d_rays_o,
                   float *d_rays_d, void *stream) {
    const DevCounts dn = take_counts();
    const int32_t *ml_dev = take_max_level();
    if (n == 0) return 0;
    NSB_REQUIRE(meta && params_half && dec && d_sdf && d_grid && d_W1 && d_b1 && d_W2 && d_b2, "%s: NULL argument", who);
    NSB_REQUIRE(x || (rays_o && rays_d && t), "%s: need x or (rays_o, rays_d, t)", who);
    if (kXGrad) NSB_REQUIRE(!x && gx_scratch, "%s: ray gradients need the points as rays (x NULL) and gx_scratch", who);
    PLMeta m;
    DecoderDevTC d;
    if (int rc = make_decoder(meta, dec, &m, &d, who)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int ml = max_level < 0 ? -1 : max_level;
    auto launch = [&](auto nf) -> int {
        constexpr int NF = decltype(nf)::value, kBwdSmem = sdf_bwd_smem<NF>(), kCtas = sdf_bwd_ctas<NF>();
        auto kern = x == nullptr ? k_sdf_bwd_tc<true, kXGrad, NF> : k_sdf_bwd_tc<false, false, NF>;
        opt_in_smem(kern, kBwdSmem);
        if (int rc = require_ctas_per_sm(kern, kTile, kBwdSmem, kCtas, who)) return rc;
        const unsigned grid = persistent_grid((n + kTile - 1) / kTile, kCtas);
        kern<<<grid, kTile, kBwdSmem, s>>>(m, (const __half *)params_half, d, x, x ? nullptr : rays_o, x ? nullptr : rays_d, x ? nullptr : ridx,
                                           x ? nullptr : t, d_sdf, n, ml, d_grid, d_W1, d_b1, d_W2, d_b2, keep, dn.a, gx_scratch, ml_dev);
        return check_launch(who);
    };
    if (int rc = feature_cols(m.n_pseudo) == 32 ? launch(std::integral_constant<int, 32>{}) : launch(std::integral_constant<int, 48>{})) return rc;
    if (kXGrad) {
        if (!d_rays_o && !d_rays_d) return 0;
        k_ray_row_sum<8><<<row_sum_blocks(n), 256, 0, s>>>(gx_scratch, ridx, keep, n, 6, ray_map, RowSumOut{{d_rays_o, d_rays_d, nullptr}, 3}, dn.a);
        return check_launch("nsb_fused_sdf_bwd_rays(ray sum)");
    }
    return 0;
}

extern "C" int nsb_fused_sdf_bwd_indexed(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                         const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf,
                                         const int64_t *keep, int64_t n, int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2,
                                         float *d_b2, void *stream) {
    return sdf_bwd<false>("nsb_fused_sdf_bwd", meta, params_half, dec, x, rays_o, rays_d, ridx, t, d_sdf, keep, n, max_level, d_grid, d_W1, d_b1, d_W2,
                          d_b2, nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int nsb_fused_sdf_bwd_rays(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *rays_o,
                                      const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf, const int64_t *keep, int64_t n,
                                      int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *gx_scratch,
                                      const int64_t *ray_map, float *d_rays_o, float *d_rays_d, void *stream) {
    return sdf_bwd<true>("nsb_fused_sdf_bwd_rays", meta, params_half, dec, nullptr, rays_o, rays_d, ridx, t, d_sdf, keep, n, max_level, d_grid, d_W1,
                         d_b1, d_W2, d_b2, gx_scratch, ray_map, d_rays_o, d_rays_d, stream);
}
