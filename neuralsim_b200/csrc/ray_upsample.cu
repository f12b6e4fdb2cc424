// The no-grad up-sampling half of the NeuS query as ONE persistent kernel (the default when the quantiles are not perturbed).
// For every ray that marched into occupied voxels it replaces, per up-sampling stage, the launches
//   k_fused_sdf_tc (sdf of the marched / new samples) -> k_upsample_cdf -> k_invert_cdf_shared_u -> k_merge_vals
// (graphics/neus.py:_query_fused, reference neus_ray_query.py:861-905) and keeps the ray's samples in shared memory in between.
// A CTA of 128 threads owns a group of 4 consecutive hit rays: warp w <-> ray w for the per-ray stages; for the SDF evaluations the four rays'
// pending samples are concatenated into 128-point tiles of the usual gather -> wgmma -> SFU pipeline (sdf_of_tile, fused_tc_common.cuh).
// The per-ray stage bodies warp_upsample_cdf, invert_cdf_one and warp_merge are the ones k_upsample_cdf, k_invert_cdf_shared_u and
// k_merge_vals call (neus_device.cuh), on the ray's samples in shared memory here; tests/test_ray_upsample_edges_gpu.py pins the kernel
// (and its group-to-group state below) to the stage kernels bit for bit and to float64 at its edges.
// Output: fine[n_hit, sum(n_fine)] -- what `torch.cat(fine_stages, -1)` is on the multi-kernel path.  A ray whose samples do not fit the
// per-ray shared-memory capacity (kCap) works on a slice of a global scratch buffer instead (same code: the stage bodies take plain
// pointers).  Overflow: overflow[j] is set to 1 (and nothing else is written to it) for a ray with more than long_cap - merged marched
// samples (merged = the samples of every stage but the last), or, without scratch (nsb_upsample_persistent), more than kCap - merged; such
// a ray is not processed: its row of `fine` is not written and none of its points is collected.  With long_cap sized from max_steps by the
// caller (graphics/neus_fused.py: max_steps + merged + 64) a marched ray never overflows.
// An empty pack (n = 0) is skipped the same way: its row is not written and nothing is collected for it (the stage kernels write NaN
// samples for it instead).  Production never passes one: the hit rays of the march hold >= 1 sample.
// Training-time sample collection (accel.collect_samples on every SDF query, renderer_mixin.py:154-164) is done in-kernel as in k_fused_sdf_tc.
#include "fused_tc_common.cuh"
#include "neus_device.cuh"

namespace nsb {

constexpr int kG = 4;            // rays per group = warps per CTA
constexpr int kCap = 192;        // samples of one ray held in shared memory (marched + all merged stages but the last)
constexpr int kMaxFine = 64;     // samples of one stage
constexpr int kMaxStage = 4;
constexpr int kCtasPerSM = 5;    // persistent grid; the scratch buffer holds one slice per CTA of that grid

struct UpsampleArgs {
    int n_stage, use_estimate;
    int n_fine[kMaxStage];
    float inv_s[kMaxStage];      // upsample_inv_s * factor_i, as the host computes it
    const float *u[kMaxStage];   // the n_fine[i] quantiles of stage i (linspace(0, 1, n + 2)[1:-1], made by torch)
    float eps, thre;
};

// NF: the feature columns of the A tile (feature_cols: 32 for tables of 1..16 levels, 48 for 17..24; 37 KB of static shared memory
// instead of 31 KB, still five CTAs per SM)
template <int NF>
__global__ void __launch_bounds__(kTile)
k_upsample_persistent(const PLMeta m, const __half *__restrict__ grid, const DecoderDevTC dec, const float *__restrict__ rays_o,
                      const float *__restrict__ rays_d, const float *__restrict__ t_starts, const int64_t *__restrict__ pack_infos,
                      const int64_t *__restrict__ ridx_hit, int64_t n_hit, int max_level, const UpsampleArgs ua, float *__restrict__ fine_all,
                      int nf_total, int32_t *__restrict__ overflow, float *__restrict__ scratch, int long_cap, const OccCollect oc,
                      const int64_t *__restrict__ n_dev, const int32_t *__restrict__ ml_dev) {
    n_hit = eff_n(n_hit, n_dev);
    __shared__ __align__(128) uint8_t sA[kTile * NF * 2];
    __shared__ __align__(128) uint8_t sB[HW * NF * 2];
    __shared__ float sb1[HW], sW2[HW], srow[kTile];
    __shared__ float sb2;
    __shared__ float s_t[2][kG][kCap], s_sdf[2][kG][kCap], s_cdf[kG][kCap];
    __shared__ float s_fine[kG][kMaxFine], s_fsdf[kG][kMaxFine];
    __shared__ float s_o[kG][3], s_d[kG][3];
    __shared__ int s_n[kG];
    __shared__ float *p_t[2][kG], *p_sdf[2][kG], *p_cdf[kG];          // where ray q's samples live: shared memory, or its slice of `scratch`

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    stage_W1<NF>(dec, sB, tid);
    stage_decoder_vectors(dec, sb1, sW2, &sb2, tid);
    tc::fence_async_smem();
    __syncthreads();
    const SdfTile ctx{m, grid, active_levels(max_level, ml_dev, m.n_pseudo), sA, tc::smem_u32(sA), tc::smem_u32(sB), srow, sb1, sW2, sb2, SoftplusK(dec.beta)};
    int room = kCap;                                     // a ray must hold its marched samples + every merged stage
    for (int i = 0; i + 1 < ua.n_stage; ++i) room -= ua.n_fine[i];

    const int64_t n_groups = (n_hit + kG - 1) / kG;
    for (int64_t g = blockIdx.x; g < n_groups; g += gridDim.x) {
        // ---- load the group: warp w <-> ray g*4 + w
        const int64_t j = g * kG + warp;
        int n = 0;
        int64_t first = 0;
        if (j < n_hit) {
            first = pack_infos[2 * j];
            n = (int)pack_infos[2 * j + 1];
        }
        bool in_smem = n <= room;
        if (!in_smem && (scratch == nullptr || n > long_cap - (kCap - room))) {      // longer than the scratch slice: flagged, row not written
            if (lane == 0) overflow[j] = 1;
            n = 0;
            in_smem = true;
        }
        if (lane == 0) {
            float *g = scratch ? scratch + ((size_t)blockIdx.x * kG + warp) * 5 * (size_t)long_cap : nullptr;
            p_t[0][warp] = in_smem ? s_t[0][warp] : g;
            p_t[1][warp] = in_smem ? s_t[1][warp] : g + long_cap;
            p_sdf[0][warp] = in_smem ? s_sdf[0][warp] : g + 2 * (size_t)long_cap;
            p_sdf[1][warp] = in_smem ? s_sdf[1][warp] : g + 3 * (size_t)long_cap;
            p_cdf[warp] = in_smem ? s_cdf[warp] : g + 4 * (size_t)long_cap;
        }
        __syncwarp();
        if (n > 0 && lane < 3) {
            const int64_t ray = ridx_hit[j];
            s_o[warp][lane] = rays_o[ray * 3 + lane];
            s_d[warp][lane] = rays_d[ray * 3 + lane];
        }
        for (int k = lane; k < n; k += 32) p_t[0][warp][k] = t_starts[first + k];
        if (lane == 0) s_n[warp] = n;
        __syncthreads();
        int cur = 0;
        // ---- sdf of the marched samples: the four rays' samples concatenated into 128-point tiles
        {
            const int total = s_n[0] + s_n[1] + s_n[2] + s_n[3];
            for (int base = 0; base < total; base += kTile) {
                int r = base + tid, q = 0;
                const bool valid = r < total;
                if (valid) { while (r >= s_n[q]) { r -= s_n[q]; ++q; } }
                float xs[3] = {0.f, 0.f, 0.f};
                if (valid) {
                    const float tt = p_t[0][q][r];
#pragma unroll
                    for (int c = 0; c < 3; ++c) xs[c] = __fmaf_rn(s_d[q][c], tt, s_o[q][c]);
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) xs[c] = to_table_space(xs[c]);
                const float v = sdf_of_tile<NF>(ctx, xs, tid);
                if (valid) {
                    p_sdf[0][q][r] = v;
                    if (oc.pcl) occ_collect_point(oc, xs, v);
                }
            }
            __syncthreads();
        }
        int off = 0;
        for (int i = 0; i < ua.n_stage; ++i) {
            const int nf = ua.n_fine[i];
            // ---- per ray: cdf of the up-sampling weights, then the nf inverse-cdf samples
            if (n > 0) {
                warp_upsample_cdf(p_sdf[cur][warp], p_t[cur][warp], n, ua.inv_s[i], ua.use_estimate, ua.eps, ua.thre, p_cdf[warp], lane);
                for (int q = lane; q < nf; q += 32) {
                    const float f = invert_cdf_one(p_t[cur][warp], p_cdf[warp], (uint32_t)n, ua.u[i][q]);
                    s_fine[warp][q] = f;
                    fine_all[j * nf_total + off + q] = f;
                }
            }
            off += nf;
            __syncthreads();
            if (i + 1 == ua.n_stage) break;              // (the reference also merges after the last stage; nothing reads that result)
            // ---- sdf of the new samples of the four rays: one (under-filled) tile per 128
            for (int base = 0; base < kG * nf; base += kTile) {
                const int r = base + tid, q = r / nf, k = r - q * nf;
                const bool valid = r < kG * nf && s_n[q] > 0;
                float xs[3] = {0.f, 0.f, 0.f};
                if (valid) {
                    const float tt = s_fine[q][k];
#pragma unroll
                    for (int c = 0; c < 3; ++c) xs[c] = __fmaf_rn(s_d[q][c], tt, s_o[q][c]);
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) xs[c] = to_table_space(xs[c]);
                const float v = sdf_of_tile<NF>(ctx, xs, tid);
                if (valid) {
                    s_fsdf[q][k] = v;
                    if (oc.pcl) occ_collect_point(oc, xs, v);
                }
            }
            __syncthreads();
            // ---- per ray: merge the new samples (and their sdf) into the ray
            if (n > 0) {
                warp_merge(p_t[cur][warp], p_sdf[cur][warp], n, s_fine[warp], s_fsdf[warp], nf, p_t[cur ^ 1][warp], p_sdf[cur ^ 1][warp], lane);
                n += nf;
            }
            cur ^= 1;
            __syncthreads();
        }
        __syncthreads();                                 // the group's shared memory is free for the next one
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_upsample_persistent(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *rays_o,
                                       const float *rays_d, const float *t_starts, const int64_t *pack_infos, const int64_t *ridx_hit, int64_t n_hit,
                                       int32_t max_level, int32_t n_stage, const int32_t *n_fine, const float *inv_s_stage, const float *const *u_stage,
                                       int32_t use_estimate_alpha, float early_stop_eps, float alpha_thre, float *fine_all, int32_t *overflow,
                                       void *stream) {
    return nsb_upsample_rays(meta, params_half, dec, rays_o, rays_d, t_starts, pack_infos, ridx_hit, n_hit, max_level, n_stage, n_fine, inv_s_stage, u_stage,
                             use_estimate_alpha, early_stop_eps, alpha_thre, fine_all, overflow, nullptr, 0, nullptr, stream);
}

static unsigned upsample_grid(int64_t n_hit) { return persistent_grid((n_hit + kG - 1) / kG, kCtasPerSM); }

// per CTA of the grid: kG rays x 5 arrays (t, sdf of two generations, cdf) of long_cap floats
extern "C" int64_t nsb_upsample_rays_scratch_floats(int64_t n_hit_cap, int32_t long_cap) {
    return (int64_t)upsample_grid(n_hit_cap) * kG * 5 * (int64_t)long_cap;
}

extern "C" int nsb_upsample_rays(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *rays_o,
                                 const float *rays_d, const float *t_starts, const int64_t *pack_infos, const int64_t *ridx_hit, int64_t n_hit,
                                 int32_t max_level, int32_t n_stage, const int32_t *n_fine, const float *inv_s_stage, const float *const *u_stage,
                                 int32_t use_estimate_alpha, float early_stop_eps, float alpha_thre, float *fine_all, int32_t *overflow,
                                 float *scratch, int32_t long_cap, const nsb_occ_collect *collect, void *stream) {
    const DevCounts dn = take_counts();
    const int32_t *ml_dev = take_max_level();
    if (n_hit == 0) return 0;
    NSB_REQUIRE(meta && params_half && dec && rays_o && rays_d && t_starts && pack_infos && ridx_hit && n_fine && inv_s_stage && u_stage && fine_all && overflow,
                "nsb_upsample_persistent: NULL argument");
    NSB_REQUIRE(n_stage >= 1 && n_stage <= kMaxStage, "nsb_upsample_persistent: 1..%d stages", kMaxStage);
    PLMeta m;
    DecoderDevTC d;
    if (int rc = make_decoder(meta, dec, &m, &d, "nsb_upsample_persistent")) return rc;
    UpsampleArgs ua{};
    ua.n_stage = n_stage;
    ua.use_estimate = use_estimate_alpha;
    ua.eps = early_stop_eps;
    ua.thre = alpha_thre;
    int nf_total = 0, merged = 0;
    for (int i = 0; i < n_stage; ++i) {
        NSB_REQUIRE(n_fine[i] >= 1 && n_fine[i] <= kMaxFine && u_stage[i], "nsb_upsample_persistent: 1..%d samples per stage", kMaxFine);
        ua.n_fine[i] = n_fine[i];
        ua.inv_s[i] = inv_s_stage[i];
        ua.u[i] = u_stage[i];
        nf_total += n_fine[i];
        if (i + 1 < n_stage) merged += n_fine[i];
    }
    NSB_REQUIRE(merged < kCap, "nsb_upsample_persistent: the merged stages alone exceed the per-ray capacity");
    NSB_REQUIRE(scratch == nullptr || long_cap > kCap, "nsb_upsample_rays: long_cap must exceed the shared-memory capacity (%d)", kCap);
    auto kern = feature_cols(m.n_pseudo) == 32 ? k_upsample_persistent<32> : k_upsample_persistent<48>;
    kern<<<upsample_grid(n_hit), kTile, 0, (cudaStream_t)stream>>>(
        m, (const __half *)params_half, d, rays_o, rays_d, t_starts, pack_infos, ridx_hit, n_hit, max_level < 0 ? -1 : max_level, ua, fine_all, nf_total,
        overflow, scratch, long_cap, occ_collect_of(collect), dn.a, ml_dev);
    return check_launch("nsb_upsample_rays");
}
