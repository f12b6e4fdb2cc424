// Occupancy-grid EMA maintenance on the device (SURVEY.md §8 a11 / f3), sm_90a.
//
// Reference: OccGridEma._step_update_occ (nr3d_lib/models/accelerations/occgrid/ema_single.py:176-190) ->
//   occ_val = normalized_logistic_density(sdf_half, inv_s)            (occgrid/utils.py:63-68, maths/common.py:122-133)
//   gidx    = ((pts / 2 + 0.5) * res).long().clamp(0, res - 1)        (ema_single.py:179)
//   + the evidence collected while rendering: the non-zero cells of _occ_val_grid_pcl, which is then zeroed (:180-186)
//   new     = scatter_max(occ_val, gidx, out = decay * grid); grid[touched] = new[touched]   (utils.py:89-101, torch_scatter)
//   occ     = grid > threshold                                       (utils.py:84-87, consider_mean = False)
// The reference runs this as ~15 ATen / torch_scatter launches over 4 x 2^20 points and a nonzero() host sync; here: fill the
// evidence scratch, ONE scatter pass over the points (atomic max on the non-negative fp32 bit pattern), ONE pass over the cells that
// merges the collected evidence, applies decay + max on the touched cells, thresholds, and (optionally) bit-packs the grid for the
// marcher.  A cell is "touched" when a point fell into it -- also when that point's evidence is exactly 0 (then the cell only
// decays), which is why the scratch starts at -1 rather than 0.
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ float r16_(float v) { return __half2float(__float2half_rn(v)); }

// every op of (1 / cosh(clamp(inv_s x / 2, -20, 20)))^2 rounds to fp16: the reference evaluates it on a half tensor
__device__ __forceinline__ float occ_evidence(float sdf, float inv_s) {
    const float a = fminf(fmaxf(r16_(r16_(__fmul_rn(sdf, inv_s)) * 0.5f), -20.f), 20.f);
    const float r = r16_(__fdiv_rn(1.f, r16_(coshf(a))));
    return r16_(__fmul_rn(r, r));
}

__global__ void __launch_bounds__(256) k_occ_fill(float *__restrict__ ev, int64_t cells) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (int64_t)gridDim.x * blockDim.x) ev[c] = -1.f;
}

// pts [n,3] in [-1,1]^3 (network space), val [n]: sdf (is_sdf) or ready-made evidence >= 0
__global__ void __launch_bounds__(256)
k_occ_scatter(const float *__restrict__ pts, const float *__restrict__ val, int64_t n, int rx, int ry, int rz, float inv_s, int is_sdf,
              float *__restrict__ ev, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float ux = __fadd_rn(__fmul_rn(pts[i * 3], 0.5f), 0.5f), uy = __fadd_rn(__fmul_rn(pts[i * 3 + 1], 0.5f), 0.5f),
                    uz = __fadd_rn(__fmul_rn(pts[i * 3 + 2], 0.5f), 0.5f);
        const int ix = min(max((int)__fmul_rn(ux, (float)rx), 0), rx - 1);
        const int iy = min(max((int)__fmul_rn(uy, (float)ry), 0), ry - 1);
        const int iz = min(max((int)__fmul_rn(uz, (float)rz), 0), rz - 1);
        float v = is_sdf ? occ_evidence(val[i], inv_s) : val[i];
        if (!(v >= 0.f)) v = 0.f;                              // evidence is a density in [0, 1]; NaN / negative inputs only mark the cell
        atomicMax(reinterpret_cast<int *>(ev) + ((int64_t)(ix * ry + iy) * rz + iz), __float_as_int(v));      // -1.f < 0 <= bits(v)
    }
}

__global__ void __launch_bounds__(256)
k_occ_finalize(float *__restrict__ ev, float *__restrict__ pcl, float *__restrict__ grid, uint8_t *__restrict__ occ, uint32_t *__restrict__ bits,
               int64_t cells, float decay, float thre, const int64_t *__restrict__ skip) {
    if (skip && *skip) return;                                 // an update that drew nothing changes nothing, the collected evidence included
    for (int64_t c0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ll; c0 < cells; c0 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = c0 + (threadIdx.x & 31);
        bool o = false;
        if (c < cells) {
            float e = ev[c];
            if (pcl) {
                const float p = pcl[c];
                if (p != 0.f) { e = fmaxf(e, p); pcl[c] = 0.f; }         // collected evidence: the non-zero cells (ema_single.py:180-186)
            }
            float g = grid[c];
            if (e >= 0.f) { g = fmaxf(__fmul_rn(decay, g), e); grid[c] = g; }
            o = g > thre;
            occ[c] = o ? 1 : 0;
        }
        const uint32_t m = __ballot_sync(0xffffffffu, o);
        if (bits && (threadIdx.x & 31) == 0 && c0 < cells) bits[c0 >> 5] = m;
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_occ_ema_update(const float *pts, const float *val, int64_t n, int32_t val_is_sdf, float inv_s, int32_t rx, int32_t ry, int32_t rz,
                                  float *pcl_or_null, float *occ_val_grid, uint8_t *occ_grid, uint32_t *occ_bits_or_null, float ema_decay,
                                  float occ_thre, float *scratch_cells, void *stream) {
    NSB_REQUIRE(occ_val_grid && occ_grid && scratch_cells, "nsb_occ_ema_update: NULL grid");
    NSB_REQUIRE(rx > 0 && ry > 0 && rz > 0, "nsb_occ_ema_update: bad resolution");
    NSB_REQUIRE(n == 0 || (pts && val), "nsb_occ_ema_update: NULL points");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)rx * ry * rz;
    k_occ_fill<<<wave_grid(cells, 256, 8), 256, 0, s>>>(scratch_cells, cells);
    if (int rc = check_launch("nsb_occ_ema_update(fill)")) return rc;
    if (n > 0) {
        k_occ_scatter<<<wave_grid(n, 256, 8), 256, 0, s>>>(pts, val, n, rx, ry, rz, inv_s, val_is_sdf, scratch_cells, nullptr);
        if (int rc = check_launch("nsb_occ_ema_update(scatter)")) return rc;
    }
    k_occ_finalize<<<wave_grid(cells, 256, 8), 256, 0, s>>>(scratch_cells, pcl_or_null, occ_val_grid, occ_grid, occ_bits_or_null, cells, ema_decay, occ_thre,
                                                            nullptr);
    return check_launch("nsb_occ_ema_update(finalize)");
}

extern "C" int nsb_occ_ema_update_count(const float *pts, const float *val, const int64_t *n_dev, int64_t n_capacity, int32_t val_is_sdf, float inv_s,
                                        int32_t rx, int32_t ry, int32_t rz, float *pcl_or_null, float *occ_val_grid, uint8_t *occ_grid,
                                        uint32_t *occ_bits_or_null, float ema_decay, float occ_thre, float *scratch_cells, const int64_t *skip_or_null,
                                        void *stream) {
    NSB_REQUIRE(occ_val_grid && occ_grid && scratch_cells && n_dev, "nsb_occ_ema_update_count: NULL grid or count");
    NSB_REQUIRE(rx > 0 && ry > 0 && rz > 0, "nsb_occ_ema_update_count: bad resolution");
    NSB_REQUIRE(n_capacity == 0 || (pts && val), "nsb_occ_ema_update_count: NULL points");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)rx * ry * rz;
    k_occ_fill<<<wave_grid(cells, 256, 8), 256, 0, s>>>(scratch_cells, cells);
    if (int rc = check_launch("nsb_occ_ema_update_count(fill)")) return rc;
    if (n_capacity > 0) {
        k_occ_scatter<<<wave_grid(n_capacity, 256, 8), 256, 0, s>>>(pts, val, n_capacity, rx, ry, rz, inv_s, val_is_sdf, scratch_cells, n_dev);
        if (int rc = check_launch("nsb_occ_ema_update_count(scatter)")) return rc;
    }
    k_occ_finalize<<<wave_grid(cells, 256, 8), 256, 0, s>>>(scratch_cells, pcl_or_null, occ_val_grid, occ_grid, occ_bits_or_null, cells, ema_decay, occ_thre,
                                                            skip_or_null);
    return check_launch("nsb_occ_ema_update_count(finalize)");
}
