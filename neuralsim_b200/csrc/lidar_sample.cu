// The LiDAR training batch of one frame, drawn inside the step: LidarDataset.sample_merged (dataio/data_loader/lidar_loader.py:119-204)
// in its merged_weighted / merged_equal modes, then the beams moved to world (MultiRaysLidarBundle.get_selected_rays,
// app/resources/observers/lidars.py:65-78, 169-175).
//
// The host splits num_rays over the frame's lidars once per frame (neuralsim_b200/lidar_sampler.py: the reference's numpy arithmetic) and
// stores the split in the frame's table row.  The reference then draws, lidar by lidar in index order, torch.randint(cumu[li],
// cumu[li + 1], [num_li]) -- random_from_to with range = count_li < 2^32, the uint32 curand4 branch (torch_uniform.cuh) -- each draw at
// the offset the previous one left, and gathers rays_o, rays_d, ranges and li at the drawn indices.  Ray r of the batch is element
// r - ray_start[li] of lidar li's draw, li the lidar whose ray segment [ray_start[li], ray_start[li + 1]) holds r.
//   k_lidar_sample      thread per ray (grid-stride): its lidar, its draw, its beam, the (lidar, frame) transform; no atomics
// World rays: o_w[i] = fma(R[i][2], o[2], fma(R[i][1], o[1], fma(R[i][0], o[0], t[i]))) and d_w[i] = fma(R[i][2], d[2], fma(R[i][1], d[1],
// R[i][0] * d[0])), each fma rounded once (__fmaf_rn), so the result is fixed whatever the compiler contracts.  The reference sums
// (R * x).sum(-1) + t in torch's reduction order; the two agree to a few ulp of sum_j |R[i][j] x[j]| (+ |t[i]|), not bit for bit.
#include "nsb_common.cuh"
#include "torch_uniform.cuh"

namespace nsb {

__global__ void __launch_bounds__(256)
k_lidar_sample(const int64_t *__restrict__ table, const int64_t *__restrict__ frame, const int64_t *__restrict__ rng, int64_t n, int64_t grid_cap,
               const float *__restrict__ rays_o, const float *__restrict__ rays_d, const float *__restrict__ ranges, const float *__restrict__ l2w,
               float *__restrict__ out_o, float *__restrict__ out_d, float *__restrict__ out_ranges, int64_t *__restrict__ li_out,
               int64_t *__restrict__ fidx_out, int64_t *__restrict__ rng_next) {
    const int64_t fi = *frame;
    const int64_t *row = table + fi * NSB_LIDAR_TABLE_WIDTH;
    const uint64_t seed = (uint64_t)rng[0], o0 = (uint64_t)rng[1];
    if (rng_next && blockIdx.x == 0 && threadIdx.x == 0) {
        rng_next[0] = rng[0];
        rng_next[1] = (int64_t)(o0 + (uint64_t)row[NSB_LIDAR_ROW_INC]);
    }
    const int64_t *ray_start = row + NSB_LIDAR_ROW_RAY_START, *cumu = row + NSB_LIDAR_ROW_CUMU, *draw_off = row + NSB_LIDAR_ROW_DRAW_OFF;
    const int64_t n_lidars = row[NSB_LIDAR_ROW_N_LIDARS];
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        // the first lidar whose segment ends past r (lidars that draw nothing have empty segments and are passed over)
        int li = 0;
#pragma unroll
        for (int k = 1; k < NSB_LIDAR_MAX; ++k)
            li += (k < n_lidars && r >= ray_start[k]) ? 1 : 0;
        const int64_t j = r - ray_start[li], num = ray_start[li + 1] - ray_start[li];
        const int64_t beam = torch_randint_at(seed, o0 + (uint64_t)draw_off[li], j, torch_uniform_stride(num, grid_cap),
                                              (uint64_t)(cumu[li + 1] - cumu[li]), cumu[li]);
        const int64_t b = row[NSB_LIDAR_ROW_DATA_OFF] + beam;
        const float *T = l2w + (row[NSB_LIDAR_ROW_POSE_BASE] + li) * 12;
        const float ox = rays_o[3 * b], oy = rays_o[3 * b + 1], oz = rays_o[3 * b + 2];
        const float dx = rays_d[3 * b], dy = rays_d[3 * b + 1], dz = rays_d[3 * b + 2];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float *Ri = T + 4 * i;
            out_o[3 * r + i] = __fmaf_rn(Ri[2], oz, __fmaf_rn(Ri[1], oy, __fmaf_rn(Ri[0], ox, Ri[3])));
            out_d[3 * r + i] = __fmaf_rn(Ri[2], dz, __fmaf_rn(Ri[1], dy, __fmul_rn(Ri[0], dx)));
        }
        out_ranges[r] = ranges[b];
        li_out[r] = li;
        fidx_out[r] = fi;
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_lidar_sample(const int64_t *table, const int64_t *frame, const int64_t *rng, int64_t n, const float *rays_o, const float *rays_d,
                                const float *ranges, const float *l2w, float *out_rays_o, float *out_rays_d, float *out_ranges, int64_t *li,
                                int64_t *rays_fidx, int64_t *rng_next, void *stream) {
    NSB_REQUIRE(n >= 1 && n < ((int64_t)1 << 31), "nsb_lidar_sample: n = %lld rays, must lie in [1, 2^31)", (long long)n);
    NSB_REQUIRE(table && frame && rng && rays_o && rays_d && ranges && l2w && out_rays_o && out_rays_d && out_ranges && li && rays_fidx,
                "nsb_lidar_sample: NULL argument");
    k_lidar_sample<<<wave_grid(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(table, frame, rng, n, torch_rand_grid_cap(), rays_o, rays_d, ranges, l2w,
                                                                          out_rays_o, out_rays_d, out_ranges, li, rays_fidx, rng_next);
    return check_launch("nsb_lidar_sample");
}
