// Occupancy-grid ray marching for sm_90a (single grid and batched grids, AABB contraction).
//
// Replaces `_occ_grid.ray_marching / batched_ray_marching`
// (nr3d_lib/csrc/occ_grid/src/ray_marching.cu:17-244, batched_marching.cu:18-287).
// The sample counts / voxel ids are integer results and are kept bit-exact with the reference by issuing the
// same sequence of fp32 roundings (explicit _rn intrinsics; the sequence was read off the SASS nvcc 12.9 emitted
// for the reference at -O3 for sm_100a -- see oracle/march.c and DESIGN.md; that the reference's sm_90a build gives the same
// counts, samples and voxel ids bit for bit is checked against its stored outputs, tests/test_ref_parity_gpu.py).
// Differences in design: the bool grid is bit-packed into shared memory once per CTA when it fits
// (64^3 -> 32 KB), so the inner loop never touches global memory; rays are processed grid-stride by
// a wave-sized grid.
#include "nsb_common.cuh"

namespace nsb {

struct MarchArgs {
    int64_t n_rays;
    const float *rays_o, *rays_d, *t_min, *t_max, *roi;
    const int32_t *batch_inds;
    int rx, ry, rz;
    const uint8_t *grid;
    float step_size, max_step_size, dt_gamma;
    uint32_t max_steps;
    const int32_t *packed_info;
    int32_t *num_steps;
    float *t_starts, *t_ends;
    int32_t *ridx, *gidx, *bidx;
    const int64_t *ray_list;       // second round only: the rays to re-march (those with samples); NULL = all n_rays
    int64_t n_list;
    const uint32_t *grid_bits;     // optional: the grid already packed 32 cells / word (nsb_pack_occ_bits), copied instead of re-packed per CTA
    const int64_t *n_dev;          // optional device-resident count (nsb_bind_device_counts): of the rays (first round: num_steps of the rays
                                   // between it and n_rays is written as 0) or of the listed rays (second round)
    float *rec_t;                  // REC only (first round): sample k of ray i is also recorded at rec_t[i max_steps + k], so that the second
                                   // march of a small batch (latency of the longest ray, twice) becomes a copy (k_march_compact)
};

__device__ __forceinline__ float calc_dt(float t, float dt_gamma, float dt_min, float dt_max) {
    return fminf(fmaxf(__fmul_rn(t, dt_gamma), dt_min), dt_max);
}

__device__ __forceinline__ float next_axis(float unit, float dir, float inv_dir, int res, float extent) {
    const float r = (float)res;
    const float a = __fmaf_rn(r, unit, 0.5f);
    const float b = __fmaf_rn(copysignf(1.0f, dir), 0.5f, a);
    const float f = floorf(b);
    const float d = __fmaf_rn(r, -unit, f);
    return __fmul_rn(__fdiv_rn(__fmul_rn(d, inv_dir), r), extent);
}

template <bool SMEM_BITS, bool REC = false>
__global__ void __launch_bounds__(256) k_ray_marching(const MarchArgs a) {
    extern __shared__ uint32_t s_bits[];
    const int64_t cells = (int64_t)a.rx * a.ry * a.rz;
    if (SMEM_BITS) {
        // pack 32 bools per word; each thread builds whole words so no atomics are needed
        const int64_t words = (cells + 31) >> 5;
        if (a.grid_bits) {
            for (int64_t w = threadIdx.x; w < words; w += blockDim.x) s_bits[w] = a.grid_bits[w];
        } else
        for (int64_t w = threadIdx.x; w < words; w += blockDim.x) {
            uint32_t bits = 0;
            const int64_t base = w << 5;
#pragma unroll 8
            for (int k = 0; k < 32; ++k) {
                const int64_t c = base + k;
                if (c < cells && a.grid[c]) bits |= (1u << k);
            }
            s_bits[w] = bits;
        }
        __syncthreads();
    }
    const bool first_round = (a.packed_info == nullptr);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_work = a.ray_list ? a.n_list : a.n_rays;
    const int64_t n_live = eff_n(n_work, a.n_dev);
    for (int64_t j_ = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j_ < n_work; j_ += stride) {
        if (j_ >= n_live) {
            if (first_round && !a.ray_list) { a.num_steps[j_] = 0; continue; }
            break;
        }
        const int64_t i = a.ray_list ? a.ray_list[j_] : j_;
        int b = 0;
        if (a.batch_inds) {
            b = a.batch_inds[i];
            if (b < 0) {  // batched_marching.cu:55 leaves num_steps uninitialised; we define it as 0
                if (first_round) a.num_steps[i] = 0;
                continue;
            }
        }
        const float *roi = a.roi + 6 * b;
        const uint8_t *grid = a.grid + cells * b;
        const float ox = a.rays_o[i * 3], oy = a.rays_o[i * 3 + 1], oz = a.rays_o[i * 3 + 2];
        const float dx = a.rays_d[i * 3], dy = a.rays_d[i * 3 + 1], dz = a.rays_d[i * 3 + 2];
        const float ix = __fdiv_rn(1.0f, dx), iy = __fdiv_rn(1.0f, dy), iz = __fdiv_rn(1.0f, dz);
        const float near = a.t_min[i], far = a.t_max[i];
        const float r0 = roi[0], r1 = roi[1], r2 = roi[2], r3 = roi[3], r4 = roi[4], r5 = roi[5];
        const float ex = __fsub_rn(r3, r0), ey = __fsub_rn(r4, r1), ez = __fsub_rn(r5, r2);
        const float dt_min = a.step_size, dt_max = a.max_step_size;
        uint32_t max_steps = a.max_steps;
        int64_t base = 0;
        if (!first_round) {
            base = a.packed_info[i * 2];
            max_steps = (uint32_t)a.packed_info[i * 2 + 1];
        }
        uint32_t j = 0;
        float t0 = near;
        float dt = calc_dt(t0, a.dt_gamma, dt_min, dt_max);
        float t1 = __fadd_rn(t0, dt);
        float t_mid = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
        while (t_mid < far && j < max_steps) {
            const float px = __fmaf_rn(t_mid, dx, ox), py = __fmaf_rn(t_mid, dy, oy), pz = __fmaf_rn(t_mid, dz, oz);
            const float ux = __fdiv_rn(__fsub_rn(px, r0), ex);
            const float uy = __fdiv_rn(__fsub_rn(py, r1), ey);
            const float uz = __fdiv_rn(__fsub_rn(pz, r2), ez);
            bool occupied = false;
            int gi = -1;
            if (!(px < r0 || px > r3 || py < r1 || py > r4 || pz < r2 || pz > r5)) {
                const int cx = min(max((int)__fmul_rn(ux, (float)a.rx), 0), a.rx - 1);
                const int cy = min(max((int)__fmul_rn(uy, (float)a.ry), 0), a.ry - 1);
                const int cz = min(max((int)__fmul_rn(uz, (float)a.rz), 0), a.rz - 1);
                gi = (cx * a.ry + cy) * a.rz + cz;
                occupied = SMEM_BITS ? ((s_bits[gi >> 5] >> (gi & 31)) & 1u) : (grid[gi] != 0);
            }
            if (occupied) {
                if (!first_round) {
                    a.t_starts[base + j] = t0;
                    if (a.t_ends) a.t_ends[base + j] = t1;
                    a.ridx[base + j] = (int32_t)i;
                    if (a.gidx) a.gidx[base + j] = (int32_t)(gi + b * cells);   // batched: flat over [B, X, Y, Z] (batched_marching.cu:62,115)
                    if (a.bidx) a.bidx[base + j] = b;
                } else if (REC) {
                    a.rec_t[i * (int64_t)a.max_steps + j] = t0;
                }
                ++j;
                t0 = t1;
                t1 = __fadd_rn(t0, calc_dt(t0, a.dt_gamma, dt_min, dt_max));
                t_mid = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
            } else {
                const float tx = next_axis(ux, dx, ix, a.rx, ex);
                const float ty = next_axis(uy, dy, iy, a.ry, ey);
                const float tz = next_axis(uz, dz, iz, a.rz, ez);
                const float t = fmaxf(fminf(fminf(tx, ty), tz), 0.0f);
                const float t_target = __fadd_rn(t_mid, t);
                float tt = t_mid;
                do { tt = __fadd_rn(tt, dt_min); } while (tt < t_target);
                t_mid = tt;
                dt = calc_dt(t_mid, a.dt_gamma, dt_min, dt_max);
                t0 = __fmaf_rn(dt, -0.5f, t_mid);
                t1 = __fmaf_rn(dt, 0.5f, t_mid);
            }
        }
        if (first_round) a.num_steps[i] = (int32_t)j;
    }
}

// Second round of a recorded march: sample k of listed ray j -> slot first + k of the packed arrays.  One warp per ray.
__global__ void __launch_bounds__(256) k_march_compact(const float *__restrict__ rec_t, uint32_t max_steps, const int32_t *__restrict__ packed_info,
                                                       const int64_t *__restrict__ ray_list, int64_t n_list, const int64_t *__restrict__ n_dev,
                                                       float *__restrict__ t_starts, int32_t *__restrict__ ridx) {
    const int lane = threadIdx.x & 31;
    const int64_t n_live = eff_n(n_list, n_dev);
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_live; j += nw) {
        const int64_t i = ray_list ? ray_list[j] : j;
        const int64_t first = packed_info[i * 2];
        const int32_t cnt = packed_info[i * 2 + 1];
        const float *src = rec_t + i * (int64_t)max_steps;
        for (int32_t k = lane; k < cnt; k += 32) {
            t_starts[first + k] = src[k];
            ridx[first + k] = (int32_t)i;
        }
    }
}

__global__ void __launch_bounds__(256) k_pack_occ_bits(const uint8_t *__restrict__ grid, int64_t cells, uint32_t *__restrict__ words) {
    const int64_t n_words = (cells + 31) >> 5;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        uint32_t bits = 0;
        const int64_t base = w << 5;
#pragma unroll 8
        for (int k = 0; k < 32; ++k) {
            const int64_t c = base + k;
            if (c < cells && grid[c]) bits |= (1u << k);
        }
        words[w] = bits;
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_pack_occ_bits(const uint8_t *grid_binary, int64_t cells, uint32_t *words, void *stream) {
    if (cells == 0) return 0;
    NSB_REQUIRE(grid_binary && words, "nsb_pack_occ_bits: NULL argument");
    k_pack_occ_bits<<<wave_grid((cells + 31) / 32, 256, 4), 256, 0, (cudaStream_t)stream>>>(grid_binary, cells, words);
    return check_launch("nsb_pack_occ_bits");
}

extern "C" int nsb_ray_marching(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min,
                                const float *t_max, const float *roi, const int32_t *batch_inds, int32_t rx, int32_t ry,
                                int32_t rz, const uint8_t *grid_binary, float step_size, float max_step_size,
                                float dt_gamma, uint32_t max_steps, const int32_t *packed_info, int32_t *num_steps,
                                float *t_starts, float *t_ends, int32_t *ridx, int32_t *gidx, int32_t *bidx, void *stream) {
    return nsb_ray_marching_listed(n_rays, rays_o, rays_d, t_min, t_max, roi, batch_inds, rx, ry, rz, grid_binary, step_size, max_step_size, dt_gamma,
                                   max_steps, packed_info, num_steps, t_starts, t_ends, ridx, gidx, bidx, nullptr, 0, nullptr, stream);
}

extern "C" int nsb_ray_marching_listed(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min, const float *t_max,
                                       const float *roi, const int32_t *batch_inds, int32_t rx, int32_t ry, int32_t rz,
                                       const uint8_t *grid_binary, float step_size, float max_step_size, float dt_gamma, uint32_t max_steps,
                                       const int32_t *packed_info, int32_t *num_steps, float *t_starts, float *t_ends, int32_t *ridx,
                                       int32_t *gidx, int32_t *bidx, const int64_t *ray_list, int64_t n_list, const uint32_t *grid_bits,
                                       void *stream) {
    const DevCounts dn = take_counts();
    if (n_rays == 0 || (ray_list && n_list == 0)) return 0;
    NSB_REQUIRE(rays_o && rays_d && t_min && t_max && roi && grid_binary, "nsb_ray_marching: NULL input");
    NSB_REQUIRE(rx > 0 && ry > 0 && rz > 0, "nsb_ray_marching: bad grid resolution");
    if (packed_info == nullptr) NSB_REQUIRE(num_steps && !ray_list, "nsb_ray_marching: first round needs num_steps (and marches every ray)");
    else NSB_REQUIRE(t_starts && ridx, "nsb_ray_marching: second round needs t_starts and ridx (t_ends / gidx / bidx are optional)");
    MarchArgs a{n_rays, rays_o, rays_d, t_min, t_max, roi, batch_inds, rx, ry, rz, grid_binary, step_size, max_step_size,
                dt_gamma, max_steps, packed_info, num_steps, t_starts, t_ends, ridx, gidx, bidx, ray_list, n_list, grid_bits, dn.a, nullptr};
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)rx * ry * rz;
    const size_t smem = (size_t)((cells + 31) / 32) * 4;
    const bool use_smem = (batch_inds == nullptr) && smem <= 96 * 1024;
    const unsigned grid = wave_grid(ray_list ? n_list : n_rays, 256, 2);
    if (use_smem) {
        opt_in_smem(k_ray_marching<true>, 96 * 1024);
        k_ray_marching<true><<<grid, 256, smem, s>>>(a);
    } else {
        k_ray_marching<false><<<grid, 256, 0, s>>>(a);
    }
    return check_launch("nsb_ray_marching");
}

extern "C" int nsb_ray_marching_record(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min, const float *t_max,
                                       const float *roi, int32_t rx, int32_t ry, int32_t rz, const uint8_t *grid_binary, float step_size,
                                       float max_step_size, float dt_gamma, uint32_t max_steps, int32_t *num_steps, float *rec_t,
                                       const uint32_t *grid_bits, void *stream) {
    const DevCounts dn = take_counts();
    if (n_rays == 0) return 0;
    NSB_REQUIRE(rays_o && rays_d && t_min && t_max && roi && grid_binary && num_steps && rec_t, "nsb_ray_marching_record: NULL argument");
    NSB_REQUIRE(rx > 0 && ry > 0 && rz > 0 && max_steps > 0, "nsb_ray_marching_record: bad grid resolution / max_steps");
    MarchArgs a{n_rays, rays_o, rays_d, t_min, t_max, roi, nullptr, rx, ry, rz, grid_binary, step_size, max_step_size, dt_gamma, max_steps,
                nullptr, num_steps, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, grid_bits, dn.a, rec_t};
    const size_t smem = (size_t)(((int64_t)rx * ry * rz + 31) / 32) * 4;
    const unsigned grid = wave_grid(n_rays, 256, 2);
    if (smem <= 96 * 1024) {
        opt_in_smem(k_ray_marching<true, true>, 96 * 1024);
        k_ray_marching<true, true><<<grid, 256, smem, (cudaStream_t)stream>>>(a);
    } else {
        k_ray_marching<false, true><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    }
    return check_launch("nsb_ray_marching_record");
}

extern "C" int nsb_march_compact(const float *rec_t, uint32_t max_steps, const int32_t *packed_info, const int64_t *ray_list, int64_t n_list,
                                 float *t_starts, int32_t *ridx, void *stream) {
    const DevCounts dn = take_counts();
    if (n_list == 0) return 0;
    NSB_REQUIRE(rec_t && packed_info && t_starts && ridx && max_steps > 0, "nsb_march_compact: NULL argument");
    k_march_compact<<<wave_grid(n_list * 32, 256, 8), 256, 0, (cudaStream_t)stream>>>(rec_t, max_steps, packed_info, ray_list, n_list, dn.a, t_starts, ridx);
    return check_launch("nsb_march_compact");
}
