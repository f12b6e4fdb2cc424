/* CPU restatement of the reference occupancy-grid ray marching kernels.  TEST INFRASTRUCTURE.
 *
 * Follows nr3d_lib/csrc/occ_grid:
 *   src/ray_marching.cu:17-134        (ray_marching_kernel, AABB contraction only)
 *   src/batched_marching.cu:18-152    (batched_ray_marching_kernel)
 *   include/occ_grid/helpers_march.h:11-76, helpers_contraction.h:10-21
 *
 * Floating-point operation order.  Sample counts and voxel indices are integer outputs that must be
 * bit-exact, so the exact sequence of fp32 roundings matters.  The sequence below (which products are
 * fused into an FMA, which divisions are IEEE) was read off the SASS that nvcc 12.9 generates for the
 * reference source at -O3 for sm_100a (cuobjdump of ray_marching.cu, see DESIGN.md "March: rounding
 * sequence"); the reference's sm_90a build produces the same outputs bit for bit (digests stored under tests/golden/,
 * tests/test_ref_parity_gpu.py):
 *   xyz          = fma(t_mid, dir, origin)
 *   unit         = (xyz - roi_min) / (roi_max - roi_min)               IEEE division
 *   ixyz         = trunc(unit * float(res))                            one multiply
 *   next-voxel   : a = fma(res, unit, 0.5); b = fma(sign(dir), 0.5, a); f = floor(b);
 *                  d = fma(res, -unit, f); t = ((d * inv_dir) / res) * (roi_max - roi_min)
 *   re-centre    : t0 = fma(dt, -0.5, t_mid); t1 = fma(dt, 0.5, t_mid)
 * Build with -ffp-contract=off so the compiler adds no fusion of its own.
 */
#include <math.h>
#include <stdint.h>
#include <stddef.h>

static inline float clampf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }
static inline float calc_dt(float t, float dt_gamma, float dt_min, float dt_max) {
    return clampf(t * dt_gamma, dt_min, dt_max);
}
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

typedef struct { float x, y, z; } f3;

static inline int grid_idx_at(f3 u, const int res[3]) {
    int ix = clampi((int)(u.x * (float)res[0]), 0, res[0] - 1);
    int iy = clampi((int)(u.y * (float)res[1]), 0, res[1] - 1);
    int iz = clampi((int)(u.z * (float)res[2]), 0, res[2] - 1);
    return ix * res[1] * res[2] + iy * res[2] + iz;
}

static inline float next_axis(float unit, float dir, float inv_dir, int res, float extent) {
    float r = (float)res;
    float a = fmaf(r, unit, 0.5f);
    float b = fmaf(copysignf(1.0f, dir), 0.5f, a);
    float f = floorf(b);
    float d = fmaf(r, -unit, f);
    return ((d * inv_dir) / r) * extent;
}

/* One ray.  grid: res[0]*res[1]*res[2] bytes (bool), z fastest.  Writes when t_starts != NULL. */
static uint32_t march_one(const float *o, const float *d, float near, float far, const float *roi,
                          const int res[3], const uint8_t *grid, float step_size, float max_step_size,
                          float dt_gamma, uint32_t max_steps, int32_t ray_id,
                          float *t_starts, float *t_ends, int32_t *ridx, int32_t *gidx) {
    const float dt_min = step_size, dt_max = max_step_size;
    const f3 inv = {1.0f / d[0], 1.0f / d[1], 1.0f / d[2]};
    const float ext[3] = {roi[3] - roi[0], roi[4] - roi[1], roi[5] - roi[2]};
    uint32_t j = 0;
    float t0 = near;
    float dt = calc_dt(t0, dt_gamma, dt_min, dt_max);
    float t1 = t0 + dt;
    float t_mid = (t0 + t1) * 0.5f;
    while (t_mid < far && j < max_steps) {
        f3 p = {fmaf(t_mid, d[0], o[0]), fmaf(t_mid, d[1], o[1]), fmaf(t_mid, d[2], o[2])};
        int occupied = 0, gi = -1;
        f3 u = {0, 0, 0};
        int inside = !(p.x < roi[0] || p.x > roi[3] || p.y < roi[1] || p.y > roi[4] || p.z < roi[2] || p.z > roi[5]);
        if (inside) {
            u.x = (p.x - roi[0]) / ext[0];
            u.y = (p.y - roi[1]) / ext[1];
            u.z = (p.z - roi[2]) / ext[2];
            gi = grid_idx_at(u, res);
            occupied = grid[gi] != 0;
        }
        if (occupied) {
            if (t_starts) {
                t_starts[j] = t0; t_ends[j] = t1; ridx[j] = ray_id;
                if (gidx) gidx[j] = gi;
            }
            ++j;
            t0 = t1;
            t1 = t0 + calc_dt(t0, dt_gamma, dt_min, dt_max);
            t_mid = (t0 + t1) * 0.5f;
        } else {
            /* distance_to_next_voxel + advance_to_next_voxel (helpers_march.h:44-76); the unit coordinates
             * are recomputed from xyz even when the point lies outside the roi. */
            f3 uu = {(p.x - roi[0]) / ext[0], (p.y - roi[1]) / ext[1], (p.z - roi[2]) / ext[2]};
            float tx = next_axis(uu.x, d[0], inv.x, res[0], ext[0]);
            float ty = next_axis(uu.y, d[1], inv.y, res[1], ext[1]);
            float tz = next_axis(uu.z, d[2], inv.z, res[2], ext[2]);
            float t = fmaxf(fminf(fminf(tx, ty), tz), 0.0f);
            float t_target = t_mid + t;
            float _t = t_mid;
            do { _t += dt_min; } while (_t < t_target);
            t_mid = _t;
            dt = calc_dt(t_mid, dt_gamma, dt_min, dt_max);
            t0 = fmaf(dt, -0.5f, t_mid);
            t1 = fmaf(dt, 0.5f, t_mid);
        }
    }
    return j;
}

/* Pass 1 (packed_info == NULL): num_steps[i].  Pass 2: fill outputs at packed_info[i] = (base, count).
 * batch_inds == NULL -> single grid; else grid is [B, rx, ry, rz], roi is [B, 6] and rays with
 * batch_inds < 0 produce no samples (batched_marching.cu:55). */
int nsb_oracle_ray_marching(int n_rays, const float *rays_o, const float *rays_d, const float *t_min,
                            const float *t_max, const float *roi, const int32_t *batch_inds, int rx, int ry,
                            int rz, const uint8_t *grid, float step_size, float max_step_size, float dt_gamma,
                            uint32_t max_steps, const int32_t *packed_info, int32_t *num_steps,
                            float *t_starts, float *t_ends, int32_t *ridx, int32_t *gidx, int32_t *bidx) {
    const int res[3] = {rx, ry, rz};
    const size_t gsz = (size_t)rx * ry * rz;
    for (int i = 0; i < n_rays; ++i) {
        int b = 0;
        if (batch_inds) {
            b = batch_inds[i];
            if (b < 0) { if (!packed_info) num_steps[i] = 0; continue; }
        }
        const float *r = roi + 6 * b;
        const uint8_t *g = grid + gsz * b;
        if (!packed_info) {
            num_steps[i] = (int32_t)march_one(rays_o + 3 * i, rays_d + 3 * i, t_min[i], t_max[i], r, res, g, step_size,
                                              max_step_size, dt_gamma, max_steps, i, NULL, NULL, NULL, NULL);
        } else {
            int32_t base = packed_info[2 * i], cnt = packed_info[2 * i + 1];
            uint32_t n = march_one(rays_o + 3 * i, rays_d + 3 * i, t_min[i], t_max[i], r, res, g, step_size, max_step_size,
                                   dt_gamma, (uint32_t)cnt, i, t_starts + base, t_ends + base, ridx + base,
                                   gidx ? gidx + base : NULL);
            /* the batched voxel index is flat over [B, X, Y, Z]: grid_idx + batch_ind * X*Y*Z (batched_marching.cu:62,115) */
            if (gidx) for (uint32_t k = 0; k < n; ++k) gidx[base + k] += (int32_t)(gsz * b);
            if (bidx) for (uint32_t k = 0; k < n; ++k) bidx[base + k] = b;
        }
    }
    return 0;
}
