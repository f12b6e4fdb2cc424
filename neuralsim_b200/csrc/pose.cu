// Camera rays from refined poses, and the pose gradient, inside the step.
//
// StreetSurf refines every camera node's per-frame pose (app/models/scene/learnable_params.py:85-113): the rotation is the quaternion
// q = q0 + dq, normalised on every use (nr3d_lib/models/attributes/transform.py:107-130: quat_apply(normalize_quat(q), x)), the
// translation is t = t0 + dt (attr.py:326-336).  A camera node under the scene root takes that transform as its world transform
// (app/resources/nodes.py:73-74), and a pixel's ray is (app/resources/observers/cameras.py:299-310)
//   rays_d = normalize(quat_apply(normalize_quat(q), v))      v: the camera-space direction intrs.lift(...) -- normalised AFTER the rotation
//   rays_o = t                                                 the camera centre: no camera-space origin is rotated
// with normalize_quat(q) = standardize_quat(q / max(|q|, 1e-12)) (nr3d_lib/maths/transforms.py:57-72), quat_apply(u, v) the vector part of
// u (0, v) u* (transforms.py:170-193, quat_raw_multiply :150-168, quat_invert :41-55) and normalize(x) = x / max(|x|, 1e-12).
//   k_pose_normalize    per pose: u = s q / max(|q|, eps) (s = -1 where the real part would be negative) and the signed norm s |q|
//   k_pose_rays         per ray: the pose index pidx[i] -> rays_o, rays_d, in the reference's operation order (explicit roundings, no FMA
//                       contraction), so that the rays are the bits of the reference's torch ops
//   k_pose_grad_partial per (chunk of rays, pose): the ray's quaternion and translation cotangents, summed over the chunk's rays of that pose
//                       in a fixed order (no atomics, no sort: rays need not be ordered by pose)
//   k_pose_grad_finish  per pose: the chunks' sums in chunk order, the adjoint of the normalisation, ADDED to d_dq / d_dt
// Every ray kernel stops at the device count (nsb_bind_device_counts).
#include "nsb_common.cuh"

namespace nsb {

constexpr float kPoseEps = 1e-12f;          // F.normalize's eps
constexpr int kPoseChunk = 4096;            // rays per chunk of k_pose_grad_partial (their pose indices in shared memory)
constexpr int kPosesPerBlock = 64;          // poses per block of k_pose_grad_partial (8 warps, 8 poses each)
constexpr int kPoseRow = 8;                 // floats per (chunk, pose) partial: d_u (4), d_t (3), 0

// the reference's quat_raw_multiply, term by term, each product and sum rounded (separate torch ops)
__device__ __forceinline__ void qmul_rn(const float a[4], const float b[4], float o[4]) {
    o[0] = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2])), __fmul_rn(a[3], b[3]));
    o[1] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0])), __fmul_rn(a[2], b[3])), __fmul_rn(a[3], b[2]));
    o[2] = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(a[0], b[2]), __fmul_rn(a[1], b[3])), __fmul_rn(a[2], b[0])), __fmul_rn(a[3], b[1]));
    o[3] = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(a[0], b[3]), __fmul_rn(a[1], b[2])), __fmul_rn(a[2], b[1])), __fmul_rn(a[3], b[0]));
}

// the plain quaternion product (the adjoint's arithmetic, where no torch op sequence is to be matched)
__device__ __forceinline__ void qmul(const float a[4], const float b[4], float o[4]) {
    o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
    o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

// torch's 2-norm over a last dimension of 4 / 3 floats, in the order its CUDA reduction adds the squares (linalg.vector_norm: two threads
// per row, thread 0 holding elements 0 and 2, thread 1 elements 1 (and 3), then one shuffle; the same bits on an H100 for every row of
// 480 000 random rows, at every row count tried)
__device__ __forceinline__ float norm4_rn(const float q[4]) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[2], q[2])), __fadd_rn(__fmul_rn(q[1], q[1]), __fmul_rn(q[3], q[3]))));
}
__device__ __forceinline__ float norm3_rn(const float r[3]) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], r[0]), __fmul_rn(r[2], r[2])), __fmul_rn(r[1], r[1])));
}

__device__ __forceinline__ float clamp_eps(float n) { return n < kPoseEps ? kPoseEps : n; }       // clamp_min: NaN stays NaN

// r = the vector part of u (0, v) u*, as quat_apply computes it
__device__ __forceinline__ void quat_apply_rn(const float u[4], const float v[3], float r[3]) {
    const float p[4] = {0.f, v[0], v[1], v[2]};
    const float ui[4] = {u[0], -u[1], -u[2], -u[3]};
    float a[4], o[4];
    qmul_rn(u, p, a);
    qmul_rn(a, ui, o);
    r[0] = o[1]; r[1] = o[2]; r[2] = o[3];
}

__global__ void __launch_bounds__(256)
k_pose_normalize(const float *__restrict__ q0, const float *__restrict__ dq, int64_t n_poses, float *__restrict__ unit, float *__restrict__ nrm) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_poses; p += (int64_t)gridDim.x * blockDim.x) {
        float q[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) q[k] = __fadd_rn(q0[p * 4 + k], dq[p * 4 + k]);
        const float n = norm4_rn(q), c = clamp_eps(n);
        float u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = __fdiv_rn(q[k], c);
        const bool flip = u[0] < 0.f;                     // standardize_quat
#pragma unroll
        for (int k = 0; k < 4; ++k) unit[p * 4 + k] = flip ? -u[k] : u[k];
        nrm[p] = flip ? -n : n;
    }
}

__global__ void __launch_bounds__(256)
k_pose_rays(const float *__restrict__ unit, const float *__restrict__ t0, const float *__restrict__ dt, const int64_t *__restrict__ pidx,
            const float *__restrict__ dirs, int64_t n, float *__restrict__ rays_o, float *__restrict__ rays_d, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = pidx[i];
        const float4 u4 = *reinterpret_cast<const float4 *>(unit + p * 4);
        const float u[4] = {u4.x, u4.y, u4.z, u4.w}, v[3] = {dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2]};
        float r[3];
        quat_apply_rn(u, v, r);
        const float c = clamp_eps(norm3_rn(r));
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            rays_d[i * 3 + k] = __fdiv_rn(r[k], c);
            rays_o[i * 3 + k] = __fadd_rn(t0[p * 3 + k], dt[p * 3 + k]);
        }
    }
}

// One ray's cotangents: d_t = g_o, and d_u, the gradient to the unit quaternion u of rays_d = normalize(r), r = vec(u p u*), p = (0, v):
//   d_r = g_d / c - [|r| >= eps] r (g_d . r) / (c^2 |r|)          (c = max(|r|, eps))
//   d_u = -2 (0, d_r) u p                                           (the sandwich's adjoint: <g, du p u*> + <g, u p du*> = <-2 g u p, du>)
__device__ __forceinline__ void pose_ray_cotangent(const float u[4], const float v[3], const float gd[3], float du[4]) {
    float r[3];
    quat_apply_rn(u, v, r);
    const float nr = norm3_rn(r), c = clamp_eps(nr);
    const float dot = gd[0] * r[0] + gd[1] * r[1] + gd[2] * r[2];
    const float k = nr >= kPoseEps ? dot / (c * c * nr) : 0.f;
    const float g[4] = {0.f, gd[0] / c - r[0] * k, gd[1] / c - r[1] * k, gd[2] / c - r[2] * k};
    const float p[4] = {0.f, v[0], v[1], v[2]};
    float h[4];
    qmul(g, u, h);
    qmul(h, p, du);
#pragma unroll
    for (int q = 0; q < 4; ++q) du[q] *= -2.f;
}

// Block (x, y): poses [64 x, 64 x + 64) over the rays of chunk y.  Warp w takes poses 64 x + w, + 8, ...; its lanes walk the chunk's rays
// lane, lane + 32, ... and add the cotangents of the rays of that pose; a fixed butterfly sums the lanes; lane 0 writes the pose's row of
// the chunk, zeros included.  The order of every sum is fixed by the ray positions alone: the same bits on every run.
__global__ void __launch_bounds__(256)
k_pose_grad_partial(const float *__restrict__ unit, int64_t n_poses, const int64_t *__restrict__ pidx, const float *__restrict__ dirs,
                    const float *__restrict__ g_o, const float *__restrict__ g_d, int64_t n, float *__restrict__ partial,
                    const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    __shared__ int32_t sp[kPoseChunk];
    const int64_t base = (int64_t)blockIdx.y * kPoseChunk;
    const int m = n - base >= kPoseChunk ? kPoseChunk : (n > base ? (int)(n - base) : 0);
    for (int j = threadIdx.x; j < kPoseChunk; j += blockDim.x) sp[j] = j < m ? (int32_t)pidx[base + j] : -1;
    __syncthreads();
    const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
    const int64_t p_end = min(n_poses, (int64_t)(blockIdx.x + 1) * kPosesPerBlock);
    for (int64_t p = (int64_t)blockIdx.x * kPosesPerBlock + warp; p < p_end; p += 8) {
        float acc[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) acc[k] = 0.f;
        const float4 u4 = *reinterpret_cast<const float4 *>(unit + p * 4);
        const float u[4] = {u4.x, u4.y, u4.z, u4.w};
        for (int j = lane; j < m; j += 32) {
            if (sp[j] != (int32_t)p) continue;
            const int64_t i = base + j;
            const float v[3] = {dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2]}, gd[3] = {g_d[i * 3], g_d[i * 3 + 1], g_d[i * 3 + 2]};
            float du[4];
            pose_ray_cotangent(u, v, gd, du);
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[k] += du[k];
#pragma unroll
            for (int k = 0; k < 3; ++k) acc[4 + k] += g_o[i * 3 + k];
        }
#pragma unroll
        for (int k = 0; k < 7; ++k)
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) acc[k] += __shfl_xor_sync(~0u, acc[k], off);
        if (lane < kPoseRow) {
            float val = 0.f;
#pragma unroll
            for (int k = 0; k < 7; ++k) val = lane == k ? acc[k] : val;
            partial[((int64_t)blockIdx.y * n_poses + p) * kPoseRow + lane] = val;
        }
    }
}

// Per pose: s = the chunks' rows summed in chunk order; the adjoint of u = s' q / max(|q|, eps) (s' the standardisation's sign, carried by
// the signed norm nrm = s' |q|):  d_q = (s_u - u (u . s_u)) / nrm  (|q| >= eps),  s_u / copysign(eps, nrm)  (clamped: the norm gets none);
// d_dq[p] += d_q, d_dt[p] += s_t (d_dq or d_dt NULL: not written).
__global__ void __launch_bounds__(256)
k_pose_grad_finish(const float *__restrict__ unit, const float *__restrict__ nrm, int64_t n_poses, const float *__restrict__ partial, int64_t n_chunks,
                   float *__restrict__ d_dq, float *__restrict__ d_dt) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_poses; p += (int64_t)gridDim.x * blockDim.x) {
        float s[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) s[k] = 0.f;
        for (int64_t c = 0; c < n_chunks; ++c) {
            const float *row = partial + (c * n_poses + p) * kPoseRow;
            const float4 a = *reinterpret_cast<const float4 *>(row), b = *reinterpret_cast<const float4 *>(row + 4);
            s[0] += a.x; s[1] += a.y; s[2] += a.z; s[3] += a.w; s[4] += b.x; s[5] += b.y; s[6] += b.z;
        }
        if (d_dq) {
            const float sn = nrm[p];
            const float u[4] = {unit[p * 4], unit[p * 4 + 1], unit[p * 4 + 2], unit[p * 4 + 3]};
            const bool clamped = !(fabsf(sn) >= kPoseEps);
            const float ud = u[0] * s[0] + u[1] * s[1] + u[2] * s[2] + u[3] * s[3];
#pragma unroll
            for (int k = 0; k < 4; ++k) d_dq[p * 4 + k] += clamped ? s[k] / copysignf(kPoseEps, sn) : (s[k] - u[k] * ud) / sn;
        }
        if (d_dt) {
#pragma unroll
            for (int k = 0; k < 3; ++k) d_dt[p * 3 + k] += s[4 + k];
        }
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int64_t nsb_pose_grad_scratch_floats(int64_t n, int64_t n_poses) {
    return ((n + kPoseChunk - 1) / kPoseChunk) * n_poses * kPoseRow;
}

extern "C" int nsb_pose_rays(const float *q0, const float *dq, const float *t0, const float *dt, int64_t n_poses, const int64_t *pidx, const float *dirs,
                             int64_t n, float *unit, float *nrm, float *rays_o, float *rays_d, void *stream) {
    const DevCounts dn = take_counts();
    NSB_REQUIRE(n >= 0 && n_poses >= 0, "nsb_pose_rays: negative size");
    NSB_REQUIRE(n_poses <= INT32_MAX, "nsb_pose_rays: at most 2^31 - 1 poses");
    NSB_REQUIRE(q0 && dq && t0 && dt && unit && nrm, "nsb_pose_rays: NULL pose argument");
    NSB_REQUIRE(n == 0 || (pidx && dirs && rays_o && rays_d), "nsb_pose_rays: NULL ray argument");
    NSB_REQUIRE(n == 0 || n_poses > 0, "nsb_pose_rays: rays need at least one pose");
    NSB_REQUIRE(((uintptr_t)unit & 15) == 0, "nsb_pose_rays: unit must be 16-byte aligned");
    if (n_poses == 0) return 0;
    k_pose_normalize<<<wave_grid(n_poses, 256, 8), 256, 0, STREAM>>>(q0, dq, n_poses, unit, nrm);
    if (check_launch("nsb_pose_rays (normalize)")) return 1;
    if (n == 0) return 0;
    k_pose_rays<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(unit, t0, dt, pidx, dirs, n, rays_o, rays_d, dn.a);
    return check_launch("nsb_pose_rays");
}

extern "C" int nsb_pose_rays_backward(const float *unit, const float *nrm, int64_t n_poses, const int64_t *pidx, const float *dirs, int64_t n,
                                      const float *d_rays_o, const float *d_rays_d, float *scratch, float *d_dq, float *d_dt, void *stream) {
    const DevCounts dn = take_counts();
    NSB_REQUIRE(n >= 0 && n_poses >= 0, "nsb_pose_rays_backward: negative size");
    NSB_REQUIRE(n_poses <= INT32_MAX, "nsb_pose_rays_backward: at most 2^31 - 1 poses");
    NSB_REQUIRE(unit && nrm, "nsb_pose_rays_backward: NULL pose argument");
    NSB_REQUIRE(n == 0 || (pidx && dirs && d_rays_o && d_rays_d && scratch), "nsb_pose_rays_backward: NULL ray argument");
    NSB_REQUIRE(n == 0 || n_poses > 0, "nsb_pose_rays_backward: rays need at least one pose");
    NSB_REQUIRE(((uintptr_t)unit & 15) == 0 && ((uintptr_t)scratch & 15) == 0, "nsb_pose_rays_backward: unit and scratch must be 16-byte aligned");
    const int64_t n_chunks = (n + kPoseChunk - 1) / kPoseChunk;
    NSB_REQUIRE(n_chunks <= 65535, "nsb_pose_rays_backward: at most 65535 x %d rays", kPoseChunk);
    if (n_poses == 0 || n == 0 || (!d_dq && !d_dt)) return 0;
    const dim3 grid((unsigned)((n_poses + kPosesPerBlock - 1) / kPosesPerBlock), (unsigned)n_chunks);
    k_pose_grad_partial<<<grid, 256, 0, STREAM>>>(unit, n_poses, pidx, dirs, d_rays_o, d_rays_d, n, scratch, dn.a);
    if (check_launch("nsb_pose_rays_backward (partial)")) return 1;
    k_pose_grad_finish<<<wave_grid(n_poses, 256, 8), 256, 0, STREAM>>>(unit, nrm, n_poses, scratch, n_chunks, d_dq, d_dt);
    return check_launch("nsb_pose_rays_backward");
}
