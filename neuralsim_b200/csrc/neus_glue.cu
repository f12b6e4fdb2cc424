// Glue of the per-ray NeuS query for sm_90a: the index bookkeeping between the big kernels (march -> up-sample -> boundary
// SDF -> alpha -> colour -> composite) that the reference does with ~200 ATen launches and ~20 host syncs per call
// (graphics/neus/neus_ray_query.py:732-1104, pack_ops.py, occgrid_raymarch.py:60-112) -- here one launch per step:
//
//   k_scan_counts        exclusive scan of per-ray counts + compaction of the non-empty rays, one CTA, totals on the device
//                        (replaces cumsum / nonzero / stack / index chains; the host reads the two totals once)
//   k_merge_vals         merge_two_packs_sorted_aligned + the scatter of both payloads (depth, sdf) into the merged buffers
//                        (pack_ops.py:529-560 + neus_ray_query.py:893-905)
//   k_assemble_boundary  depths_1 = sort(cat(fine stages)); merge_two_batch_a_includes_b with the coarse samples; ridx;
//                        mid-points  (neus_ray_query.py:907-976)
//   k_compact_samples    packed_volume_render_compression's gather of the kept samples (pack_ops.py:286-291 + :1010-1030)
//
// All outputs are the reference's values (same fp32 roundings).  Equal depths keep a fixed order: in the merge a b goes before an equal
// a, in the boundary assembly the order is (coarse, run 0, run 1, ...).  The step's ties carry equal payloads, so only the sign bit
// of a +0.0 / -0.0 tie shows it (tests/test_glue_edges_gpu.py pins it).
#include "neus_device.cuh"

namespace nsb {

__device__ __forceinline__ int64_t gwarp_() { return ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int64_t nwarps_() { return ((int64_t)gridDim.x * blockDim.x) >> 5; }

// ------------------------------------------------------------------------------------------------ scan + compaction
// counts[N] (int32, >= 0)  ->  first[N] (exclusive prefix sum), and for the non-zero entries, in order:
// nz_index[j] = i, nz_pack[j] = (first_i, counts_i) (int64), optionally gathered values nz_src[j] = src[i];
// info2[N,2] = (first_i, counts_i) int32 (the reference's `packed_info`); totals = (sum, number of non-zeros).
constexpr int kScanT = 1024, kScanI = 8, kScanMaxBlocks = 128;
struct ScanWs {                                                      // zero-filled by the caller before every launch
    long long sum[kScanMaxBlocks];
    int nz[kScanMaxBlocks];
    int flag[kScanMaxBlocks];
    int ticket;                                                      // segments are handed out in the order the blocks START: a block only waits for
};                                                                   // blocks that are already running (no co-residency assumption, no deadlock)

__device__ __forceinline__ void block_scan_pair(int64_t &ps, int32_t &pz, int lane, int warp, int64_t *s_sum, int32_t *s_nz) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t a = __shfl_up_sync(0xffffffffu, ps, o);
        const int32_t b = __shfl_up_sync(0xffffffffu, pz, o);
        if (lane >= o) { ps += a; pz += b; }
    }
    __syncthreads();                                      // s_sum / s_nz of the previous sweep have been read
    if (lane == 31) { s_sum[warp] = ps; s_nz[warp] = pz; }
    __syncthreads();
    if (warp == 0) {
        int64_t a = s_sum[lane];
        int32_t b = s_nz[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t a2 = __shfl_up_sync(0xffffffffu, a, o);
            const int32_t b2 = __shfl_up_sync(0xffffffffu, b, o);
            if (lane >= o) { a += a2; b += b2; }
        }
        s_sum[lane] = a;
        s_nz[lane] = b;
    }
    __syncthreads();
}

// Block b owns the contiguous segment [b seg, (b+1) seg): (1) segment totals -> published, (2) wait for the predecessors' totals,
// (3) scan the segment with that carry.  One launch, a few microseconds for 10^5..10^6 counts.
__global__ void __launch_bounds__(kScanT)
k_scan_counts(const int32_t *__restrict__ counts, int64_t n, int64_t seg, ScanWs *__restrict__ ws, int32_t *__restrict__ first,
              int32_t *__restrict__ info2, int64_t *__restrict__ nz_index, int64_t *__restrict__ nz_pack, const int64_t *__restrict__ src,
              int64_t *__restrict__ nz_src, int64_t *totals, const int64_t *__restrict__ extra_src, int64_t ticket) {
    __shared__ int64_t s_sum[32];
    __shared__ int32_t s_nz[32];
    __shared__ int64_t s_carry_sum;
    __shared__ int32_t s_carry_nz;
    __shared__ int s_b;
    if (threadIdx.x == 0) s_b = atomicAdd(&ws->ticket, 1);
    __syncthreads();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = s_b;
    const int64_t lo = (int64_t)b * seg, hi = min(n, lo + seg);
    // ---- (1) totals of my segment
    int64_t ps = 0;
    int32_t pz = 0;
    for (int64_t i = lo + tid; i < hi; i += kScanT) { const int32_t c = counts[i]; ps += c; pz += c > 0 ? 1 : 0; }
    block_scan_pair(ps, pz, lane, warp, s_sum, s_nz);
    const int64_t my_sum = s_sum[31];
    const int32_t my_nz = s_nz[31];
    if (tid == 0) {
        ws->sum[b] = my_sum;
        ws->nz[b] = my_nz;
        __threadfence();
        atomicExch(&ws->flag[b], 1);
    }
    // ---- (2) carry = totals of the blocks before me
    ps = 0;
    pz = 0;
    if (tid < b) {
        while (atomicAdd(&ws->flag[tid], 0) == 0) {}
        __threadfence();
        ps = *((volatile long long *)&ws->sum[tid]);
        pz = *((volatile int *)&ws->nz[tid]);
    }
    block_scan_pair(ps, pz, lane, warp, s_sum, s_nz);
    if (tid == 0) { s_carry_sum = s_sum[31]; s_carry_nz = s_nz[31]; }
    __syncthreads();
    int64_t carry_sum = s_carry_sum;
    int32_t carry_nz = s_carry_nz;
    if (b == gridDim.x - 1 && tid == 0) {
        // `totals` may be mapped pinned host memory that the host polls (no driver call on its side): values first, then the ticket
        volatile int64_t *tv = totals;
        tv[0] = carry_sum + my_sum;
        tv[1] = carry_nz + my_nz;
        if (extra_src) tv[2] = extra_src[0];
        if (ticket) {
            __threadfence_system();
            tv[3] = ticket;
        }
    }
    // ---- (3) scan my segment, kScanI consecutive items per thread and sweep
    for (int64_t base = lo; base < hi; base += (int64_t)kScanT * kScanI) {
        const int64_t i0 = base + (int64_t)tid * kScanI;
        int32_t c[kScanI];
        ps = 0;
        pz = 0;
#pragma unroll
        for (int k = 0; k < kScanI; ++k) {
            c[k] = (i0 + k < hi) ? counts[i0 + k] : 0;
            ps += c[k];
            pz += c[k] > 0 ? 1 : 0;
        }
        const int64_t tsum = ps;
        const int32_t tnz = pz;
        block_scan_pair(ps, pz, lane, warp, s_sum, s_nz);
        int64_t excl = carry_sum + (warp ? s_sum[warp - 1] : 0) + ps - tsum;
        int32_t rank = carry_nz + (warp ? s_nz[warp - 1] : 0) + pz - tnz;
#pragma unroll
        for (int k = 0; k < kScanI; ++k) {
            const int64_t i = i0 + k;
            if (i < hi) {
                if (first) first[i] = (int32_t)excl;
                if (info2) { info2[2 * i] = (int32_t)excl; info2[2 * i + 1] = c[k]; }
                if (c[k] > 0) {
                    if (nz_index) nz_index[rank] = i;
                    if (nz_pack) { nz_pack[2 * rank] = excl; nz_pack[2 * rank + 1] = c[k]; }
                    if (nz_src) nz_src[rank] = src[i];
                    ++rank;
                }
            }
            excl += c[k];
        }
        carry_sum += s_sum[31];
        carry_nz += s_nz[31];
    }
}

// ------------------------------------------------------------------------------------------------ merge with payloads
// pack p of a: (dep_a, sdf_a)[pi_a[p]] sorted by depth; pack p of b: row p of (dep_b, sdf_b)[P, nb], sorted; merged by warp_merge.
// pi_m[p] = (pi_a[p].first + p * nb, n_a + nb).  One warp per pack; b lives in shared memory.
constexpr int kMergeWarps = 8;
__global__ void __launch_bounds__(kMergeWarps * 32)
k_merge_vals(const float *__restrict__ dep_a, const float *__restrict__ sdf_a, const int64_t *__restrict__ pi_a, const float *__restrict__ dep_b,
             const float *__restrict__ sdf_b, int64_t n_packs, int nb, float *__restrict__ dep_m, float *__restrict__ sdf_m,
             int64_t *__restrict__ pi_m, const int64_t *__restrict__ n_dev) {
    extern __shared__ float s_b[];                        // [warps][nb]
    n_packs = eff_n(n_packs, n_dev);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float *bb = s_b + w * nb;
    for (int64_t p = gwarp_(); p < n_packs; p += nwarps_()) {
        const int64_t a0 = pi_a[2 * p], na = pi_a[2 * p + 1];
        const int64_t m0 = a0 + p * nb;
        __syncwarp();
        for (int j = lane; j < nb; j += 32) bb[j] = dep_b[p * nb + j];
        __syncwarp();
        if (lane == 0) { pi_m[2 * p] = m0; pi_m[2 * p + 1] = na + nb; }
        warp_merge(dep_a + a0, sdf_a + a0, (int)na, bb, sdf_b + p * nb, nb, dep_m + m0, sdf_m ? sdf_m + m0 : nullptr, lane);
    }
}

// ------------------------------------------------------------------------------------------------ boundary samples
// Ray r of the R tested rays carries nc coarse depths (sorted); if r == ridx_hit[j] it also carries the nf fine depths of
// row j (a concatenation of sorted runs).  Output pack r = the sorted union; first_r = nc r + nf #{hit rays < r}.
//   d1[first + k] = k-th smallest;  mid[first + k] = d1_k + (d1_{k+1} - d1_k) / 2 (last: + 0);  ridx_all = r.
constexpr int kAsmWarps = 8, kAsmMaxRuns = 8, kAsmChunk = 8;
struct AsmRuns { int n, len[kAsmMaxRuns]; };              // the fine row is a concatenation of `n` sorted runs (one per up-sampling stage)

// mid[k] of a sorted pack: d_k + (d_{k+1} - d_k) / 2, the last sample's own depth + 0 (k_assemble_boundary, k_compact_samples)
__device__ __forceinline__ float interval_mid(float v, float next, bool last) {
    const float diff = last ? 0.f : __fsub_rn(next, v);
    return __fadd_rn(v, __fmul_rn(diff, 0.5f));
}

// kAsmChunk consecutive rays per warp trip: ONE search of the first ray in ridx_hit (18 dependent L2 loads on a frame -- half of the
// kernel's time when every ray searched for itself), the next kAsmChunk entries of the list in registers, a running rank for the rest.
__global__ void __launch_bounds__(kAsmWarps * 32)
k_assemble_boundary(const float *__restrict__ coarse, int64_t n_rays, int nc, const int64_t *__restrict__ ridx_hit, int64_t n_hit,
                    const float *__restrict__ fine, int nf, const AsmRuns runs, float *__restrict__ d1, float *__restrict__ mid,
                    int64_t *__restrict__ ridx_all, int64_t *__restrict__ pack_infos, const int64_t *__restrict__ n_rays_dev,
                    const int64_t *__restrict__ n_hit_dev) {
    extern __shared__ float s_v[];                        // [warps][2][nc + nf]
    static_assert(kAsmChunk >= 1 && kAsmChunk <= 32, "one candidate per lane");
    n_rays = eff_n(n_rays, n_rays_dev);
    n_hit = eff_n(n_hit, n_hit_dev);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, cap = nc + nf;
    float *raw = s_v + (size_t)w * 2 * cap, *srt = raw + cap;
    const int64_t n_chunks = (n_rays + kAsmChunk - 1) / kAsmChunk;
    for (int64_t c = gwarp_(); c < n_chunks; c += nwarps_()) {
        const int64_t r0 = c * kAsmChunk;
        const int64_t lo0 = partition_point(ridx_hit, n_hit, [&](int64_t x) { return x < r0; });     // lower bound of r0 in ridx_hit
        long long cand = -1;                              // lane k: the k-th listed ray at or after r0
        if (lane < kAsmChunk && lo0 + lane < n_hit) cand = ridx_hit[lo0 + lane];
        int used = 0;                                     // listed rays among r0 .. r - 1
        for (int j = 0; j < kAsmChunk; ++j) {
            const int64_t r = r0 + j;
            if (r >= n_rays) break;
            const bool hit = __shfl_sync(0xffffffffu, cand, used) == r;      // used <= j < kAsmChunk
            const int64_t lo = lo0 + used;
            const int n = nc + (hit ? nf : 0);
            const int64_t first = (int64_t)nc * r + (int64_t)nf * lo;
            if (lane == 0) { pack_infos[2 * r] = first; pack_infos[2 * r + 1] = n; }
            if (!hit) {                                   // the coarse row is already sorted: straight copy
                for (int k = lane; k < nc; k += 32) {
                    const float v = coarse[r * nc + k];
                    d1[first + k] = v;
                    if (mid) mid[first + k] = interval_mid(v, k < nc - 1 ? coarse[r * nc + k + 1] : 0.f, k == nc - 1);
                    if (ridx_all) ridx_all[first + k] = r;
                }
                continue;
            }
            ++used;
            __syncwarp();
            for (int k = lane; k < nc; k += 32) raw[k] = coarse[r * nc + k];
            for (int k = lane; k < nf; k += 32) raw[nc + k] = fine[lo * nf + k];
            __syncwarp();
            // stable rank of every element among the 1 + runs.n sorted runs: own index + (<=-count in earlier runs) + (<-count in later runs)
            for (int e = lane; e < n; e += 32) {
                const float v = raw[e];
                int rank = 0, start = 0;
                for (int q = -1; q < runs.n; ++q) {
                    const int len = q < 0 ? nc : runs.len[q];
                    if (e >= start && e < start + len) rank += e - start;
                    else rank += partition_point(raw + start, len, [&](float u) { return start < e ? u <= v : u < v; });
                    start += len;
                }
                srt[rank] = v;
            }
            __syncwarp();
            for (int k = lane; k < n; k += 32) {
                const float v = srt[k];
                d1[first + k] = v;
                if (mid) mid[first + k] = interval_mid(v, k < n - 1 ? srt[k + 1] : 0.f, k == n - 1);
                if (ridx_all) ridx_all[first + k] = r;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ compaction of the kept samples
// selector[S] marks the samples packed_volume_render_compression keeps; first_out[p] = exclusive scan of the kept counts.
// Kept sample s of pack p -> slot first_out[p] + (number of kept samples before s in the pack).  Without ridx_all the ray is the pack;
// without t the depth is the mid-point of the sample's interval in d1 (what k_assemble_boundary writes to `mid`).
__global__ void __launch_bounds__(256)
k_compact_samples(const uint8_t *__restrict__ selector, const int64_t *__restrict__ pi, const int32_t *__restrict__ first_out,
                  const int32_t *__restrict__ kept, int64_t n_packs, const int64_t *__restrict__ ridx_all, const float *__restrict__ t,
                  const float *__restrict__ d1, const float *__restrict__ alpha, int64_t *__restrict__ pidx, int64_t *__restrict__ ridx_c, float *__restrict__ t_c,
                  float *__restrict__ alpha_c, const int64_t *__restrict__ n_dev) {
    const int lane = threadIdx.x & 31;
    n_packs = eff_n(n_packs, n_dev);
    for (int64_t p = gwarp_(); p < n_packs; p += nwarps_()) {
        const int32_t kp = kept[p];
        if (kp == 0) continue;
        const int64_t b = pi[2 * p], n = pi[2 * p + 1];
        int64_t out = first_out[p];
        int32_t done = 0;
        for (int64_t k0 = 0; k0 < n && done < kp; k0 += 32) {
            const int64_t k = k0 + lane;
            const bool sel = k < n && selector[b + k] != 0;
            const uint32_t m = __ballot_sync(0xffffffffu, sel);
            if (sel) {
                const int64_t o = out + __popc(m & ((1u << lane) - 1u));
                pidx[o] = b + k;
                ridx_c[o] = ridx_all ? ridx_all[b + k] : p;
                t_c[o] = t ? t[b + k] : interval_mid(d1[b + k], k < n - 1 ? d1[b + k + 1] : 0.f, k == n - 1);
                alpha_c[o] = alpha[b + k];
            }
            const int c = __popc(m);
            out += c;
            done += c;
        }
    }
}

// dst[idx[j]] = src[j]  (adjoint of a gather with unique indices; dst is zero-filled by the caller)
__global__ void __launch_bounds__(256)
k_scatter_f32(const float *__restrict__ src, const int64_t *__restrict__ idx, int64_t n, float *__restrict__ dst, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) dst[idx[j]] = src[j];
}


// ------------------------------------------------------------------------------------------------ AABB ray test
// AABBSpace.ray_test (models/spatial/aabb.py:71-99) + ray_box_intersection_fast_float_nocheck (graphics/raytest.py:162-167):
// o' = (o - c) / r, d' = d / r; slab test against [-1,1]^3; clamp by near / far; flag = the reference's mask.
// torch.minimum / maximum / max(dim) / clamp propagate NaN -- so do these helpers (a NaN interval fails every comparison).
__device__ __forceinline__ float min_nan(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b); }
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }

struct RayTestArgs {
    float c[3], r[3];
    float near_clip, far_clip;
    int has_near, has_far;
};

__global__ void __launch_bounds__(256)
k_ray_test_aabb(const float *__restrict__ rays_o, const float *__restrict__ rays_d, int64_t n, const RayTestArgs a, float *__restrict__ o_n,
                float *__restrict__ d_n, float *__restrict__ near, float *__restrict__ far, int32_t *__restrict__ flag,
                unsigned long long *__restrict__ coherent_pairs, unsigned long long *__restrict__ row_len) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int close = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (row_len && i >= 2) {                         // image row length: the first i where the image-x step of the direction reverses
            float rev = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) rev += (rays_d[i * 3 + d] - rays_d[(i - 1) * 3 + d]) * (rays_d[3 + d] - rays_d[d]);
            if (rev < 0.f) atomicMin(row_len, (unsigned long long)i);
        }
        if (coherent_pairs && i > 0) {                   // is ray i a neighbour of ray i-1 (image order)?  -> traversal order of the queries
            float dd = 0.f, od = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                dd = fmaxf(dd, fabsf(rays_d[i * 3 + d] - rays_d[(i - 1) * 3 + d]));
                od = fmaxf(od, fabsf(rays_o[i * 3 + d] - rays_o[(i - 1) * 3 + d]) / a.r[d]);
            }
            const float len = fmaxf(fmaxf(fabsf(rays_d[i * 3]), fabsf(rays_d[i * 3 + 1])), fabsf(rays_d[i * 3 + 2]));
            close += (dd <= 0.03f * len && od <= 0.03f) ? 1u : 0u;
        }
        float tn = 0.f, tf = 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float o = __fdiv_rn(__fsub_rn(rays_o[i * 3 + d], a.c[d]), a.r[d]);
            const float v = __fdiv_rn(rays_d[i * 3 + d], a.r[d]);
            o_n[i * 3 + d] = o;
            d_n[i * 3 + d] = v;
            const float ta = __fdiv_rn(__fsub_rn(-1.f, o), v), tb = __fdiv_rn(__fsub_rn(1.f, o), v);
            const float lo = min_nan(ta, tb), hi = max_nan(ta, tb);
            tn = d == 0 ? lo : max_nan(tn, lo);
            tf = d == 0 ? hi : min_nan(tf, hi);
        }
        if (a.has_near && tn == tn) tn = fmaxf(tn, a.near_clip);      // clamp_min_ keeps NaN
        if (a.has_far && tf == tf) tf = fminf(tf, a.far_clip);
        bool m = (tf > tn) && (tf > (a.has_near ? a.near_clip : 0.f));
        if (a.has_far) m = m && (tn < a.far_clip);
        near[i] = tn;
        far[i] = tf;
        flag[i] = m ? 1 : 0;
    }
    if (coherent_pairs) {
        close = __reduce_add_sync(0xffffffffu, close);
        if ((threadIdx.x & 31) == 0 && close) atomicAdd(coherent_pairs, (unsigned long long)close);
    }
}

// ------------------------------------------------------------------------------------------------ 8 x 4 pixel-block order of the packs
// order[j] = the pack in slot j when the live packs, in ascending pixel order, are re-sorted by (py / 4, px / 8, (py % 4) 8 + px % 8),
// pixel = pix[via ? via[p] : p] = py W + px.  A block row (4 image rows) is a contiguous range of packs; one CTA per block row marks
// the occupied pixels of each 8 x 4 block in a 32-bit mask, scans the popcounts over the blocks, and writes every pack to
// range start + packs in earlier blocks + occupied pixels of its block before it.  Identity without row structure.
constexpr int kOrdT = 256, kOrdMaxBx = 4096;              // blocks per block row: image rows up to 32768 pixels
constexpr int kBlkW = 8, kBlkH = 4;                       // block shape: kBlkW x kBlkH = 32 pixels = one group of the ray-tiled query

__device__ __forceinline__ int64_t pixel_of(const int64_t *__restrict__ pix, const int64_t *__restrict__ via, int64_t p) {
    return pix[via ? via[p] : p];
}

__device__ int64_t lower_bound_pixel(const int64_t *__restrict__ pix, const int64_t *__restrict__ via, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (pixel_of(pix, via, mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kOrdT)
k_ray_block_order(const int64_t *__restrict__ pix, const int64_t *__restrict__ via, int64_t n, int64_t n_rays, const int64_t *__restrict__ pairs,
                  const int64_t *__restrict__ row_len, int64_t *__restrict__ order, const int64_t *__restrict__ n_dev) {
    __shared__ uint32_t mask[kOrdMaxBx];
    __shared__ int32_t offs[kOrdMaxBx];
    __shared__ int32_t wsum[kOrdT / 32];
    n = eff_n(n, n_dev);
    const int64_t W = *row_len;
    const bool coherent = n_rays > 64 && 4 * *pairs >= 3 * (n_rays - 1);   // the host-sized path's test (fields/space.py)
    const int64_t nbx = (W + kBlkW - 1) / kBlkW;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (n == 0) return;
    if (!coherent || W < 2 || nbx > kOrdMaxBx) {
        for (int64_t j = (int64_t)blockIdx.x * kOrdT + tid; j < n; j += (int64_t)gridDim.x * kOrdT) order[j] = j;
        return;
    }
    const int64_t rows = kBlkH * W, n_brows = pixel_of(pix, via, n - 1) / rows + 1;
    constexpr int kPer = kOrdMaxBx / kOrdT;
    for (int64_t by = blockIdx.x; by < n_brows; by += gridDim.x) {
        const int64_t lo = lower_bound_pixel(pix, via, n, by * rows), hi = lower_bound_pixel(pix, via, n, (by + 1) * rows);
        for (int64_t b = tid; b < nbx; b += kOrdT) mask[b] = 0u;
        __syncthreads();
        for (int64_t p = lo + tid; p < hi; p += kOrdT) {
            const int64_t q = pixel_of(pix, via, p) - by * rows, py = q / W, px = q - py * W;
            atomicOr(&mask[px / kBlkW], 1u << (py * kBlkW + px % kBlkW));
        }
        __syncthreads();
        int loc = 0;                                          // exclusive scan of the block popcounts: kPer consecutive blocks per thread
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int b = tid * kPer + k;
            if (b < nbx) loc += __popc(mask[b]);
        }
        int incl = loc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        int run = incl - loc;
        for (int w = 0; w < warp; ++w) run += wsum[w];
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int b = tid * kPer + k;
            if (b < nbx) { offs[b] = run; run += __popc(mask[b]); }
        }
        __syncthreads();
        for (int64_t p = lo + tid; p < hi; p += kOrdT) {
            const int64_t q = pixel_of(pix, via, p) - by * rows, py = q / W, px = q - py * W;
            const uint32_t bit = (uint32_t)(py * kBlkW + px % kBlkW);
            order[lo + offs[px / kBlkW] + __popc(mask[px / kBlkW] & ((1u << bit) - 1u))] = p;
        }
        __syncthreads();                                      // mask / offs are rewritten for the next block row
    }
}

// compaction of the rays that passed: row j of every output = row idx[j] of the inputs
__global__ void __launch_bounds__(256)
k_gather_rays(const int64_t *__restrict__ idx, int64_t n, const float *__restrict__ o_n, const float *__restrict__ d_n, const float *__restrict__ near,
              const float *__restrict__ far, float *__restrict__ o_c, float *__restrict__ d_c, float *__restrict__ near_c, float *__restrict__ far_c,
              const float *__restrict__ extra, float *__restrict__ extra_c, int extra_cols, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const int64_t i = idx[j];
#pragma unroll
        for (int d = 0; d < 3; ++d) { o_c[j * 3 + d] = o_n[i * 3 + d]; d_c[j * 3 + d] = d_n[i * 3 + d]; }
        near_c[j] = near[i];
        far_c[j] = far[i];
        for (int c = 0; c < extra_cols; ++c) extra_c[j * extra_cols + c] = extra[i * extra_cols + c];     // per-ray payload (h_appear)
    }
}

// Adjoint of the ray test's normalisation and gather, and of the view directions, for learnable rays:
//   o' = (o - c) / r, d' = d / r              (nr3d_lib/models/spatial/aabb.py:71-80, normalize_rays)
//   o_c = o'[idx], d_c = d'[idx]              (k_gather_rays; aabb.py:97-99 indexes the rays that pass)
//   view_dirs = d_c / clamp(|d_c|, 1e-10)     with the norm detached (nr3d_lib/graphics/neus/neus_ray_query.py:793-794)
// g_o, g_d, g_vd hold the loss's gradient to o_c, d_c and view_dirs of compacted ray j at row idx[j] (the caller's order: the SDF and
// colour backward passes add their per-ray sums there through the ray map idx); vnorm[j] is the clamped norm the forward divided by.
// For j below the count, with i = idx[j]:
//   d_o[i] = (0 + g_o[i]) / r          d_d[i] = (0 + (g_d[i] + g_vd[i] / vnorm[j])) / r          (per axis; g_vd NULL: no view term)
// which is what torch autograd computes for the same chain: the three contributions to d_c arrive as colour + boundary (both inside
// g_d) and then the view term (DivBackward of view_dirs, created before both ops, runs after them), the index backward adds onto zeros,
// and the division's backward divides by r (IEEE division, not a reciprocal).  Rows of rays that fail the test are not written.
__global__ void __launch_bounds__(256)
k_gather_rays_backward(const int64_t *__restrict__ idx, int64_t n, const float r0, const float r1, const float r2,
                       const float *__restrict__ g_o, const float *__restrict__ g_d, const float *__restrict__ g_vd, const float *__restrict__ vnorm,
                       float *__restrict__ d_o, float *__restrict__ d_d, const int64_t *__restrict__ n_dev) {
    n = eff_n(n, n_dev);
    const float r[3] = {r0, r1, r2};
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const int64_t i = idx[j];
        const float vn = g_vd ? vnorm[j] : 1.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            float gd = g_d[i * 3 + d];
            if (g_vd) gd = __fadd_rn(gd, __fdiv_rn(g_vd[i * 3 + d], vn));
            d_o[i * 3 + d] = __fdiv_rn(__fadd_rn(0.f, g_o[i * 3 + d]), r[d]);
            d_d[i * 3 + d] = __fdiv_rn(__fadd_rn(0.f, gd), r[d]);
        }
    }
}

// flag[i] = (v[i] != 0) for i < n_eff, 0 up to the capacity n: the input of the scan that compacts the samples with a non-zero cotangent
__global__ void __launch_bounds__(256)
k_flag_nonzero(const float *__restrict__ v, int64_t n, int32_t *__restrict__ flag, const int64_t *__restrict__ n_dev) {
    const int64_t ne = eff_n(n, n_dev), stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) flag[i] = (i < ne && v[i] != 0.f) ? 1 : 0;
}

// Derived sizes of one NeuS query, kept on the device (nsb_query_counts; slot layout in include/neuralsim_b200.h).
__global__ void k_query_counts(int64_t *__restrict__ c, int phase, int nc, int n_stage, int nf0, int nf1, int nf2, int nf3, int64_t march_cap,
                               int64_t kept_cap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (phase == 0) {                                     // after the scan of the march counts: c[3] = M, c[4] = n_hit
        const int nf[4] = {nf0, nf1, nf2, nf3};
        int64_t M = c[3], nh = c[4];
        int64_t worst = M, tot = 0;
        for (int q = 0; q + 1 < n_stage; ++q) worst += nh * nf[q];        // the merged buffers grow by nf_q samples per hit ray and stage
        if (worst > march_cap) { c[20] |= 1; M = 0; nh = 0; }             // arena too small: the step renders nothing and says so
        c[12] = M;
        c[13] = nh;
        int64_t merged = M;
        for (int q = 0; q < 4; ++q) {
            c[14 + q] = q < n_stage ? nh * nf[q] : 0;
            if (q < n_stage) tot += nf[q];
            if (q + 1 < n_stage) merged += nh * nf[q];
            c[22 + q] = merged;                           // samples in the merged buffer after stage q
        }
        c[18] = c[0] * nc + nh * tot;                      // S: boundary samples
    } else {                                              // after the scan of the kept counts: c[6] = K, c[7] = rays that keep samples
        int64_t K = c[6], pu = c[7];
        const bool fits = K <= kept_cap;
        if (!fits) { c[20] |= 2; K = 0; pu = 0; }
        c[19] = K;
        c[21] = pu;
        c[26] = fits ? c[0] : 0;                           // packs the compaction of the kept samples may walk
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

extern "C" int nsb_flag_nonzero(const float *v, int64_t n, int32_t *flag, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(v && flag, "nsb_flag_nonzero: NULL argument");
    k_flag_nonzero<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(v, n, flag, dn.a);
    return check_launch("nsb_flag_nonzero");
}

extern "C" int nsb_query_counts(int64_t *counts, int32_t phase, int32_t n_coarse, const int32_t *n_fine_host, int32_t n_stage, int64_t march_cap,
                                int64_t kept_cap, void *stream) {
    NSB_REQUIRE(counts, "nsb_query_counts: counts is NULL");
    NSB_REQUIRE(n_stage >= 0 && n_stage <= 4 && (n_stage == 0 || n_fine_host), "nsb_query_counts: at most 4 up-sampling stages");
    int nf[4] = {0, 0, 0, 0};
    for (int q = 0; q < n_stage; ++q) nf[q] = n_fine_host[q];
    k_query_counts<<<1, 32, 0, STREAM>>>(counts, phase, n_coarse, n_stage, nf[0], nf[1], nf[2], nf[3], march_cap, kept_cap);
    return check_launch("nsb_query_counts");
}

extern "C" int64_t nsb_scan_workspace_bytes(void) { return (int64_t)sizeof(ScanWs); }

extern "C" int nsb_scan_counts(const int32_t *counts, int64_t n, int32_t *first, int32_t *info2, int64_t *nz_index, int64_t *nz_pack,
                               const int64_t *src, int64_t *nz_src, int64_t *totals, const int64_t *extra_src, int64_t ticket,
                               void *workspace_zeroed, void *stream) {
    NSB_REQUIRE(totals && workspace_zeroed, "nsb_scan_counts: totals / workspace is NULL");
    NSB_REQUIRE(n == 0 || counts, "nsb_scan_counts: counts is NULL");
    NSB_REQUIRE(!nz_src || src, "nsb_scan_counts: nz_src needs src");
    int64_t nb = (n + (int64_t)kScanT * kScanI - 1) / ((int64_t)kScanT * kScanI);
    const int64_t cap = sm_count() < kScanMaxBlocks ? sm_count() : kScanMaxBlocks;
    if (nb > cap) nb = cap;
    if (nb < 1) nb = 1;
    int64_t seg = (n + nb - 1) / nb;
    seg = (seg + kScanI - 1) / kScanI * kScanI;
    k_scan_counts<<<(unsigned)nb, kScanT, 0, STREAM>>>(counts, n, seg, (ScanWs *)workspace_zeroed, first, info2, nz_index, nz_pack, src, nz_src, totals, extra_src, ticket);
    return check_launch("nsb_scan_counts");
}

extern "C" int nsb_merge_sorted_vals(const float *dep_a, const float *sdf_a, const int64_t *pack_infos_a, const float *dep_b, const float *sdf_b,
                                     int64_t n_packs, int32_t n_b, float *dep_m, float *sdf_m, int64_t *pack_infos_m, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(dep_a && pack_infos_a && dep_b && dep_m && pack_infos_m, "nsb_merge_sorted_vals: NULL argument");
    NSB_REQUIRE((sdf_m == nullptr) || (sdf_a && sdf_b), "nsb_merge_sorted_vals: sdf_m needs sdf_a and sdf_b");
    NSB_REQUIRE(n_b > 0 && n_b <= 1024, "nsb_merge_sorted_vals: n_b must be in [1, 1024]");
    const size_t smem = (size_t)kMergeWarps * n_b * sizeof(float);
    k_merge_vals<<<wave_grid(n_packs * 32, kMergeWarps * 32, 8), kMergeWarps * 32, smem, STREAM>>>(dep_a, sdf_a, pack_infos_a, dep_b, sdf_b, n_packs, n_b,
                                                                                                 dep_m, sdf_m, pack_infos_m, dn.a);
    return check_launch("nsb_merge_sorted_vals");
}

extern "C" int nsb_assemble_boundary(const float *coarse, int64_t n_rays, int32_t n_coarse, const int64_t *ridx_hit, int64_t n_hit, const float *fine,
                                     int32_t n_fine, const int32_t *run_len, int32_t n_runs, float *d1, float *mid, int64_t *ridx_all,
                                     int64_t *pack_infos, void *stream) {
    const DevCounts dn = take_counts();
    if (n_rays == 0) return 0;
    NSB_REQUIRE(coarse && d1 && pack_infos, "nsb_assemble_boundary: NULL argument");
    NSB_REQUIRE(n_hit == 0 || (ridx_hit && fine), "nsb_assemble_boundary: hit rays need ridx_hit and fine");
    NSB_REQUIRE(n_coarse > 0 && n_fine >= 0 && n_coarse + n_fine <= 1024, "nsb_assemble_boundary: n_coarse + n_fine must be <= 1024");
    const size_t smem = (size_t)kAsmWarps * 2 * (n_coarse + n_fine) * sizeof(float);
    NSB_REQUIRE(smem <= 96 * 1024, "nsb_assemble_boundary: too many samples per ray for shared memory");
    AsmRuns runs{};
    NSB_REQUIRE(n_runs >= 0 && n_runs <= kAsmMaxRuns && (n_runs == 0 || run_len), "nsb_assemble_boundary: at most %d sorted runs", kAsmMaxRuns);
    int tot = 0;
    for (int q = 0; q < n_runs; ++q) { runs.len[q] = run_len[q]; tot += run_len[q]; }
    runs.n = n_runs;
    NSB_REQUIRE(tot == n_fine, "nsb_assemble_boundary: run lengths must add up to n_fine");
    const unsigned grid = wave_grid(n_rays * 32, kAsmWarps * 32, 8);
    opt_in_smem(k_assemble_boundary, 96 * 1024);
    k_assemble_boundary<<<grid, kAsmWarps * 32, smem, STREAM>>>(coarse, n_rays, n_coarse, ridx_hit, n_hit, fine, n_fine, runs, d1, mid, ridx_all, pack_infos,
                                                               dn.a, dn.b);
    return check_launch("nsb_assemble_boundary");
}

extern "C" int nsb_compact_samples(const uint8_t *selector, const int64_t *pack_infos, const int32_t *first_out, const int32_t *kept, int64_t n_packs,
                                   const int64_t *ridx_all, const float *t, const float *d1, const float *alpha, int64_t *pidx, int64_t *ridx_c,
                                   float *t_c, float *alpha_c, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(selector && pack_infos && first_out && kept && (t || d1) && alpha && pidx && ridx_c && t_c && alpha_c,
                "nsb_compact_samples: NULL argument");
    k_compact_samples<<<wave_grid(n_packs * 32, 256, 8), 256, 0, STREAM>>>(selector, pack_infos, first_out, kept, n_packs, ridx_all, t, d1, alpha, pidx,
                                                                          ridx_c, t_c, alpha_c, dn.a);
    return check_launch("nsb_compact_samples");
}

extern "C" int nsb_scatter_f32(const float *src, const int64_t *idx, int64_t n, float *dst, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(src && idx && dst, "nsb_scatter_f32: NULL argument");
    k_scatter_f32<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(src, idx, n, dst, dn.a);
    return check_launch("nsb_scatter_f32");
}

extern "C" int nsb_ray_test_aabb(const float *rays_o, const float *rays_d, int64_t n, const float *center3, const float *radius3, int has_near,
                                 float near_clip, int has_far, float far_clip, float *o_n, float *d_n, float *near, float *far, int32_t *flag,
                                 int64_t *coherent_pairs, int64_t *row_len, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(rays_o && rays_d && center3 && radius3 && o_n && d_n && near && far && flag, "nsb_ray_test_aabb: NULL argument");
    RayTestArgs a{{center3[0], center3[1], center3[2]}, {radius3[0], radius3[1], radius3[2]}, near_clip, far_clip, has_near, has_far};
    if (row_len && cudaMemsetAsync(row_len, 0xff, sizeof(int64_t), STREAM) != cudaSuccess) return check_launch("nsb_ray_test_aabb (row length)");
    k_ray_test_aabb<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(rays_o, rays_d, n, a, o_n, d_n, near, far, flag, (unsigned long long *)coherent_pairs,
                                                           (unsigned long long *)row_len);
    return check_launch("nsb_ray_test_aabb");
}

extern "C" int nsb_ray_block_order(const int64_t *pix, const int64_t *via, int64_t n_packs, int64_t n_rays, const int64_t *pairs, const int64_t *row_len,
                                   int64_t *order, void *stream) {
    const DevCounts dn = take_counts();
    if (n_packs == 0) return 0;
    NSB_REQUIRE(pix && pairs && row_len && order, "nsb_ray_block_order: NULL argument");
    k_ray_block_order<<<wave_grid(n_packs, 4 * 32 * 8, 1), kOrdT, 0, STREAM>>>(pix, via, n_packs, n_rays, pairs, row_len, order, dn.a);
    return check_launch("nsb_ray_block_order");
}

extern "C" int nsb_gather_rays(const int64_t *idx, int64_t n, const float *o_n, const float *d_n, const float *near, const float *far, float *o_c,
                               float *d_c, float *near_c, float *far_c, const float *extra, float *extra_c, int32_t extra_cols, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(idx && o_n && d_n && near && far && o_c && d_c && near_c && far_c, "nsb_gather_rays: NULL argument");
    NSB_REQUIRE(extra_cols == 0 || (extra && extra_c), "nsb_gather_rays: extra payload needs both pointers");
    k_gather_rays<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(idx, n, o_n, d_n, near, far, o_c, d_c, near_c, far_c, extra, extra_c, extra_cols, dn.a);
    return check_launch("nsb_gather_rays");
}

extern "C" int nsb_gather_rays_backward(const int64_t *idx, int64_t n, const float *radius3, const float *g_o, const float *g_d, const float *g_vd,
                                        const float *vnorm, float *d_rays_o, float *d_rays_d, void *stream) {
    const DevCounts dn = take_counts();
    if (n == 0) return 0;
    NSB_REQUIRE(idx && radius3 && g_o && g_d && d_rays_o && d_rays_d, "nsb_gather_rays_backward: NULL argument");
    NSB_REQUIRE(!g_vd || vnorm, "nsb_gather_rays_backward: the view-direction term needs vnorm");
    k_gather_rays_backward<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(idx, n, radius3[0], radius3[1], radius3[2], g_o, g_d, g_vd, vnorm, d_rays_o,
                                                                     d_rays_d, dn.a);
    return check_launch("nsb_gather_rays_backward");
}
