// Device-side building blocks of the LoTD encoding shared by lotd.cu and the fused kernels.
// Index / hash arithmetic follows nr3d_lib/csrc/lotd/include/lotd/lotd_cuda.h:92-143,
// position arithmetic lotd_cuda.h:959-984 (InterpolationType::Linear).
#pragma once
#include <type_traits>

#include "nsb_common.cuh"

namespace nsb {

constexpr int kMaxPseudo = 32;

// Per-pseudo-level view of nsb_lotd_meta, passed to kernels by value (~1.6 KB of kernel parameters).
struct PLMeta {
    uint32_t n_pseudo, n_out, D, F;
    uint32_t level[kMaxPseudo];     // actual level of the pseudo level (for max_level masking)
    uint32_t res[kMaxPseudo][NSB_MAX_DIMS];
    uint32_t base[kMaxPseudo];      // element offset of (level, pseudo slot) inside the flat table
    uint32_t nfeat[kMaxPseudo];     // feature width of the actual level (row stride of a cell)
    uint32_t size[kMaxPseudo];      // cells of the level (hash modulus)
    uint32_t mask[kMaxPseudo];      // size-1 when the hash modulus is a power of two, else 0
    uint32_t is_hash;               // bit p set -> hashed level
};

inline int make_plmeta(const nsb_lotd_meta *m, PLMeta *o) {
    if (m->n_pseudo_levels > (uint32_t)kMaxPseudo) {
        set_error("LoTD: %u pseudo levels exceed the built maximum %d", m->n_pseudo_levels, kMaxPseudo);
        return 2;
    }
    memset(o, 0, sizeof(*o));
    o->n_pseudo = m->n_pseudo_levels;
    o->n_out = m->n_encoded_dims;
    o->D = m->n_dims_to_encode;
    o->F = m->n_feat_per_pseudo_lvl;
    for (uint32_t p = 0; p < m->n_pseudo_levels; ++p) {
        const uint32_t l = m->map_levels[p];
        o->level[p] = l;
        for (int d = 0; d < NSB_MAX_DIMS; ++d) o->res[p][d] = m->level_res[l][d];
        o->base[p] = m->level_offsets[l] + m->map_cnt[p] * m->n_feat_per_pseudo_lvl;
        o->nfeat[p] = m->level_n_feats[l];
        o->size[p] = m->level_sizes[l];
        o->mask[p] = (o->size[p] & (o->size[p] - 1)) == 0 ? o->size[p] - 1 : 0;
        if (m->level_types[l] == NSB_LOD_HASH) {
            if (p >= 32) { set_error("LoTD: hashed pseudo level index >= 32 unsupported"); return 2; }
            o->is_hash |= (1u << p);
        }
    }
    return 0;
}

template <bool HALF> struct ValT { using type = float; };
template <> struct ValT<true> { using type = __half; };

__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <typename T> __device__ __forceinline__ T add_st(T a, T b);
template <> __device__ __forceinline__ float add_st<float>(float a, float b) { return __fadd_rn(a, b); }
template <> __device__ __forceinline__ __half add_st<__half>(__half a, __half b) { return __hadd(a, b); }

// network space [-1,1] -> table space [0,1] (lotd_encoding.py:165), clamped (lotd.py:60)
__device__ __forceinline__ float to_table_space(float x) { return fminf(fmaxf(__fmaf_rn(x, 0.5f, 0.5f), 1.0e-6f), 1.f - 1.0e-6f); }

// cell = floor(x*scale+0.5), frac = the remainder; scale = res-2 (lotd_hash_only.h:67).  One FMA, as nvcc emits
// for the reference expression `positions[dim] * scale[dim] + 0.5f`.
template <int D>
__device__ __forceinline__ void level_pos(const PLMeta &m, uint32_t p, const float (&xs)[D], uint32_t (&cell)[D],
                                          float (&fr)[D], float (&scale)[D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
        scale[d] = (float)(m.res[p][d] - 2u);
        const float v = __fmaf_rn(xs[d], scale[d], 0.5f);
        const float fl = floorf(v);
        cell[d] = (uint32_t)fl;
        fr[d] = v - fl;
    }
}

// weight of corner c: prod_d (bit d of c ? frac_d : 1-frac_d), multiplied in dimension order.
template <int D>
__device__ __forceinline__ float corner_weight(const float (&fr)[D], int c) {
    float w = (c & 1) ? fr[0] : __fsub_rn(1.f, fr[0]);
#pragma unroll
    for (int d = 1; d < D; ++d) w = __fmul_rn(w, (c & (1 << d)) ? fr[d] : __fsub_rn(1.f, fr[d]));
    return w;
}

template <int D>
__device__ __forceinline__ uint32_t corner_index(const PLMeta &m, uint32_t p, const uint32_t (&cell)[D], int c) {
    uint32_t idx;
    if (m.is_hash & (1u << p)) {
        constexpr uint32_t primes[4] = {1u, 2654435761u, 805459861u, 3674653429u};
        idx = 0;
#pragma unroll
        for (int d = 0; d < D; ++d) idx ^= (cell[d] + ((c >> d) & 1)) * primes[d];
        idx %= m.size[p];
    } else {
        idx = 0;
        uint32_t stride = 1;
#pragma unroll
        for (int d = D - 1; d >= 0; --d) {  // last dimension contiguous
            idx += (cell[d] + ((c >> d) & 1)) * stride;
            stride *= m.res[p][d];
        }
    }
    return idx * m.nfeat[p] + m.base[p];
}

template <int D, int F, typename VT>
__device__ __forceinline__ void load_corner(const PLMeta &m, uint32_t p, const VT *__restrict__ grid,
                                            const uint32_t (&cell)[D], int c, VT (&out)[F]) {
    const uint32_t e = corner_index<D>(m, p, cell, c);
    if constexpr (std::is_same<VT, __half>::value) {
#pragma unroll
        for (int f = 0; f < F; f += 2) {
            const uint32_t raw = ld_nc_u32(grid + e + f);
            out[f] = __ushort_as_half((unsigned short)(raw & 0xffffu));
            out[f + 1] = __ushort_as_half((unsigned short)(raw >> 16));
        }
    } else {
#pragma unroll
        for (int f = 0; f < F; ++f) out[f] = __ldg(grid + e + f);
    }
}

// All 8 corner element offsets and trilinear weights of one 3-D level with few instructions: dense strides / hash terms
// are formed once and combined per corner (uint32 wrap-around arithmetic, identical to corner_index<3>), and the
// modulus is a mask when the table size is a power of two.  Weights keep the (wx*wy)*wz rounding order.
__device__ __forceinline__ void level_corners3(const PLMeta &m, uint32_t p, const float (&xs)[3], uint32_t (&idx)[8], float (&w)[8]) {
    const uint32_t rx = m.res[p][0], ry = m.res[p][1], rz = m.res[p][2];
    uint32_t cell[3];
    float fr[3];
    {
        const float sx = (float)(rx - 2u), sy = (float)(ry - 2u), sz = (float)(rz - 2u);
        const float vx = __fmaf_rn(xs[0], sx, 0.5f), vy = __fmaf_rn(xs[1], sy, 0.5f), vz = __fmaf_rn(xs[2], sz, 0.5f);
        const float fx = floorf(vx), fy = floorf(vy), fz = floorf(vz);
        cell[0] = (uint32_t)fx; cell[1] = (uint32_t)fy; cell[2] = (uint32_t)fz;
        fr[0] = vx - fx; fr[1] = vy - fy; fr[2] = vz - fz;
    }
    const float wx0 = __fsub_rn(1.f, fr[0]), wy0 = __fsub_rn(1.f, fr[1]), wz0 = __fsub_rn(1.f, fr[2]);
    const float w00 = __fmul_rn(wx0, wy0), w10 = __fmul_rn(fr[0], wy0), w01 = __fmul_rn(wx0, fr[1]), w11 = __fmul_rn(fr[0], fr[1]);
    w[0] = __fmul_rn(w00, wz0); w[1] = __fmul_rn(w10, wz0); w[2] = __fmul_rn(w01, wz0); w[3] = __fmul_rn(w11, wz0);
    w[4] = __fmul_rn(w00, fr[2]); w[5] = __fmul_rn(w10, fr[2]); w[6] = __fmul_rn(w01, fr[2]); w[7] = __fmul_rn(w11, fr[2]);
    const uint32_t nf = m.nfeat[p], base = m.base[p];
    if (m.is_hash & (1u << p)) {
        const uint32_t hx0 = cell[0], hx1 = cell[0] + 1u;
        const uint32_t hy0 = cell[1] * 2654435761u, hy1 = hy0 + 2654435761u;
        const uint32_t hz0 = cell[2] * 805459861u, hz1 = hz0 + 805459861u;
        const uint32_t a00 = hy0 ^ hz0, a10 = hy1 ^ hz0, a01 = hy0 ^ hz1, a11 = hy1 ^ hz1;
        uint32_t h[8] = {hx0 ^ a00, hx1 ^ a00, hx0 ^ a10, hx1 ^ a10, hx0 ^ a01, hx1 ^ a01, hx0 ^ a11, hx1 ^ a11};
        const uint32_t mask = m.mask[p], size = m.size[p];
#pragma unroll
        for (int c = 0; c < 8; ++c) idx[c] = (mask ? (h[c] & mask) : (h[c] % size)) * nf + base;
    } else {
        const uint32_t sy_ = rz, sx_ = ry * rz;
        const uint32_t b0 = (cell[0] * ry + cell[1]) * rz + cell[2];
#pragma unroll
        for (int c = 0; c < 8; ++c) idx[c] = (b0 + ((c & 1) ? sx_ : 0u) + ((c & 2) ? sy_ : 0u) + ((c & 4) ? 1u : 0u)) * nf + base;
    }
}

// ---- fast path of the fused kernels: every level carries 2 features per cell (one cell == one 32-bit word of the fp16
// table, one float2 of the fp32 gradient), so a corner is addressed as `level_pointer + cell` with ONE wide multiply-add.
// floor() is taken with the 2^23 trick (v in [0.5, 2^22): fadd.rm(v, 2^23) = 2^23 + floor(v), the integer sits in the
// mantissa) -- two full-rate FADDs instead of FRND + F2I; `v - floor(v)` is the same fp32 value as in level_corners3.
__device__ __forceinline__ void level_cells3(const PLMeta &m, uint32_t p, const float (&xs)[3], uint32_t (&cell)[8], float (&w)[8],
                                             float (&fr)[3], float (&sc)[3]) {
    const uint32_t rx = m.res[p][0], ry = m.res[p][1], rz = m.res[p][2];
    sc[0] = (float)(rx - 2u); sc[1] = (float)(ry - 2u); sc[2] = (float)(rz - 2u);
    const float vx = __fmaf_rn(xs[0], sc[0], 0.5f), vy = __fmaf_rn(xs[1], sc[1], 0.5f), vz = __fmaf_rn(xs[2], sc[2], 0.5f);
    const float tx = __fadd_rd(vx, 8388608.f), ty = __fadd_rd(vy, 8388608.f), tz = __fadd_rd(vz, 8388608.f);
    const uint32_t cx = __float_as_uint(tx) - 0x4B000000u, cy = __float_as_uint(ty) - 0x4B000000u, cz = __float_as_uint(tz) - 0x4B000000u;
    fr[0] = vx - (tx - 8388608.f); fr[1] = vy - (ty - 8388608.f); fr[2] = vz - (tz - 8388608.f);
    const float wx0 = __fsub_rn(1.f, fr[0]), wy0 = __fsub_rn(1.f, fr[1]), wz0 = __fsub_rn(1.f, fr[2]);
    const float w00 = __fmul_rn(wx0, wy0), w10 = __fmul_rn(fr[0], wy0), w01 = __fmul_rn(wx0, fr[1]), w11 = __fmul_rn(fr[0], fr[1]);
    w[0] = __fmul_rn(w00, wz0); w[1] = __fmul_rn(w10, wz0); w[2] = __fmul_rn(w01, wz0); w[3] = __fmul_rn(w11, wz0);
    w[4] = __fmul_rn(w00, fr[2]); w[5] = __fmul_rn(w10, fr[2]); w[6] = __fmul_rn(w01, fr[2]); w[7] = __fmul_rn(w11, fr[2]);
    if (m.is_hash & (1u << p)) {
        const uint32_t hx0 = cx, hx1 = cx + 1u;
        const uint32_t hy0 = cy * 2654435761u, hy1 = hy0 + 2654435761u;
        const uint32_t hz0 = cz * 805459861u, hz1 = hz0 + 805459861u;
        const uint32_t a00 = hy0 ^ hz0, a10 = hy1 ^ hz0, a01 = hy0 ^ hz1, a11 = hy1 ^ hz1;
        const uint32_t h[8] = {hx0 ^ a00, hx1 ^ a00, hx0 ^ a10, hx1 ^ a10, hx0 ^ a01, hx1 ^ a01, hx0 ^ a11, hx1 ^ a11};
        const uint32_t mask = m.mask[p];
        if (mask) {
#pragma unroll
            for (int c = 0; c < 8; ++c) cell[c] = h[c] & mask;
        } else {
            const uint32_t size = m.size[p];
#pragma unroll
            for (int c = 0; c < 8; ++c) cell[c] = h[c] % size;
        }
    } else {
        const uint32_t sy_ = rz, sx_ = ry * rz;
        const uint32_t b0 = (cx * ry + cy) * rz + cz;
        cell[0] = b0; cell[1] = b0 + sx_; cell[2] = b0 + sy_; cell[3] = cell[1] + sy_;
        cell[4] = b0 + 1u; cell[5] = cell[1] + 1u; cell[6] = cell[2] + 1u; cell[7] = cell[3] + 1u;
    }
}

__device__ __forceinline__ void level_cells3(const PLMeta &m, uint32_t p, const float (&xs)[3], uint32_t (&cell)[8], float (&w)[8]) {
    float fr[3], sc[3];
    level_cells3(m, p, xs, cell, w, fr, sc);
}

// fp16 table viewed as 32-bit cells of level p / fp32 gradient viewed as float2 cells of level p
// (the empty asm keeps the level pointer in an ordinary 64-bit register: `pointer + cell` is then ONE IMAD.WIDE with an immediate
//  stride; with the pointer in a uniform register ptxas needs an extra MOV per corner for the stride)
__device__ __forceinline__ const uint32_t *level_cells_ptr(const PLMeta &m, uint32_t p, const __half *grid) {
    const uint32_t *q = reinterpret_cast<const uint32_t *>(grid + m.base[p]);
    asm volatile("" : "+l"(q));
    return q;
}
__device__ __forceinline__ float2 *level_grad_ptr(const PLMeta &m, uint32_t p, float *d_grid) {
    float2 *q = reinterpret_cast<float2 *>(d_grid + m.base[p]);
    asm volatile("" : "+l"(q));
    return q;
}

// the fp16 feature pair of one level from its 8 corner cells as loaded (two fp16 features per 32-bit word) and their trilinear weights
__device__ __forceinline__ uint32_t feat2_from_raw(const uint32_t (&raw)[8], const float (&w)[8]) {
    __half2 acc = __floats2half2_rn(0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float2 v = __half22float2(*reinterpret_cast<const __half2 *>(&raw[c]));
        acc = __hadd2(acc, __floats2half2_rn(__fmul_rn(w[c], v.x), __fmul_rn(w[c], v.y)));
    }
    return *reinterpret_cast<uint32_t *>(&acc);
}

__device__ __forceinline__ uint32_t level_feat2_cells(const uint32_t *__restrict__ lp, const uint32_t (&cell)[8], const float (&w)[8]) {
    uint32_t raw[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) raw[c] = ld_nc_u32(lp + cell[c]);
    return feat2_from_raw(raw, w);
}

__device__ __forceinline__ void red_add2(float2 *dst, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
}

// ---- warp-merged table-gradient updates.  The fp32 atomics themselves bound the table
// backward (the same rate whether the points are ordered or shuffled, at any occupancy), so the lever is FEWER atomics.
// The lanes of a warp are consecutive samples of a ray; neighbouring samples fall into the same cell on the coarse and middle levels,
// and on the finest levels too where the up-sampled samples crowd around the surface.  Runs of lanes with equal integer cell
// coordinates are summed with shuffles (segmented reduction over contiguous runs; the run structure is one ballot) and only the run's
// first lane issues the 8 reductions.
// `key` must identify the cell exactly (not its hash); lanes that carry no gradient pass active = false.
constexpr uint32_t kCellKeyBits = 21;                  // per axis: the three cell coordinates of any level with res <= 2^21 per axis
__device__ __forceinline__ uint64_t cell_key3(const PLMeta &m, uint32_t p, const float (&xs)[3]) {
    uint64_t k = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float v = __fmaf_rn(xs[d], (float)(m.res[p][d] - 2u), 0.5f);
        k |= (uint64_t)(__float_as_uint(__fadd_rd(v, 8388608.f)) - 0x4B000000u) << (kCellKeyBits * d);
    }
    return k;
}
// host: every axis of every pseudo level fits the key (a cell coordinate is < res)
inline bool plmeta_cell_key_fits(const PLMeta &m) {
    for (uint32_t p = 0; p < m.n_pseudo; ++p)
        for (uint32_t d = 0; d < m.D; ++d)
            if (m.res[p][d] > (1u << kCellKeyBits)) return false;
    return true;
}

// a[c], b[c]: this lane's updates of corner c (feature 0 / 1).  On return the lanes for which the result is true hold the sums of
// their run and must issue them; the others are done.  Every lane of the warp must call (shuffles).
__device__ __forceinline__ bool warp_merge_updates(uint64_t key, bool active, float (&a)[8], float (&b)[8], int lane) {
    const uint64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
    const uint32_t act = __ballot_sync(0xffffffffu, active);
    const bool prev_act = lane > 0 && ((act >> (lane - 1)) & 1u);
    const bool head = !active || !prev_act || key != prev;       // inactive lanes are runs of their own
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    if (__popc(heads) > 24) return active;                       // (warp-uniform) little to merge: everyone issues its own
    const uint32_t after = lane == 31 ? 0xffffffffu : (heads >> (lane + 1));   // bit j: lane + 1 + j starts a new run
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const bool take = (lane + o < 32) && ((after & ((1u << o) - 1u)) == 0u);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float av = __shfl_down_sync(0xffffffffu, a[c], o), bv = __shfl_down_sync(0xffffffffu, b[c], o);
            if (take) { a[c] += av; b[c] += bv; }
        }
    }
    return active && head;
}

// true when every pseudo level is a 2-feature level stored at an even element offset (the fast path's precondition)
inline bool plmeta_two_feature_cells(const PLMeta &m) {
    for (uint32_t p = 0; p < m.n_pseudo; ++p)
        if (m.nfeat[p] != 2u || (m.base[p] & 1u)) return false;
    return m.F == 2u;
}

// grad[dst .. dst+F) += g[f] * w, fp32, fire-and-forget vector reductions (8-byte aligned: F even, offsets even).
template <int F>
__device__ __forceinline__ void red_add(float *dst, const float (&g)[F], float w) {
#pragma unroll
    for (int f = 0; f < F; f += 2) {
        const float a = g[f] * w, b = g[f + 1] * w;
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + f), "f"(a), "f"(b) : "memory");
    }
}

}  // namespace nsb
