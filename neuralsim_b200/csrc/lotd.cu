// LoTD (Dense + Hash multi-resolution grid) encoding kernels for sm_90a and their C entry points.
//
// Replaces the reference's `_lotd` extension for the c_hash_only path
// (nr3d_lib/csrc/lotd/include/lotd/lotd_hash_only.h).  Different design:
//   * point-major: one thread walks all pseudo-levels of its point, so the [N,F] feature row is produced
//     contiguously (the reference runs a (points x levels) grid and writes a transposed [F,N] tensor);
//   * fp32 gradient accumulation with vector reductions (red.global.add.v2.f32) instead of fp16 atomics;
//   * the rounding sequence of the forward pass is pinned with explicit _rn intrinsics so that y is
//     bit-identical to the reference's <float, half, float> instantiation (fp16 accumulation over the
//     corners in corner order, linear_interpolate.cuh:102-120).
#include "lotd_device.cuh"

namespace nsb {

// Which table a point reads, for `params` holding several tables (lotd_hash_only.h:44-55): the point's batch is inds[i]
// (negative: the point is skipped), else i / data_size (data_size != 0), else 0; its table starts at offsets[batch], else
// at batch * table_size.  The start is formed in 64 bits (the reference's is a uint32_t and wraps past 2^32 elements).
struct LotdBatch {
    const int64_t *inds;
    const int64_t *offsets;
    uint32_t data_size;
    uint32_t table_size;        // elements of one table (n_params)
};

// false: point i is skipped.  BATCHED = false: one table at offset 0 and no loads, the unbatched code.
template <bool BATCHED>
__device__ __forceinline__ bool table_base(const LotdBatch &b, int64_t i, int64_t &base) {
    base = 0;
    if (!BATCHED) return true;
    int64_t k = 0;
    if (b.inds) {
        k = b.inds[i];
        if (k < 0) return false;
    } else if (b.data_size) {
        k = i / b.data_size;
    }
    base = b.offsets ? b.offsets[k] : k * (int64_t)b.table_size;
    return true;
}

// ------------------------------------------------------------------------------------------------ forward
template <int D, int F, bool HALF, bool DYDX, bool BATCHED>
__global__ void __launch_bounds__(256)
k_lotd_fwd(const PLMeta m, const float *__restrict__ x, const void *__restrict__ grid_, int64_t n, int max_level,
           const LotdBatch batch, void *__restrict__ y_, float *__restrict__ dy_dx) {
    using VT = typename ValT<HALF>::type;
    VT *y = (VT *)y_;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        VT *yo = y + i * m.n_out;
        float *go = DYDX ? dy_dx + i * (int64_t)m.n_out * D : nullptr;
        int64_t tb;
        if (!table_base<BATCHED>(batch, i, tb)) {       // skipped point: zero row, as the reference's at::zeros outputs
            for (uint32_t k = 0; k < m.n_out; ++k) yo[k] = from_float<VT>(0.f);
            if (DYDX)
                for (uint32_t k = 0; k < m.n_out * D; ++k) go[k] = 0.f;
            continue;
        }
        const VT *grid = (const VT *)grid_ + tb;
        float xs[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xs[d] = x[i * D + d];
        for (uint32_t p = 0; p < m.n_pseudo; ++p) {
            if ((int)m.level[p] > max_level) {
#pragma unroll
                for (int f = 0; f < F; ++f) yo[p * F + f] = from_float<VT>(0.f);
                if (DYDX) {
#pragma unroll
                    for (int k = 0; k < F * D; ++k) go[p * F * D + k] = 0.f;
                }
                continue;
            }
            uint32_t cell[D];
            float fr[D], scale[D];
            level_pos<D>(m, p, xs, cell, fr, scale);
            VT v[1 << D][F];
#pragma unroll
            for (int c = 0; c < (1 << D); ++c) load_corner<D, F, VT>(m, p, grid, cell, c, v[c]);
            // y: sequential accumulation in the storage type, corner order 0..2^D-1
            VT acc[F];
#pragma unroll
            for (int f = 0; f < F; ++f) acc[f] = from_float<VT>(0.f);
#pragma unroll
            for (int c = 0; c < (1 << D); ++c) {
                float w = corner_weight<D>(fr, c);
#pragma unroll
                for (int f = 0; f < F; ++f) acc[f] = add_st<VT>(acc[f], from_float<VT>(__fmul_rn(w, to_float(v[c][f]))));
            }
#pragma unroll
            for (int f = 0; f < F; ++f) yo[p * F + f] = acc[f];
            if (DYDX) {
                float g[F][D];
#pragma unroll
                for (int gd = 0; gd < D; ++gd) {
#pragma unroll
                    for (int f = 0; f < F; ++f) g[f][gd] = 0.f;
#pragma unroll
                    for (int c = 0; c < (1 << (D - 1)); ++c) {
                        float w = scale[gd];
                        int left = 0;
#pragma unroll
                        for (int k = 0; k < D - 1; ++k) {
                            const int d = k >= gd ? k + 1 : k;
                            if (c & (1 << k)) { w = __fmul_rn(w, fr[d]); left += 1 << d; }
                            else w = __fmul_rn(w, __fsub_rn(1.f, fr[d]));
                        }
                        const int right = left + (1 << gd);
#pragma unroll
                        for (int f = 0; f < F; ++f)
                            g[f][gd] = __fmaf_rn(w, __fsub_rn(to_float(v[right][f]), to_float(v[left][f])), g[f][gd]);
                    }
                }
#pragma unroll
                for (int f = 0; f < F; ++f)
#pragma unroll
                    for (int d = 0; d < D; ++d) go[(p * F + f) * D + d] = g[f][d];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward (grid)
// one thread per (point, pseudo-level), pseudo-level fastest: a warp reads 64 contiguous bytes of dL_dy per
// point and spreads its reductions over 16 different level tables.
template <int D, int F, bool HALF, bool BATCHED>
__global__ void __launch_bounds__(256)
k_lotd_bwd_grid(const PLMeta m, const void *__restrict__ dL_dy_, const float *__restrict__ x, int64_t n, int max_level,
                const LotdBatch batch, float scale_out, float *__restrict__ grad) {
    using VT = typename ValT<HALF>::type;
    const VT *dL_dy = (const VT *)dL_dy_;
    const int64_t total = n * m.n_pseudo;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t i = t / m.n_pseudo;
        const uint32_t p = (uint32_t)(t - i * m.n_pseudo);
        if ((int)m.level[p] > max_level) continue;
        float xs[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xs[d] = x[i * D + d];
        float g[F];
        bool any = false;
#pragma unroll
        for (int f = 0; f < F; ++f) {
            g[f] = to_float(dL_dy[i * m.n_out + p * F + f]) * scale_out;
            any |= (g[f] != 0.f);
        }
        if (!any) continue;
        int64_t tb;
        if (!table_base<BATCHED>(batch, i, tb)) continue;
        uint32_t cell[D];
        float fr[D], sc[D];
        level_pos<D>(m, p, xs, cell, fr, sc);
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            const float w = corner_weight<D>(fr, c);
            float *dst = grad + tb + corner_index<D>(m, p, cell, c);
            red_add<F>(dst, g, w);
        }
    }
}

// ------------------------------------------------------------------------------------------------ dL_dx = J^T dL_dy
template <bool HALF, bool BATCHED>
__global__ void __launch_bounds__(256)
k_lotd_bwd_input(const void *__restrict__ dL_dy_, const float *__restrict__ dy_dx, int64_t n, int nf, int D,
                 const LotdBatch batch, float scale, float *__restrict__ dL_dx) {
    using VT = typename ValT<HALF>::type;
    const VT *dL_dy = (const VT *)dL_dy_;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (BATCHED && batch.inds && batch.inds[i] < 0) {
            for (int d = 0; d < D; ++d) dL_dx[i * D + d] = 0.f;
            continue;
        }
        float acc[NSB_MAX_DIMS] = {0.f, 0.f, 0.f, 0.f};
        const float *J = dy_dx + i * (int64_t)nf * D;
        for (int f = 0; f < nf; ++f) {
            const float g = to_float(dL_dy[i * nf + f]);
            for (int d = 0; d < D; ++d) acc[d] = __fmaf_rn(g, J[f * D + d], acc[d]);
        }
        for (int d = 0; d < D; ++d) dL_dx[i * D + d] = acc[d] * scale;
    }
}

// ------------------------------------------------------------------------------------------------ second order
template <bool BATCHED>
__global__ void __launch_bounds__(256)
k_lotd_ddLdy(const float *__restrict__ dL_ddLdx, const float *__restrict__ dy_dx, int64_t n, int nf, int D,
             const LotdBatch batch, float *__restrict__ out) {
    const int64_t total = n * nf;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t i = t / nf;
        if (BATCHED && batch.inds && batch.inds[i] < 0) {
            out[t] = 0.f;
            continue;
        }
        float a = 0.f;
        for (int d = 0; d < D; ++d) a = __fmaf_rn(dL_ddLdx[i * D + d], dy_dx[t * D + d], a);
        out[t] = a;
    }
}

template <int D, int F, bool HALF, bool BATCHED>
__global__ void __launch_bounds__(256)
k_lotd_bwd_bwd_grid(const PLMeta m, const float *__restrict__ dL_ddLdx, const void *__restrict__ dL_dy_,
                    const float *__restrict__ x, int64_t n, int max_level, const LotdBatch batch, float scale_out,
                    float *__restrict__ grad) {
    using VT = typename ValT<HALF>::type;
    const VT *dL_dy = (const VT *)dL_dy_;
    const int64_t total = n * m.n_pseudo;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t i = t / m.n_pseudo;
        const uint32_t p = (uint32_t)(t - i * m.n_pseudo);
        if ((int)m.level[p] > max_level) continue;
        float g[F];
        bool any = false;
#pragma unroll
        for (int f = 0; f < F; ++f) {
            g[f] = to_float(dL_dy[i * m.n_out + p * F + f]) * scale_out;
            any |= (g[f] != 0.f);
        }
        if (!any) continue;
        int64_t tb;
        if (!table_base<BATCHED>(batch, i, tb)) continue;
        float xs[D], gin[D];
#pragma unroll
        for (int d = 0; d < D; ++d) { xs[d] = x[i * D + d]; gin[d] = dL_ddLdx[i * D + d]; }
        uint32_t cell[D];
        float fr[D], sc[D];
        level_pos<D>(m, p, xs, cell, fr, sc);
        // d(dL_dx_gd)/dgrid: +-scale_gd * gin_gd * prod_{d != gd} w_d on the two corners along gd.
        // Corner c collects, over gd, sign_gd(c) * scale_gd*gin_gd * prod_{d!=gd} w_d(c).
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            float wsum = 0.f;
#pragma unroll
            for (int gd = 0; gd < D; ++gd) {
                float w = __fmul_rn(sc[gd], gin[gd]);
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    if (d == gd) continue;
                    w = __fmul_rn(w, (c & (1 << d)) ? fr[d] : __fsub_rn(1.f, fr[d]));
                }
                wsum += (c & (1 << gd)) ? w : -w;
            }
            float *dst = grad + tb + corner_index<D>(m, p, cell, c);
            red_add<F>(dst, g, wsum);
        }
    }
}

}  // namespace nsb

// ================================================================================================ C ABI
using namespace nsb;

extern "C" int nsb_lotd_meta_create(int32_t n_dims, int32_t n_levels, const int32_t *lod_res, const int32_t *lod_n_feats,
                                    const int32_t *lod_types, uint32_t hashmap_size, nsb_lotd_meta *out) {
    // Restates LoDMeta::create_meta (lotd_torch_api.cu:29-230) for Dense / Hash levels.
    NSB_REQUIRE(out != nullptr, "nsb_lotd_meta_create: out is NULL");
    NSB_REQUIRE(n_dims == 2 || n_dims == 3 || n_dims == 4, "LoTDEncoding: `n_input_dim` must be 2/3/4.");
    NSB_REQUIRE(n_levels > 0 && n_levels <= NSB_MAX_LEVELS, "LoTDEncoding: `num_level`=%d exceeds maximum level=%d",
                n_levels, NSB_MAX_LEVELS);
    memset(out, 0, sizeof(*out));
    uint32_t g = 0;
    for (uint32_t cand : {8u, 4u, 2u}) {
        bool ok = true;
        for (int l = 0; l < n_levels; ++l) ok &= (lod_n_feats[l] > 0 && lod_n_feats[l] % cand == 0);
        if (ok) { g = cand; break; }
    }
    NSB_REQUIRE(g != 0, "LoTDEncoding: the greatest common divisor of `lod_n_feats` must be at least 2");
    out->n_dims_to_encode = n_dims;
    out->n_levels = n_levels;
    out->n_feat_per_pseudo_lvl = g;
    uint64_t acc = 0;
    uint32_t npl = 0;
    for (int l = 0; l < n_levels; ++l) {
        uint64_t size = 1;
        for (int d = 0; d < n_dims; ++d) {
            int32_t r = lod_res[l * n_dims + d];
            NSB_REQUIRE(r > 2, "LoTDEncoding: only support grid resolutions >= 3");
            out->level_res[l][d] = (uint32_t)r;
            size *= (uint64_t)r;
        }
        if (lod_types[l] == NSB_LOD_HASH) {
            NSB_REQUIRE(hashmap_size != 0, "LoTDEncoding: Hash mode need `hashmap_size`");
            size = hashmap_size;
        } else {
            NSB_REQUIRE(lod_types[l] == NSB_LOD_DENSE, "neuralsim_b200 supports Dense and Hash LoTD levels only (got type %d)",
                        lod_types[l]);
        }
        uint32_t nf = (uint32_t)lod_n_feats[l];
        out->level_types[l] = (uint32_t)lod_types[l];
        out->level_n_feats[l] = nf;
        out->level_sizes[l] = (uint32_t)size;
        out->level_offsets[l] = (uint32_t)acc;
        acc += size * nf;
        NSB_REQUIRE(acc < (1ull << 31), "LoTDEncoding: param size too large.");
        for (uint32_t j = 0; j < nf / g; ++j) {
            NSB_REQUIRE(npl < NSB_MAX_LEVELS * 4, "LoTDEncoding: too many pseudo levels");
            out->map_levels[npl] = l;
            out->map_cnt[npl] = j;
            ++npl;
        }
        out->n_encoded_dims += nf;
    }
    out->level_offsets[n_levels] = (uint32_t)acc;
    out->n_params = (uint32_t)acc;
    out->n_pseudo_levels = npl;
    NSB_REQUIRE(out->n_encoded_dims <= 1024, "LoTDEncoding: total number of features too large. Shoule be <= 1024.");
    return 0;
}

namespace {
template <typename Fn>
int dispatch_DF(const nsb_lotd_meta *meta, const char *who, Fn &&fn) {
    const uint32_t D = meta->n_dims_to_encode, F = meta->n_feat_per_pseudo_lvl;
    if (D == 3 && F == 2) return fn(std::integral_constant<int, 3>{}, std::integral_constant<int, 2>{});
    if (D == 3 && F == 4) return fn(std::integral_constant<int, 3>{}, std::integral_constant<int, 4>{});
    if (D == 4 && F == 2) return fn(std::integral_constant<int, 4>{}, std::integral_constant<int, 2>{});
    if (D == 2 && F == 2) return fn(std::integral_constant<int, 2>{}, std::integral_constant<int, 2>{});
    set_error("%s: unsupported (n_dims_to_encode=%u, n_feat_per_pseudo_lvl=%u); built: (3,2) (3,4) (4,2) (2,2)", who, D, F);
    return 2;
}

// the kernels' view of an nsb_lotd_batch; *batched = false: no batch argument (NULL, or all three fields empty), the unbatched kernels
int make_batch(const nsb_lotd_batch *b, const nsb_lotd_meta *meta, int64_t n, const char *who, LotdBatch *o, bool *batched) {
    *o = LotdBatch{nullptr, nullptr, 0u, meta ? meta->n_params : 0u};
    *batched = b && (b->inds || b->offsets || b->data_size);
    if (!*batched) return 0;
    NSB_REQUIRE(b->data_size == 0 || n % b->data_size == 0,
                "%s: Expect nonzero `batch_data_size`=%u to be a divisor of `batch_size`=%lld", who, b->data_size, (long long)n);
    o->inds = b->inds;
    o->offsets = b->offsets;
    o->data_size = b->data_size;
    return 0;
}

template <typename Fn>
int dispatch_batched(bool batched, Fn &&fn) {
    return batched ? fn(std::true_type{}) : fn(std::false_type{});
}
}  // namespace

// Replaces lod_fwd_common (lotd_torch_api.cu:232-365) with lod_hash_only_fwd_impl and its kernel (lotd_hash_only.h:15-110),
// batch arguments included (lotd_hash_only.h:44-55).
extern "C" int nsb_lotd_fwd_batched(const nsb_lotd_meta *meta, const float *input, const void *params, int params_is_half,
                                    int64_t n, int32_t max_level, const nsb_lotd_batch *batch_host, void *y, float *dy_dx,
                                    void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(meta && y && input && params, "nsb_lotd_fwd: NULL argument");
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    LotdBatch b;
    bool batched;
    if (make_batch(batch_host, meta, n, "LoTDEncoding::fwd", &b, &batched)) return 2;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t esz = params_is_half ? 2 : 4;
    if (max_level <= -1) {  // lotd_torch_api.cu:294-297: zeros
        cudaMemsetAsync(y, 0, (size_t)n * m.n_out * esz, s);
        if (dy_dx) cudaMemsetAsync(dy_dx, 0, (size_t)n * m.n_out * m.D * sizeof(float), s);
        return 0;
    }
    const unsigned grid = wave_grid(n, 256, 4);
    return dispatch_DF(meta, "nsb_lotd_fwd", [&](auto Dc, auto Fc) {
        constexpr int D = decltype(Dc)::value, F = decltype(Fc)::value;
        return dispatch_batched(batched, [&](auto Bc) {
            constexpr bool B = decltype(Bc)::value;
            if (params_is_half) {
                if (dy_dx) k_lotd_fwd<D, F, true, true, B><<<grid, 256, 0, s>>>(m, input, params, n, max_level, b, y, dy_dx);
                else k_lotd_fwd<D, F, true, false, B><<<grid, 256, 0, s>>>(m, input, params, n, max_level, b, y, nullptr);
            } else {
                if (dy_dx) k_lotd_fwd<D, F, false, true, B><<<grid, 256, 0, s>>>(m, input, params, n, max_level, b, y, dy_dx);
                else k_lotd_fwd<D, F, false, false, B><<<grid, 256, 0, s>>>(m, input, params, n, max_level, b, y, nullptr);
            }
            return check_launch("nsb_lotd_fwd");
        });
    });
}

extern "C" int nsb_lotd_fwd(const nsb_lotd_meta *meta, const float *input, const void *params, int params_is_half,
                            int64_t n, int32_t max_level, void *y, float *dy_dx, void *stream) {
    return nsb_lotd_fwd_batched(meta, input, params, params_is_half, n, max_level, nullptr, y, dy_dx, stream);
}

// Replaces the parameter part of lod_bwd_common (lotd_torch_api.cu:397-537): lod_hash_only_bwd_impl and its kernel
// (lotd_hash_only.h:380-470), batch arguments included (lotd_hash_only.h:413-426).
extern "C" int nsb_lotd_bwd_grid_batched(const nsb_lotd_meta *meta, const void *dL_dy, int dL_dy_is_half, const float *input,
                                         int64_t n, int32_t max_level, const nsb_lotd_batch *batch_host, float scale,
                                         float *dL_dparam, void *stream) {
    NSB_REQUIRE(meta && dL_dparam, "nsb_lotd_bwd_grid: NULL argument");
    LotdBatch b;
    bool batched;
    if (make_batch(batch_host, meta, n, "LoTDEncoding::bwd", &b, &batched)) return 2;
    if (n == 0 || max_level <= -1) return 0;
    NSB_REQUIRE(dL_dy && input, "nsb_lotd_bwd_grid: NULL argument");
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned grid = wave_grid(n * m.n_pseudo, 256, 4);
    return dispatch_DF(meta, "nsb_lotd_bwd_grid", [&](auto Dc, auto Fc) {
        constexpr int D = decltype(Dc)::value, F = decltype(Fc)::value;
        return dispatch_batched(batched, [&](auto Bc) {
            constexpr bool B = decltype(Bc)::value;
            if (dL_dy_is_half) k_lotd_bwd_grid<D, F, true, B><<<grid, 256, 0, s>>>(m, dL_dy, input, n, max_level, b, scale, dL_dparam);
            else k_lotd_bwd_grid<D, F, false, B><<<grid, 256, 0, s>>>(m, dL_dy, input, n, max_level, b, scale, dL_dparam);
            return check_launch("nsb_lotd_bwd_grid");
        });
    });
}

extern "C" int nsb_lotd_bwd_grid(const nsb_lotd_meta *meta, const void *dL_dy, int dL_dy_is_half, const float *input,
                                 int64_t n, int32_t max_level, float scale, float *dL_dparam, void *stream) {
    return nsb_lotd_bwd_grid_batched(meta, dL_dy, dL_dy_is_half, input, n, max_level, nullptr, scale, dL_dparam, stream);
}

// Replaces the input part of lod_hash_only_bwd_impl (lotd_hash_only.h:839-856).  Of the batch only `inds` matters: skipped
// points get zero rows (the reference's come out zero from the zero rows of its dy_dx).
extern "C" int nsb_lotd_bwd_input_batched(const void *dL_dy, int dL_dy_is_half, const float *dy_dx, int64_t n, int32_t n_feat,
                                          int32_t n_dims, const nsb_lotd_batch *batch_host, float scale, float *dL_dx,
                                          void *stream) {
    LotdBatch b;
    bool batched;
    if (make_batch(batch_host, nullptr, n, "LoTDEncoding::bwd", &b, &batched)) return 2;
    if (n == 0) return 0;
    NSB_REQUIRE(dL_dy && dy_dx && dL_dx, "nsb_lotd_bwd_input: NULL argument");
    NSB_REQUIRE(n_dims >= 1 && n_dims <= NSB_MAX_DIMS, "nsb_lotd_bwd_input: n_dims out of range");
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned grid = wave_grid(n, 256, 4);
    return dispatch_batched(batched, [&](auto Bc) {
        constexpr bool B = decltype(Bc)::value;
        if (dL_dy_is_half) k_lotd_bwd_input<true, B><<<grid, 256, 0, s>>>(dL_dy, dy_dx, n, n_feat, n_dims, b, scale, dL_dx);
        else k_lotd_bwd_input<false, B><<<grid, 256, 0, s>>>(dL_dy, dy_dx, n, n_feat, n_dims, b, scale, dL_dx);
        return check_launch("nsb_lotd_bwd_input");
    });
}

extern "C" int nsb_lotd_bwd_input(const void *dL_dy, int dL_dy_is_half, const float *dy_dx, int64_t n, int32_t n_feat,
                                  int32_t n_dims, float scale, float *dL_dx, void *stream) {
    return nsb_lotd_bwd_input_batched(dL_dy, dL_dy_is_half, dy_dx, n, n_feat, n_dims, nullptr, scale, dL_dx, stream);
}

// Replaces lod_bwd_bwd_input_common (lotd_torch_api.cu:575-729) with lod_hash_only_bwd_bwd_input_impl
// (lotd_hash_only.h:951-1056) and its grid kernel (lotd_hash_only.h:472-574), batch arguments included (:507-520).
extern "C" int nsb_lotd_bwd_bwd_input_batched(const nsb_lotd_meta *meta, const float *dL_ddLdx, const void *dL_dy,
                                              int dL_dy_is_half, const float *input, const float *dy_dx, int64_t n,
                                              int32_t max_level, const nsb_lotd_batch *batch_host, float scale,
                                              float *dL_ddLdy, float *dL_dparam, void *stream) {
    NSB_REQUIRE(meta, "nsb_lotd_bwd_bwd_input: NULL meta");
    LotdBatch b;
    bool batched;
    if (make_batch(batch_host, meta, n, "LoTDEncoding::bwd_bwd_input", &b, &batched)) return 2;
    if (n == 0) return 0;
    NSB_REQUIRE(dL_ddLdx, "nsb_lotd_bwd_bwd_input: NULL dL_ddLdx");
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    cudaStream_t s = (cudaStream_t)stream;
    int rc = 0;
    if (dL_ddLdy) {
        NSB_REQUIRE(dy_dx, "LoTDEncoding::bwd_bwd_input: need `dy_dx` to compute `dL_d(dLdy)`.");
        if (max_level <= -1) cudaMemsetAsync(dL_ddLdy, 0, (size_t)n * m.n_out * sizeof(float), s);
        else {
            rc |= dispatch_batched(batched, [&](auto Bc) {
                k_lotd_ddLdy<decltype(Bc)::value><<<wave_grid(n * m.n_out, 256, 4), 256, 0, s>>>(dL_ddLdx, dy_dx, n, m.n_out, m.D, b, dL_ddLdy);
                return check_launch("nsb_lotd_bwd_bwd_input(ddLdy)");
            });
        }
    }
    if (dL_dparam && max_level > -1) {
        NSB_REQUIRE(dL_dy && input, "nsb_lotd_bwd_bwd_input: NULL dL_dy/input");
        const unsigned grid = wave_grid(n * m.n_pseudo, 256, 4);
        rc |= dispatch_DF(meta, "nsb_lotd_bwd_bwd_input", [&](auto Dc, auto Fc) {
            constexpr int D = decltype(Dc)::value, F = decltype(Fc)::value;
            return dispatch_batched(batched, [&](auto Bc) {
                constexpr bool B = decltype(Bc)::value;
                if (dL_dy_is_half)
                    k_lotd_bwd_bwd_grid<D, F, true, B><<<grid, 256, 0, s>>>(m, dL_ddLdx, dL_dy, input, n, max_level, b, scale, dL_dparam);
                else
                    k_lotd_bwd_bwd_grid<D, F, false, B><<<grid, 256, 0, s>>>(m, dL_ddLdx, dL_dy, input, n, max_level, b, scale, dL_dparam);
                return check_launch("nsb_lotd_bwd_bwd_input(grid)");
            });
        });
    }
    return rc;
}

extern "C" int nsb_lotd_bwd_bwd_input(const nsb_lotd_meta *meta, const float *dL_ddLdx, const void *dL_dy,
                                      int dL_dy_is_half, const float *input, const float *dy_dx, int64_t n,
                                      int32_t max_level, float scale, float *dL_ddLdy, float *dL_dparam, void *stream) {
    return nsb_lotd_bwd_bwd_input_batched(meta, dL_ddLdx, dL_dy, dL_dy_is_half, input, dy_dx, n, max_level, nullptr, scale,
                                          dL_ddLdy, dL_dparam, stream);
}
