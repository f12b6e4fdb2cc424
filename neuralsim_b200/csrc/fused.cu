// Fused "forward_sdf" for sm_90a: LoTD gather -> SDF decoder MLP (F -> W -> 1, Softplus(beta)) in one kernel.
//
// Replaces, for no-grad SDF queries, the chain
//   LoTDEncoding.forward (lotd_encoding.py:150-166)  -> 16 gather kernels + transpose
//   MLP.forward under autocast (blocks/mlp.py:104-118, layers.py:302-312) -> 2 cuBLAS GEMMs + softplus + casts
// of the reference (called by LoTDSDF.forward, nr3d_lib/models/fields/sdf/lotd_sdf.py:176-200).
// Numerics contract (DESIGN.md): identical fp16 rounding points as the autocast graph --
//   h   : fp16, accumulated in fp16 over the 8 corners (reference LoTD kernel semantics)
//   z   : fp16( sum_k h_k*W1_jk [fp32] + b1_j )            W1,b1 = fp16(fp32 masters)
//   a   : fp16( softplus_beta(float(z)) )                   softplus evaluated in fp32 (autocast fp32 list)
//   sdf : fp16( sum_j a_j*W2_j [fp32] + b2 )
// The 32x64 layer is evaluated here on CUDA cores with weights staged once per CTA in shared memory
// (fp32, float4 broadcast loads); the tensor-core variant of the same contract lives in fused_tc.cu.
#include "lotd_device.cuh"

namespace nsb {

constexpr int kMaxW = 64;
constexpr int kMaxNF = 32;

struct DecoderDev {
    const __half *W1, *b1, *W2, *b2;
    int width;
    float beta;
};

// gathers the whole feature row of one point (fp16 values widened to fp32 registers)
template <int D, int F>
__device__ __forceinline__ void gather_row(const PLMeta &m, const __half *__restrict__ grid, const float (&xs)[D],
                                           int max_level, float *h) {
    for (uint32_t p = 0; p < m.n_pseudo; ++p) {
        if ((int)m.level[p] > max_level) {
#pragma unroll
            for (int f = 0; f < F; ++f) h[p * F + f] = 0.f;
            continue;
        }
        uint32_t cell[D];
        float fr[D], scale[D];
        level_pos<D>(m, p, xs, cell, fr, scale);
        __half v[1 << D][F];
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) load_corner<D, F, __half>(m, p, grid, cell, c, v[c]);
        __half acc[F];
#pragma unroll
        for (int f = 0; f < F; ++f) acc[f] = __float2half_rn(0.f);
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            const float w = corner_weight<D>(fr, c);
#pragma unroll
            for (int f = 0; f < F; ++f) acc[f] = __hadd(acc[f], __float2half_rn(__fmul_rn(w, __half2float(v[c][f]))));
        }
#pragma unroll
        for (int f = 0; f < F; ++f) h[p * F + f] = __half2float(acc[f]);
    }
}

__device__ __forceinline__ float softplus_beta(float z, float beta) {
    const float zb = z * beta;
    return zb > 20.f ? z : log1pf(expf(zb)) / beta;   // ATen softplus, threshold 20
}

template <int NF>
__device__ __forceinline__ float decode_sdf(const float *h, const float *sW1, const float *sb1, const float *sW2, float b2,
                                            int width, float beta) {
    float out = 0.f;
    for (int j = 0; j < width; ++j) {
        const float4 *w = reinterpret_cast<const float4 *>(sW1 + j * NF);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < NF / 4; ++k) {
            const float4 ww = w[k];
            acc = fmaf(h[4 * k], ww.x, acc);
            acc = fmaf(h[4 * k + 1], ww.y, acc);
            acc = fmaf(h[4 * k + 2], ww.z, acc);
            acc = fmaf(h[4 * k + 3], ww.w, acc);
        }
        const float z = __half2float(__float2half_rn(acc + sb1[j]));
        const float a = __half2float(__float2half_rn(softplus_beta(z, beta)));
        out = fmaf(a, sW2[j], out);
    }
    return __half2float(__float2half_rn(out + b2));
}

template <int D, int F, int NF, bool FROM_RAYS>
__global__ void __launch_bounds__(256)
k_fused_sdf(const PLMeta m, const __half *__restrict__ grid, const DecoderDev dec, const float *__restrict__ x,
            const float *__restrict__ rays_o, const float *__restrict__ rays_d, const int64_t *__restrict__ ridx,
            const float *__restrict__ t, int64_t n, int max_level, float *__restrict__ sdf, __half *__restrict__ h_out) {
    __shared__ __align__(16) float sW1[kMaxW * NF];
    __shared__ float sb1[kMaxW], sW2[kMaxW];
    __shared__ float sb2;
    for (int k = threadIdx.x; k < dec.width * NF; k += blockDim.x) sW1[k] = __half2float(dec.W1[k]);
    for (int k = threadIdx.x; k < dec.width; k += blockDim.x) {
        sb1[k] = __half2float(dec.b1[k]);
        sW2[k] = __half2float(dec.W2[k]);
    }
    if (threadIdx.x == 0) sb2 = __half2float(dec.b2[0]);
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float xs[D];
        if (FROM_RAYS) {
            const int64_t r = ridx ? ridx[i] : i;
            const float tt = t[i];
#pragma unroll
            for (int d = 0; d < D; ++d) xs[d] = __fmaf_rn(rays_d[r * D + d], tt, rays_o[r * D + d]);
        } else {
#pragma unroll
            for (int d = 0; d < D; ++d) xs[d] = x[i * D + d];
        }
        // network space [-1,1] -> table space [0,1] (lotd_encoding.py:165), clamp (lotd.py:60)
#pragma unroll
        for (int d = 0; d < D; ++d) xs[d] = fminf(fmaxf(__fmaf_rn(xs[d], 0.5f, 0.5f), 1.0e-6f), 1.f - 1.0e-6f);
        float h[NF];
        gather_row<D, F>(m, grid, xs, max_level, h);
        if (h_out) {
#pragma unroll
            for (int k = 0; k < NF; ++k) h_out[i * NF + k] = __float2half_rn(h[k]);
        }
        sdf[i] = decode_sdf<NF>(h, sW1, sb1, sW2, sb2, dec.width, dec.beta);
    }
}

}  // namespace nsb

using namespace nsb;
namespace nsb { extern std::atomic<int> g_opt_sdf_simt; }
extern "C" int nsb_fused_sdf_tc_launch(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                                       const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                                       int32_t max_level, float *sdf, void *stream, int mode, const int64_t *pack_infos,
                                       const int64_t *pack_ray, int64_t n_packs, const nsb_occ_collect *collect);

static int launch_fused_sdf(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                            const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                            int32_t max_level, float *sdf, void *h_out, void *stream, bool from_rays) {
    NSB_REQUIRE(meta && dec && sdf, "nsb_fused_sdf: NULL argument");
    if (n == 0) return 0;
    NSB_REQUIRE(params_half && dec->W1 && dec->b1 && dec->W2 && dec->b2, "nsb_fused_sdf: NULL weights");
    NSB_REQUIRE(meta->n_dims_to_encode == 3 && meta->n_feat_per_pseudo_lvl == 2 && meta->n_encoded_dims == 32,
                "nsb_fused_sdf: built for 3-D LoTD with 16 x 2 features (got D=%u F=%u NF=%u)", meta->n_dims_to_encode,
                meta->n_feat_per_pseudo_lvl, meta->n_encoded_dims);
    NSB_REQUIRE(dec->width >= 1 && dec->width <= kMaxW, "nsb_fused_sdf: decoder width %d out of range (<= %d)", dec->width, kMaxW);
    if (!g_opt_sdf_simt.load() && h_out == nullptr && meta->n_pseudo_levels == 16)   // tensor-core kernel (csrc/fused_tc.cu)
        return nsb_fused_sdf_tc_launch(meta, params_half, dec, x, rays_o, rays_d, ridx, t, n, max_level, sdf, stream, from_rays ? 1 : 0, nullptr, nullptr, 0, nullptr);
    PLMeta m;
    if (make_plmeta(meta, &m)) return 2;
    DecoderDev d{(const __half *)dec->W1, (const __half *)dec->b1, (const __half *)dec->W2, (const __half *)dec->b2,
                 dec->width, dec->beta};
    const int ml = max_level < 0 ? -1 : max_level;
    const unsigned grid = wave_grid(n, 256, 3);
    cudaStream_t s = (cudaStream_t)stream;
    if (from_rays)
        k_fused_sdf<3, 2, 32, true><<<grid, 256, 0, s>>>(m, (const __half *)params_half, d, nullptr, rays_o, rays_d, ridx, t, n,
                                                        ml, sdf, (__half *)h_out);
    else
        k_fused_sdf<3, 2, 32, false><<<grid, 256, 0, s>>>(m, (const __half *)params_half, d, x, nullptr, nullptr, nullptr,
                                                         nullptr, n, ml, sdf, (__half *)h_out);
    return check_launch("nsb_fused_sdf");
}

extern "C" int nsb_fused_sdf(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x,
                             int64_t n, int32_t max_level, float *sdf, void *h_out_half, void *stream) {
    NSB_REQUIRE(x || n == 0, "nsb_fused_sdf: NULL x");
    return launch_fused_sdf(meta, params_half, dec, x, nullptr, nullptr, nullptr, nullptr, n, max_level, sdf, h_out_half, stream,
                            false);
}

extern "C" int nsb_fused_sdf_rays(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec,
                                  const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                                  int32_t max_level, float *sdf, void *stream) {
    NSB_REQUIRE((rays_o && rays_d && t) || n == 0, "nsb_fused_sdf_rays: NULL rays");
    return launch_fused_sdf(meta, params_half, dec, nullptr, rays_o, rays_d, ridx, t, n, max_level, sdf, nullptr, stream, true);
}

extern "C" int nsb_fused_sdf_packs(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *rays_o,
                                   const float *rays_d, const int64_t *pack_infos, const int64_t *pack_ray, int64_t n_packs, const float *t,
                                   int32_t max_level, float *sdf, void *stream) {
    NSB_REQUIRE(meta && dec && (sdf || n_packs == 0), "nsb_fused_sdf_packs: NULL argument");
    if (n_packs == 0) return 0;
    NSB_REQUIRE(rays_o && rays_d && pack_infos && t && params_half && dec->W1 && dec->b1 && dec->W2 && dec->b2, "nsb_fused_sdf_packs: NULL argument");
    NSB_REQUIRE(meta->n_dims_to_encode == 3 && meta->n_feat_per_pseudo_lvl == 2 && meta->n_encoded_dims == 32 && meta->n_pseudo_levels == 16,
                "nsb_fused_sdf_packs: built for 3-D LoTD with 16 x 2 features");
    NSB_REQUIRE(dec->width >= 1 && dec->width <= kMaxW, "nsb_fused_sdf_packs: decoder width %d out of range (<= %d)", dec->width, kMaxW);
    return nsb_fused_sdf_tc_launch(meta, params_half, dec, nullptr, rays_o, rays_d, nullptr, t, 0, max_level, sdf, stream, 2, pack_infos, pack_ray, n_packs, nullptr);
}

extern "C" int nsb_fused_sdf_collect(const nsb_lotd_meta *meta, const void *params_half, const nsb_sdf_decoder *dec, const float *x, const float *rays_o,
                                     const float *rays_d, const int64_t *ridx, const float *t, int64_t n, const int64_t *pack_infos,
                                     const int64_t *pack_ray, int64_t n_packs, int32_t mode, int32_t max_level, float *sdf,
                                     const nsb_occ_collect *collect, void *stream) {
    NSB_REQUIRE(meta && dec && params_half && dec->W1 && dec->b1 && dec->W2 && dec->b2, "nsb_fused_sdf_collect: NULL argument");
    NSB_REQUIRE(mode >= 0 && mode <= 2, "nsb_fused_sdf_collect: mode must be 0 (points), 1 (rays) or 2 (packs)");
    if ((mode == 2 && n_packs == 0) || (mode != 2 && n == 0)) return 0;
    NSB_REQUIRE(sdf && (mode == 0 ? x != nullptr : (rays_o && rays_d && t)) && (mode != 2 || pack_infos), "nsb_fused_sdf_collect: NULL argument");
    NSB_REQUIRE(meta->n_dims_to_encode == 3 && meta->n_feat_per_pseudo_lvl == 2 && meta->n_encoded_dims == 32 && meta->n_pseudo_levels == 16,
                "nsb_fused_sdf_collect: built for 3-D LoTD with 16 x 2 features");
    NSB_REQUIRE(dec->width >= 1 && dec->width <= kMaxW, "nsb_fused_sdf_collect: decoder width %d out of range (<= %d)", dec->width, kMaxW);
    NSB_REQUIRE(!collect || !collect->grid_pcl || (collect->res[0] > 0 && collect->res[1] > 0 && collect->res[2] > 0), "nsb_fused_sdf_collect: bad grid resolution");
    return nsb_fused_sdf_tc_launch(meta, params_half, dec, x, rays_o, rays_d, ridx, t, n, max_level, sdf, stream, mode, pack_infos, pack_ray, n_packs, collect);
}
