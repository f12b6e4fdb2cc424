/* neuralsim_b200 -- C ABI of the H100-native (sm_90a) NeuS volume-rendering hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b): every entry point is what the reference's own
 * native extensions (`nr3d_lib.bindings._lotd / _pack_ops / _occ_grid / _shencoder`, built by
 * nr3d_lib/setup.py:134,184,239,516) expose to Python, restated as plain C: raw *device*
 * pointers + sizes + a stream, no torch / ATen types.  The pybind11 / ctypes shim a maintainer would put on
 * top is shown in INTEGRATION.md; `neuralsim_b200/bindings/*.py` is that shim over ctypes.
 *
 * Conventions
 *   - all pointers are device pointers unless the name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - every function returns 0 on success, non-zero on failure; nsb_last_error() gives the message
 *     (thread-local), mirroring the C++ exceptions -> RuntimeError behaviour of the reference;
 *   - pack_infos is int64 [P,2] = (first, length), exactly the reference's layout
 *     (csrc/pack_ops/pack_ops.h:11-65); packed_info of the marcher is int32 [R,2];
 *   - fp16 tensors are IEEE binary16 (`__half`), passed as void* / uint16_t*.
 */
#ifndef NEURALSIM_B200_H
#define NEURALSIM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NSB_MAX_LEVELS 32
#define NSB_MAX_DIMS 4

/* lotd::LoDType values used on the path (csrc/lotd/include/lotd/lotd_types.h:16-26). */
#define NSB_LOD_DENSE 0
#define NSB_LOD_HASH 7

/* Plain-C image of lotd::torch::LoDMeta (csrc/lotd/include/lotd/lotd_torch_api.h:143-200) restricted to
 * Dense/Hash levels with linear interpolation -- the `c_hash_only` fast path of the reference. */
typedef struct nsb_lotd_meta {
    uint32_t n_dims_to_encode;
    uint32_t n_levels;
    uint32_t n_pseudo_levels;
    uint32_t n_feat_per_pseudo_lvl;
    uint32_t n_encoded_dims;
    uint32_t n_params;
    uint32_t level_res[NSB_MAX_LEVELS][NSB_MAX_DIMS];
    uint32_t level_n_feats[NSB_MAX_LEVELS];
    uint32_t level_types[NSB_MAX_LEVELS];
    uint32_t level_sizes[NSB_MAX_LEVELS];
    uint32_t level_offsets[NSB_MAX_LEVELS + 1];
    uint32_t map_levels[NSB_MAX_LEVELS * 4];
    uint32_t map_cnt[NSB_MAX_LEVELS * 4];
} nsb_lotd_meta;

const char *nsb_last_error(void);
int nsb_version(void);
/* Number of kernels this library has launched in the calling process (bench.py's `gpu_launches`). */
uint64_t nsb_launch_count(void);
/* Self-check switch: key "sdf_simt" (0|1) routes nsb_fused_sdf* through the CUDA-core cross-check kernel.  Any other key is an error. */
int nsb_set_option(const char *key, int value);

/* ------------------------------------------------------------------------------------------------
 * _lotd  (csrc/lotd/src/lotd.cpp:22-107)
 * ---------------------------------------------------------------------------------------------- */
/* LoDMeta(n_input_dims, lod_res_multidim, lod_n_feats, lod_types, hashmap_size)   lotd_torch_api.cu:29-230
 * lod_res_host: [n_levels * n_dims]; lod_types_host: NSB_LOD_* per level.  Host-only, no device work. */
int nsb_lotd_meta_create(int32_t n_dims, int32_t n_levels, const int32_t *lod_res_host,
                         const int32_t *lod_n_feats_host, const int32_t *lod_types_host,
                         uint32_t hashmap_size, nsb_lotd_meta *out_host);

/* lod_fwd(meta, input[N,D] f32 in [0,1], params f16|f32, max_level, need_input_grad)
 *   -> y[N,F] (params dtype, row-major), dy_dx[N,F,D] f32 or NULL            lotd_torch_api.cu:232-365
 * `input` must already be clamped to [1e-6, 1-1e-6] (the reference clamps in lotd.py:60). */
int nsb_lotd_fwd(const nsb_lotd_meta *meta_host, const float *input, const void *params, int params_is_half,
                 int64_t n, int32_t max_level, void *y, float *dy_dx, void *stream);

/* lod_bwd, parameter part: dL_dparam[P] (fp32, accumulated -- caller zero-fills) += scatter(dL_dy * w)
 *                                                                           lotd_hash_only.h:380-470
 * dL_dy is [N,F] in the params dtype.  `scale` multiplies every contribution (the reference's
 * 1/loss_scale, lotd.py:105). */
int nsb_lotd_bwd_grid(const nsb_lotd_meta *meta_host, const void *dL_dy, int dL_dy_is_half, const float *input,
                      int64_t n, int32_t max_level, float scale, float *dL_dparam, void *stream);

/* lod_bwd, input part: dL_dx[N,D] = sum_f float(dL_dy[N,f]) * dy_dx[N,f,D]     lotd_hash_only.h:839-856 */
int nsb_lotd_bwd_input(const void *dL_dy, int dL_dy_is_half, const float *dy_dx, int64_t n, int32_t n_feat,
                       int32_t n_dims, float scale, float *dL_dx, void *stream);

/* lod_bwd_bwd_input                                                         lotd_hash_only.h:951-1056
 *   dL_ddLdy[N,F] f32 (may be NULL) = sum_d dL_ddLdx[N,d] * dy_dx[N,f,d]
 *   dL_dparam[P] f32 (may be NULL, accumulated) += 2nd-order scatter of dL_ddLdx (x) dL_dy
 * dy_dx may be NULL when dL_ddLdy is NULL. */
int nsb_lotd_bwd_bwd_input(const nsb_lotd_meta *meta_host, const float *dL_ddLdx, const void *dL_dy,
                           int dL_dy_is_half, const float *input, const float *dy_dx, int64_t n,
                           int32_t max_level, float scale, float *dL_ddLdy, float *dL_dparam, void *stream);

/* Batched tables (lotd_hash_only.h:44-55, lotd_torch_api.cu:263-290): `params` holds several tables of n_params elements.
 * Point i reads the table of batch b = inds[i] if inds is set (a negative inds[i] skips the point: zero y / dy_dx / dL_dx /
 * dL_ddLdy rows, no table gradient), else b = i / data_size if data_size is non-zero, else b = 0.  The table starts at element
 * offsets[b] if offsets is set, else at b * n_params; the start is formed in 64 bits.  Batches may share a table: their
 * gradients add up.  Offsets must be even (feature pairs are read and reduced as one access); index and offset values are not
 * range-checked here (bindings/_lotd.py checks them).  A NULL batch, or one with all three fields empty, is the unbatched
 * call; a non-zero data_size must divide n. */
typedef struct nsb_lotd_batch {
    const int64_t *inds;        /* [N] int64, or NULL */
    const int64_t *offsets;     /* [B] int64 element offsets, or NULL */
    uint32_t data_size;         /* points per batch (consecutive), or 0 */
} nsb_lotd_batch;

/* The four entries above with a batch argument (batch_host: host pointer, may be NULL); the entries above are these with
 * batch_host = NULL.  For nsb_lotd_bwd_input_batched only `inds` matters (it has no table). */
int nsb_lotd_fwd_batched(const nsb_lotd_meta *meta_host, const float *input, const void *params, int params_is_half,
                         int64_t n, int32_t max_level, const nsb_lotd_batch *batch_host, void *y, float *dy_dx, void *stream);
int nsb_lotd_bwd_grid_batched(const nsb_lotd_meta *meta_host, const void *dL_dy, int dL_dy_is_half, const float *input,
                              int64_t n, int32_t max_level, const nsb_lotd_batch *batch_host, float scale, float *dL_dparam,
                              void *stream);
int nsb_lotd_bwd_input_batched(const void *dL_dy, int dL_dy_is_half, const float *dy_dx, int64_t n, int32_t n_feat,
                               int32_t n_dims, const nsb_lotd_batch *batch_host, float scale, float *dL_dx, void *stream);
int nsb_lotd_bwd_bwd_input_batched(const nsb_lotd_meta *meta_host, const float *dL_ddLdx, const void *dL_dy,
                                   int dL_dy_is_half, const float *input, const float *dy_dx, int64_t n, int32_t max_level,
                                   const nsb_lotd_batch *batch_host, float scale, float *dL_ddLdy, float *dL_dparam,
                                   void *stream);

/* ------------------------------------------------------------------------------------------------
 * _occ_grid  (csrc/occ_grid/src/occ_grid.cpp:21-33, include/occ_grid/cpp_api.h:14-65)
 * ray_marching / batched_ray_marching, AABB contraction.  Two calls, as the reference's two kernel
 * rounds (ray_marching.cu:179-241): first with packed_info == NULL to fill num_steps[R]; the caller
 * builds packed_info = (exclusive cumsum, num_steps) and calls again to fill the sample arrays.
 * batch_inds == NULL -> single grid bool[rx,ry,rz], roi[6]; else grid bool[B,rx,ry,rz], roi[B,6].
 * ---------------------------------------------------------------------------------------------- */
int nsb_ray_marching(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min,
                     const float *t_max, const float *roi, const int32_t *batch_inds, int32_t rx, int32_t ry,
                     int32_t rz, const uint8_t *grid_binary, float step_size, float max_step_size,
                     float dt_gamma, uint32_t max_steps, const int32_t *packed_info, int32_t *num_steps,
                     float *t_starts, float *t_ends, int32_t *ridx, int32_t *gidx, int32_t *bidx, void *stream);
/* The same with the second round restricted to the rays ray_list[0..n_list) (those whose first-round count is non-zero: on an
 * image ~10 % of the rays); ray_list == NULL marches all n_rays.  t_ends / gidx / bidx may be NULL in the second round.
 * grid_bits: NULL or nsb_pack_occ_bits(grid_binary). */
int nsb_ray_marching_listed(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min, const float *t_max,
                            const float *roi, const int32_t *batch_inds, int32_t rx, int32_t ry, int32_t rz,
                            const uint8_t *grid_binary, float step_size, float max_step_size, float dt_gamma, uint32_t max_steps,
                            const int32_t *packed_info, int32_t *num_steps, float *t_starts, float *t_ends, int32_t *ridx,
                            int32_t *gidx, int32_t *bidx, const int64_t *ray_list, int64_t n_list, const uint32_t *grid_bits, void *stream);
/* Small batches (the time of a march is the latency of its longest ray, and the reference pays it twice, ray_marching.cu:179-241): the
 * first round of the single-grid march that ALSO records sample k of ray i at rec_t[i * max_steps + k] (t_start), and the copy that
 * replaces the second round: for the listed rays j < n_list (ray_list == NULL: every ray), i = ray_list[j],
 * (first, n) = packed_info[i]: t_starts[first + k] = rec_t[i * max_steps + k], ridx[first + k] = i.  Same values as the two-round
 * march bit for bit (the same arithmetic, run once).  Both count-aware (nsb_bind_device_counts: the rays / the listed rays). */
int nsb_ray_marching_record(int64_t n_rays, const float *rays_o, const float *rays_d, const float *t_min, const float *t_max,
                            const float *roi, int32_t rx, int32_t ry, int32_t rz, const uint8_t *grid_binary, float step_size,
                            float max_step_size, float dt_gamma, uint32_t max_steps, int32_t *num_steps, float *rec_t,
                            const uint32_t *grid_bits, void *stream);
int nsb_march_compact(const float *rec_t, uint32_t max_steps, const int32_t *packed_info, const int64_t *ray_list, int64_t n_list,
                      float *t_starts, int32_t *ridx, void *stream);
/* words[(cells + 31) / 32]: the bool grid packed 32 cells per word (bit k of word w = cell 32 w + k).  Passing it as `grid_bits`
 * (single-grid marching only) saves every CTA the re-packing of the 64^3 grid into shared memory. */
int nsb_pack_occ_bits(const uint8_t *grid_binary, int64_t cells, uint32_t *words, void *stream);

/* ------------------------------------------------------------------------------------------------
 * _pack_ops  (csrc/pack_ops/pack_ops.cpp:20-58, pack_ops.h:11-65).  fp32 features unless noted.
 * ---------------------------------------------------------------------------------------------- */
enum { NSB_OP_ADD = 0, NSB_OP_SUB, NSB_OP_MUL, NSB_OP_DIV, NSB_OP_GT, NSB_OP_GEQ, NSB_OP_LT, NSB_OP_LEQ,
       NSB_OP_EQ, NSB_OP_NEQ };
/* packed_{add,sub,mul,div}: out[i,c] = feats[i,c] (op) other[pack(i),c]; compare ops write uint8. */
int nsb_packed_binary(int op, const float *feats, const float *other, const int64_t *pack_infos, int64_t n_packs,
                      int32_t feat_dim, void *out, void *stream);
int nsb_packed_sum(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim, float *out,
                   void *stream);
int nsb_packed_cumsum(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim,
                      int exclusive, int reverse, float *out, void *stream);
/* packed_diff / packed_backward_diff with optional per-pack appends|last_fill / prepends|first_fill. */
int nsb_packed_diff(const float *feats, const int64_t *pack_infos, int64_t n_packs, int32_t feat_dim,
                    const float *appends, const float *last_fill, int backward, float *out, void *stream);
int nsb_packed_searchsorted(const float *bins, const float *vals, const int64_t *pack_infos, int64_t n_packs,
                            int32_t n_vals, int64_t *out_idx, void *stream);
int nsb_packed_invert_cdf(const float *bins, const float *cdfs, const float *u, const int64_t *pack_infos,
                          int64_t n_packs, int32_t n_samples, float *samples, int64_t *bin_idx, void *stream);
/* try_merge_two_packs_sorted_aligned: pack_infos_out [P,2] must hold (first,len) of the merged packs. */
int nsb_merge_two_packs_sorted_aligned(const float *vals_a, const int64_t *pack_infos_a, const float *vals_b,
                                       const int64_t *pack_infos_b, const int64_t *pack_infos_out,
                                       int64_t n_packs, int b_sorted, int64_t *pidx_a, int64_t *pidx_b,
                                       void *stream);
/* packed_alpha_to_vw_forward: weights (may be NULL), num_steps int64[P] + selector uint8[S] (may be NULL). */
int nsb_packed_alpha_to_vw_forward(const float *alphas, const int64_t *pack_infos, int64_t n_packs,
                                   float early_stop_eps, float alpha_thre, float *weights, int64_t *num_steps,
                                   uint8_t *selector, void *stream);
int nsb_packed_alpha_to_vw_backward(const float *weights, const float *grad_weights, const float *alphas,
                                    const int64_t *pack_infos, int64_t n_packs, float early_stop_eps,
                                    float alpha_thre, float *grad_alphas, void *stream);
/* interleave_arange / interleave_linstep: cumsum_steps is the inclusive cumsum of num_steps (int64[P]). */
int nsb_interleave_linstep(const float *start, const int64_t *num_steps, const int64_t *cumsum_steps,
                           const float *step_size, float step_scalar, int64_t n_packs, float *out, int64_t *nidx,
                           void *stream);
int nsb_interleave_arange(const int64_t *num_steps, const int64_t *cumsum_steps, int64_t n_packs, int64_t *out,
                          int64_t *nidx, void *stream);
/* packed_sort_qsort: ascending per pack (stable, NaN last), in place on vals [n_vals]; the last pack must end at n_vals.
 * idx (may be NULL) receives the global gather indices of the packed elements; elements between packs are not touched. */
int nsb_packed_sort(float *vals, int64_t n_vals, const int64_t *pack_infos, int64_t n_packs, int64_t *idx, void *stream);
int nsb_mark_pack_boundaries(const int64_t *ids, int64_t n, int32_t *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * _shencoder  (externals/shencoder/bindings.cpp, shencoder.h): real SH basis, degree C in [1,4].
 * ---------------------------------------------------------------------------------------------- */
int nsb_sh_encode_forward(const float *inputs, float *outputs, int64_t n, int32_t degree, float *dy_dx,
                          void *stream);
int nsb_sh_encode_backward(const float *grad, const float *dy_dx, int64_t n, int32_t degree, float *grad_inputs,
                           void *stream);

/* ------------------------------------------------------------------------------------------------
 * Fused entry points (the coarser L2->L1 boundary of SURVEY.md §8b "Fused boundary we add").
 * They replace chains of the calls above + the autocast MLPs of nr3d_lib/models/blocks/mlp.py with one
 * kernel each; numerics follow the same fp16 rounding points (see DESIGN.md "Numerics contract").
 * ---------------------------------------------------------------------------------------------- */
typedef struct nsb_sdf_decoder {       /* LoTDSDF decoder F->W->1, Softplus(beta)  (lotd_sdf.py:176-200), F = n_encoded_dims */
    const void *W1;                    /* fp16 [W, F]   (fp32 master rounded by the caller; row stride F) */
    const void *b1;                    /* fp16 [W] */
    const void *W2;                    /* fp16 [W] */
    const void *b2;                    /* fp16 [1] */
    int32_t width;                     /* W (<= 64, multiple of 16) */
    float beta;                        /* 100 */
} nsb_sdf_decoder;

/* Optional side effect of every training-time SDF query: `accel.collect_samples(x, sdf)` (renderer_mixin.py:154-164 ->
 * OccGridEma._collect_samples, ema_single.py:201-203 -> update_occ_val_grid_(grid_pcl, pts, occ_val_fn(sdf), ema_decay = 1), utils.py:93-109):
 * grid_pcl[voxel(x)] = max(grid_pcl[voxel(x)], (1 / cosh(clamp(inv_s sdf / 2, -20, 20)))^2), evaluated in fp16 like the reference
 * (its sdf is a half tensor), accumulated with an atomic max inside the query kernel.  Pass NULL to disable. */
typedef struct nsb_occ_collect {
    float *grid_pcl;                   /* fp32 [res0, res1, res2], values >= 0 */
    int32_t res[3];
    float inv_s;
} nsb_occ_collect;

/* The tensor-core SDF, colour and up-sampling entry points below take 3-D LoTD tables of L = 1..24 pseudo levels with
 * n_feat_per_pseudo_lvl == 2 and n_encoded_dims == 2L; the decoder's W1 is then [W x 2L].  Tables of 1..16 levels run kernels with a
 * 32-column feature tile, tables of 17..24 levels the same kernels with a 48-column one (chosen from L, not from max_level).  Tables of
 * more than 24 levels are refused (the error names the limit) and run on the unfused LoTD entry points.  h_out of nsb_fused_sdf and its
 * SIMT kernel need 16 levels. */
/* forward_sdf on N points: x in network space [-1,1]^3 (not yet /2+0.5).  sdf fp32 (fp16-valued). */
int nsb_fused_sdf(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host,
                  const float *x, int64_t n, int32_t max_level, float *sdf, void *h_out_half, void *stream);
/* the three queries below with the occupancy-evidence side effect (collect may be NULL = the plain query) */
int nsb_fused_sdf_collect(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *x,
                          const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                          const int64_t *pack_infos, const int64_t *pack_ray, const int64_t *pack_order, int64_t n_packs, int32_t mode,
                          int32_t max_level, float *sdf, const nsb_occ_collect *collect, void *stream);
/* mode 2 (packs) walks the packs in groups of 32: pack_order[32 g .. 32 g + 32) (a permutation of the live packs, nsb_ray_block_order)
 * or, with pack_order == NULL, packs 32 g .. 32 g + 32.  The order changes which samples share a gather instruction, not any value. */

/* x = o[ridx] + d[ridx] * t, then forward_sdf.  ridx int64[N] indexes rays_o / rays_d [R,3]. */
int nsb_fused_sdf_rays(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host,
                       const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                       int32_t max_level, float *sdf, void *stream);

/* The same query for PACKED samples of coherent rays (an image): pack p = samples t[first_p .. first_p + n_p) of ray pack_ray[p]
 * (NULL = p), pack_infos int64 [n_packs,2] = (first, n).  Traversal is ray-tiled (32 rays x 4 samples per tile) so that the lanes of
 * a gather instruction sit in neighbouring cells; sdf is written to the packed slots -- results identical to nsb_fused_sdf_rays. */
int nsb_fused_sdf_packs(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *rays_o,
                        const float *rays_d, const int64_t *pack_infos, const int64_t *pack_ray, int64_t n_packs, const float *t,
                        int32_t max_level, float *sdf, void *stream);

/* Backward of nsb_fused_sdf / nsb_fused_sdf_rays wrt. the table and the decoder weights (nothing is saved by the
 * forward: features and pre-activations are recomputed).  Pass x != NULL, or x == NULL with (rays_o, rays_d, ridx, t).
 * All outputs are fp32 and ACCUMULATED into (caller zero-fills): d_grid[P], d_W1[W*F], d_b1[W], d_W2[W], d_b2[1].
 * Replaces the autograd chain LoTDFunction.backward (lotd.py:83-119) + the autocast MLP backward. */
int nsb_fused_sdf_bwd(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host,
                      const float *x, const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t,
                      const float *d_sdf, int64_t n, int32_t max_level, float *d_grid, float *d_W1, float *d_b1,
                      float *d_W2, float *d_b2, void *stream);

/* the same with an index list: row i of the launch is sample keep[i] of (ridx, t, d_sdf) / (x, d_sdf) -- the compaction of the samples
 * with a non-zero cotangent (most boundary samples of a NeuS ray carry none) without a gather of the operands.  keep == NULL: identity. */
int nsb_fused_sdf_bwd_indexed(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host,
                              const float *x, const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t,
                              const float *d_sdf, const int64_t *keep, int64_t n, int32_t max_level, float *d_grid, float *d_W1,
                              float *d_b1, float *d_W2, float *d_b2, void *stream);

/* nsb_fused_sdf_bwd_indexed on samples of rays, plus the gradient to the rays.  The depths t are constants (the reference computes them
 * without grad) and the encoding's input gradient is first order (its input Hessian is not formed on the reference's hot path), so
 * sample x = o + d t gets g_x = (1/2) sum over levels of J^T dL/dh (at the point the table clamps x / 2 + 1/2 to, unmasked), and
 *   d_rays_o[ray_map[r]] += sum over the samples s of ray r of g_x(s),   d_rays_d[ray_map[r]] += sum of t_s g_x(s)
 * (ray_map NULL: row r; a NULL output is not written).  gx_scratch[n, 8] fp32 workspace (one row per launch row).  The samples of a ray must
 * be consecutive (packed samples) for the sums to be deterministic: each ray's samples are summed by one warp in a fixed order and added
 * once onto the caller's zeros.  Rays without a sample are not written; with device counts, neither are rows or rays past the count.
 * Table and decoder gradients: the same bits as nsb_fused_sdf_bwd_indexed. */
int nsb_fused_sdf_bwd_rays(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *rays_o,
                           const float *rays_d, const int64_t *ridx, const float *t, const float *d_sdf, const int64_t *keep, int64_t n,
                           int32_t max_level, float *d_grid, float *d_W1, float *d_b1, float *d_W2, float *d_b2, float *gx_scratch,
                           const int64_t *ray_map, float *d_rays_o, float *d_rays_d, void *stream);

/* ---------------------------------------------------------------- device-resident sizes (a step without host reads)
 * The reference reads every data-dependent size back to the host (`.item()`, `nonzero()`: ~25 syncs per ray_query, SURVEY.md §8a a9).
 * Here a size may stay in device memory: nsb_bind_device_counts(c0, c1) binds one or two device int64 to the calling thread; the NEXT
 * count-aware entry point of that thread consumes (and clears) the binding and its kernel processes min(n_arg, *c0) items -- n_arg
 * (the `n` / `n_packs` / `n_rays` / `n_list` argument) then is the CAPACITY the buffers and the grid were sized for.  c1 is the second
 * count of nsb_assemble_boundary (n_hit).  Count-aware: nsb_gather_rays / _backward, nsb_ray_marching_listed (first round: num_steps of the rays
 * in [*c0, n_rays) is written as 0; second round: the listed rays), nsb_ray_marching_record / nsb_march_compact (the same), nsb_fused_sdf_collect / _rays / _packs, nsb_ray_block_order, nsb_fused_sdf_bwd(_indexed),
 * nsb_neus_upsample_cdf, nsb_packed_invert_cdf_shared_u, nsb_merge_sorted_vals, nsb_assemble_boundary, nsb_neus_alpha_forward
 * (num_steps of the packs in [*c0, n_packs) is written as 0) / _backward / _backward_kept / _backward_kept_list, nsb_compact_samples, nsb_scatter_f32, nsb_flag_nonzero,
 * nsb_fused_color_fwd / _bwd, nsb_composite_forward / _backward, nsb_lidar_los_rows / _loss_reduce / _los_backward.  With every size on the device a whole fwd+bwd step has no host
 * read and can be captured in a CUDA graph (neuralsim_b200/graphics/neus_static.py). */
int nsb_bind_device_counts(const int64_t *count0, const int64_t *count1);
/* The LoTD level bound in device memory, for a step whose level changes between graph replays (the hard-mask level schedule of an
 * annealed encoding): nsb_bind_device_max_level(level) binds one device int32 to the calling thread; the NEXT level-aware entry point of
 * that thread consumes (and clears) the binding, and its kernels read *level (clamped to [-1, L-1]) instead of the max_level argument.
 * Level-aware: the tensor-core SDF query (nsb_fused_sdf_collect in all modes, nsb_fused_sdf_packs, and nsb_fused_sdf / _rays unless they
 * run the CUDA-core kernel: h_out or the "sdf_simt" option), nsb_fused_sdf_bwd / _bwd_indexed / _bwd_rays, nsb_fused_color_fwd,
 * nsb_fused_color_bwd / _bwd_appear / _bwd_grads, nsb_upsample_rays / nsb_upsample_persistent.  NULL: the max_level argument (the default). */
int nsb_bind_device_max_level(const int32_t *level);
/* flag[i] = (v[i] != 0) for i < live count, 0 up to n (count-aware). */
int nsb_flag_nonzero(const float *v, int64_t n, int32_t *flag, void *stream);
/* Derived sizes of one NeuS query in a device block `counts` of >= 32 int64 (zero-filled once per query):
 *   written by nsb_ray_test_aabb: [2] coherent neighbour pairs, [27] image row length (-1: none found)
 *   written by nsb_scan_counts (totals = counts + 0 / + 3 / + 6 / + 9):
 *     [0] rays that pass the box test  [3] M marched samples  [4] n_hit rays with samples
 *     [6] K samples kept by the compression  [7] rays that keep samples   [9] samples with a non-zero cotangent (backward)
 *   written here, phase 0 (after the march scan):  [12] M and [13] n_hit (both 0 if the arena `march_cap` cannot hold the merged
 *     samples -- then bit 0 of [20] is set), [14+q] n_hit * n_fine[q], [22+q] samples in the merged buffer after stage q,
 *     [18] S = n_rays n_coarse + n_hit sum(n_fine)
 *   phase 1 (after the scan of the kept counts): [19] K and [21] rays that keep samples (0 and bit 1 of [20] if K > kept_cap),
 *     [26] = [0] if K fits, else 0 (the count nsb_compact_samples is bound to). */
int nsb_query_counts(int64_t *counts, int32_t phase, int32_t n_coarse, const int32_t *n_fine_host, int32_t n_stage, int64_t march_cap,
                     int64_t kept_cap, void *stream);

/* ---------------------------------------------------------------- fused per-ray NeuS stages (csrc/neus_fused.cu)
 * One warp per ray (pack).  Each entry point replaces a chain of the reference's Python-level calls with one launch;
 * the pack_ops entry points above remain the drop-in for `_pack_ops` itself.
 *
 * nsb_neus_upsample_cdf: cdf[S] = packed_div(packed_cumsum(packed_alpha_to_vw(alpha), exclusive), max(last, 1e-5)) with
 *   alpha = neus_packed_sdf_to_alpha(sdf, inv_s) or, if use_estimate_alpha, neus_packed_sdf_to_upsample_alpha(sdf, depth, inv_s)
 *   (nr3d_lib/graphics/neus/neus_ray_query.py:873-884, neus_utils.py:88-111,164-188). */
int nsb_neus_upsample_cdf(const float *sdf, const float *depth, const int64_t *pack_infos, int64_t n_packs, float inv_s,
                          int use_estimate_alpha, float early_stop_eps, float alpha_thre, float *cdf, void *stream);
/* packed_invert_cdf (pack_ops_cuda.cu:1634-1682) with ONE u[n_samples] row shared by every pack -> samples[n_packs, n_samples]
 * (what packed_sample_cdf(perturb=False) feeds it, graphics/raysample.py:38-61).  An empty pack's samples are NaN (bins / cdfs are
 * not read for it; the reference's kernel reads bins[first], one past the pack). */
int nsb_packed_invert_cdf_shared_u(const float *bins, const float *cdfs, const float *u, const int64_t *pack_infos, int64_t n_packs,
                                   int32_t n_samples, float *samples, void *stream);
/* alpha[S] = neus_packed_sdf_to_alpha(sdf, *inv_s_dev) and, in the same pass, the compression selector / kept-count per pack
 * of packed_volume_render_compression (pack_ops.py:286-291).  inv_s is read from device memory (no host sync). */
int nsb_neus_alpha_forward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, float early_stop_eps,
                           float alpha_thre, float *alpha, uint8_t *selector, int32_t *num_steps, void *stream);
/* adjoint of the above: d_sdf[S] (written), d_inv_s[1] (accumulated; caller zero-fills). */
int nsb_neus_alpha_backward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, const float *d_alpha,
                            float *d_sdf, float *d_inv_s, void *stream);
/* The same adjoint over the kept samples only, for a d_alpha that is zero outside them (the cotangent of the compression's gather).
 * Inputs are nsb_scan_counts' outputs over the kept counts: nidx[j] = the pack of the j-th ray that keeps samples, pack_infos_kept[j] =
 * its range in kept order, pidx[K] = the sample index of every kept sample, d_alpha[K] in kept order.  Pass 1 writes d_sdf[S] ONLY at
 * the samples next to a kept interval with a non-zero cotangent (nothing else of d_sdf is touched), counts[j] = the non-zero d_sdf of
 * ray j (0 for j in [live, n_packs)), and accumulates d_inv_s[1].  d_sdf equals nsb_neus_alpha_backward's bit for bit.  Pass 2, after
 * offsets = exclusive scan of counts: list[offsets[j] + ..] = the sample indices with non-zero d_sdf, ascending (= flag(d_sdf != 0) +
 * scan over all S samples), and ray[i] = the pack of every listed sample i.  Both count-aware (the rays that keep samples). */
int nsb_neus_alpha_backward_kept(const float *sdf, const int64_t *pack_infos, const int64_t *nidx, const int64_t *pack_infos_kept,
                                 const int64_t *pidx, int64_t n_packs, const float *inv_s_dev, const float *d_alpha, float *d_sdf,
                                 int32_t *counts, float *d_inv_s, void *stream);
int nsb_neus_alpha_backward_kept_list(const int64_t *pack_infos, const int64_t *nidx, const int64_t *pack_infos_kept, const int64_t *pidx,
                                      const float *d_alpha, const float *d_sdf, const int32_t *offsets, int64_t n_packs, int64_t *list,
                                      int64_t *ray, void *stream);
/* Volume integration of one packed buffer (app/renderers/single_volume_renderer.py:73-102): vw = alpha_to_vw(alpha);
 * mask = sum vw; depth = sum vw t / (mask + 1e-10) (or sum vw t); rgb_out = sum vw rgb; nablas_out = sum vw nablas.
 * rgb / nablas ([K,3]) may be NULL.  ray_index[n_packs] (or NULL = identity): the per-ray outputs of pack p are written at
 * slot ray_index[p] of mask / depth / rgb_out / nablas_out (the scatter `rendered[k][rays_inds_hit] = ...` of the renderer). */
int nsb_composite_forward(const float *alpha, const float *t, const float *rgb, const float *nablas, const int64_t *pack_infos,
                          int64_t n_packs, float early_stop_eps, float alpha_thre, int normalize_depth, const int64_t *ray_index,
                          float *vw, float *mask, float *depth, float *rgb_out, float *nablas_out, void *stream);
/* its adjoint; any of g_* may be NULL (= zero cotangent); writes d_alpha[K], d_rgb[K,3], d_nablas[K,3]. */
int nsb_composite_backward(const float *alpha, const float *t, const float *rgb, const float *nablas, const float *vw,
                           const int64_t *pack_infos, int64_t n_packs, float early_stop_eps, float alpha_thre, int normalize_depth,
                           const float *mask, const float *depth, const float *g_mask, const float *g_depth, const float *g_rgb,
                           const float *g_nablas, const float *g_vw, const int64_t *ray_index, float *d_alpha, float *d_rgb,
                           float *d_nablas, void *stream);

/* ---------------------------------------------------------------- glue of the per-ray query (csrc/neus_glue.cu)
 * nsb_scan_counts: one launch for cumsum + nonzero + stack of the reference's wrappers (occgrid_raymarch.py:60-75,
 *   pack_ops.py:286-291): first[n] = exclusive prefix sum of counts; info2[n,2] = (first, count) int32 (`packed_info`);
 *   for the non-zero entries in order: nz_index[j] = i, nz_pack[j] = (first_i, count_i), nz_src[j] = src[i];
 *   totals[2] = (sum of counts, number of non-zero entries), on the device.  Outputs other than totals may be NULL.
 *   first / info2 are int32 and valid only while the sum of counts is below 2^31; totals and nz_pack are int64 and always exact.
 *   workspace_zeroed: nsb_scan_workspace_bytes() of device memory, zero-filled before every call.
 *   Host hand-off without a driver call: `totals` may point to mapped pinned host memory of >= 4 int64; with ticket != 0 the kernel
 *   writes totals[2] = *extra_src (if given) and, after a system-scope fence, totals[3] = ticket, which the host polls. */
int nsb_scan_counts(const int32_t *counts, int64_t n, int32_t *first, int32_t *info2, int64_t *nz_index, int64_t *nz_pack,
                    const int64_t *src, int64_t *nz_src, int64_t *totals, const int64_t *extra_src, int64_t ticket,
                    void *workspace_zeroed, void *stream);
/* bytes of the zero-filled device workspace nsb_scan_counts needs (inter-block totals + ready flags of its one-launch scan) */
int64_t nsb_scan_workspace_bytes(void);
/* merge_two_packs_sorted_aligned (pack_ops.py:529-560) fused with the scatter of the payloads: packs of (dep_a, sdf_a) and rows
 * of (dep_b, sdf_b)[n_packs, n_b], both sorted by depth -> merged (dep_m, sdf_m) and pack_infos_m.  sdf_* may be NULL. */
int nsb_merge_sorted_vals(const float *dep_a, const float *sdf_a, const int64_t *pack_infos_a, const float *dep_b, const float *sdf_b,
                          int64_t n_packs, int32_t n_b, float *dep_m, float *sdf_m, int64_t *pack_infos_m, void *stream);
/* sort(cat(fine stages)) + merge_two_batch_a_includes_b with the coarse samples + ray ids + interval mid-points
 * (neus_ray_query.py:907-976): coarse[n_rays, n_coarse] sorted rows; fine[n_hit, n_fine] rows of the rays ridx_hit (which must be
 * ascending and unique: the kernel finds a ray in the list by binary search), each a concatenation of n_runs sorted runs of run_len_host[q] samples (one per up-sampling stage; HOST array, <= 8 runs).
 * -> d1, mid [S], ridx_all [S], pack_infos [n_rays, 2], S = n_rays n_coarse + n_hit n_fine.  mid and ridx_all may be NULL
 * (not written: nsb_compact_samples can derive both at the kept samples). */
int nsb_assemble_boundary(const float *coarse, int64_t n_rays, int32_t n_coarse, const int64_t *ridx_hit, int64_t n_hit, const float *fine,
                          int32_t n_fine, const int32_t *run_len_host, int32_t n_runs, float *d1, float *mid, int64_t *ridx_all,
                          int64_t *pack_infos, void *stream);
/* gather of the samples packed_volume_render_compression keeps (pack_ops.py:286-291): slot = first_out[p] + rank inside the pack.
 * ridx_all == NULL: ridx_c = the pack index.  t == NULL: t_c = the interval mid-point of nsb_assemble_boundary computed from `d1`
 * (the same value bit for bit); otherwise t_c = t[sample] and d1 is unused. */
int nsb_compact_samples(const uint8_t *selector, const int64_t *pack_infos, const int32_t *first_out, const int32_t *kept, int64_t n_packs,
                        const int64_t *ridx_all, const float *t, const float *d1, const float *alpha, int64_t *pidx, int64_t *ridx_c,
                        float *t_c, float *alpha_c, void *stream);
/* dst[idx[j]] = src[j] (unique idx; adjoint of the gather above). */
int nsb_scatter_f32(const float *src, const int64_t *idx, int64_t n, float *dst, void *stream);
/* AABBSpace.ray_test (nr3d_lib/models/spatial/aabb.py:71-99): normalised rays o_n, d_n [n,3], clamped slab interval near / far [n]
 * and flag[n] = the reference's validity mask.  center3 / radius3 are HOST pointers to 3 floats.  coherent_pairs (device, may be
 * NULL) is incremented by the number of rays i whose origin and direction are within 3 % of ray i-1's (image-ordered rays).
 * row_len (device, may be NULL) is set to the image row length W of image-ordered rays: the first i >= 2 at which the step
 * d[i] - d[i-1] of the direction points against d[1] - d[0] (the return to the start of the next row); -1 if there is none. */
int nsb_ray_test_aabb(const float *rays_o, const float *rays_d, int64_t n, const float *center3, const float *radius3, int has_near,
                      float near_clip, int has_far, float far_clip, float *o_n, float *d_n, float *near, float *far, int32_t *flag,
                      int64_t *coherent_pairs, int64_t *row_len, void *stream);
/* The 8 x 4 pixel-block order of packs for nsb_fused_sdf_collect's mode 2 (count-aware: n_packs live packs).  Pack p lies on pixel
 * pix[via[p]] (via == NULL: pix[p]) of an image with row length *row_len, and the live packs are in ascending pixel order with no pixel
 * twice (what the compactions produce).  order[n_packs] := the packs sorted by (py / 4, px / 8, (py % 4) 8 + px % 8), so that 32
 * consecutive entries are one 8 x 4 block when the block is whole.  The identity if the n_rays rays the ray test saw are not
 * image-ordered by its test (n_rays > 64 and *pairs >= 3/4 (n_rays - 1)), if *row_len < 2, or if a row is wider than 32768. */
int nsb_ray_block_order(const int64_t *pix, const int64_t *via, int64_t n_packs, int64_t n_rays, const int64_t *pairs, const int64_t *row_len,
                        int64_t *order, void *stream);
/* rows idx[j] of (o_n, d_n, near, far) and of one optional per-ray fp32 payload extra[., extra_cols] (rays_h_appear) -> row j of
 * the compacted outputs. */
int nsb_gather_rays(const int64_t *idx, int64_t n, const float *o_n, const float *d_n, const float *near, const float *far, float *o_c,
                    float *d_c, float *near_c, float *far_c, const float *extra, float *extra_c, int32_t extra_cols, void *stream);
/* The adjoint of nsb_ray_test_aabb's normalisation (o' = (o - c) / r, d' = d / r), of nsb_gather_rays, and of the view directions
 * view_dirs = d_c / clamp(|d_c|, 1e-10) with the norm held constant (aabb.py normalize_rays; neus_ray_query.py:793-794): the gradient to
 * the caller's rays for learnable rays.  g_o, g_d, g_vd [R, 3]: the gradient to the compacted ray j's o_c, d_c and view_dirs, held at row
 * idx[j] (the ray map the SDF and colour backward passes add through); vnorm[n]: the clamped norms the forward divided by, in compacted
 * order (needed with g_vd; g_vd NULL: no view-direction term, as for rays that render no rgb).  radius3: HOST pointer to 3 floats.
 * For j < n, i = idx[j]:  d_rays_o[i] = (0 + g_o[i]) / r,  d_rays_d[i] = (0 + (g_d[i] + g_vd[i] / vnorm[j])) / r  (IEEE division, the
 * order torch autograd adds and divides in).  Other rows are not written: the caller zero-fills them. */
int nsb_gather_rays_backward(const int64_t *idx, int64_t n, const float *radius3, const float *g_o, const float *g_d, const float *g_vd,
                             const float *vnorm, float *d_rays_o, float *d_rays_d, void *stream);

/* ---------------------------------------------------------------- camera rays from refined poses (csrc/pose.cu)
 * The StreetSurf camera pose refinement (app/models/scene/learnable_params.py:85-113; nr3d_lib/models/attributes/transform.py:107-130,
 * attr.py:326-336): pose p is the quaternion q0[p] + dq[p] (real part first), normalised on every use, and the translation t0[p] + dt[p].
 * Ray i of pose pidx[i] with camera-space direction dirs[i] is (app/resources/observers/cameras.py:299-310; nr3d_lib/maths/transforms.py:
 * 41-72, 150-193):  rays_d = normalize(quat_apply(normalize_quat(q), dirs[i])),  rays_o = t  -- the direction normalised after the rotation,
 * the origin the camera centre.  normalize(x) = x / max(|x|, 1e-12); normalize_quat also flips a quaternion whose real part is negative.
 * The arithmetic is the reference's torch op sequence, each op rounded, so the rays are the reference's fp32 bits.
 * nsb_pose_rays writes unit[n_poses, 4] (16-byte aligned; the normalised, standardised quaternion, once per pose) and nrm[n_poses] (|q|,
 * negated where the quaternion was flipped; the backward's input), then rays_o, rays_d [n, 3] (count-aware: the rays below the count).
 * pidx must lie in [0, n_poses): the caller checks it (the kernels do not).
 * nsb_pose_rays_backward: from the cotangents d_rays_o, d_rays_d [n, 3] of the same rays (and the forward's unit, nrm), ADDS the gradient
 * to dq into d_dq[n_poses, 4] and to dt into d_dt[n_poses, 3] (either may be NULL: not written).  Each pose's rays are summed in an order
 * fixed by their positions (chunks of 4096 rays, lanes, a fixed butterfly, then the chunks in order): the same bits on every run, for rays
 * in any pose order; a pose without rays gets 0.  Count-aware: rays past the count are not read.  scratch: 16-byte aligned,
 * nsb_pose_grad_scratch_floats(n, n_poses) floats (n the capacity), no initialisation needed. */
int64_t nsb_pose_grad_scratch_floats(int64_t n, int64_t n_poses);
int nsb_pose_rays(const float *q0, const float *dq, const float *t0, const float *dt, int64_t n_poses, const int64_t *pidx, const float *dirs,
                  int64_t n, float *unit, float *nrm, float *rays_o, float *rays_d, void *stream);
int nsb_pose_rays_backward(const float *unit, const float *nrm, int64_t n_poses, const int64_t *pidx, const float *dirs, int64_t n,
                           const float *d_rays_o, const float *d_rays_d, float *scratch, float *d_dq, float *d_dt, void *stream);

/* ---------------------------------------------------------------- perturbed samples from torch's random stream (csrc/perturb.cu)
 * With perturb=True a NeuS query draws from torch's CUDA generator, in order (nr3d_lib/graphics/neus/neus_ray_query.py:803, :821, :889):
 * torch.rand([n_rays, nc1]) for the coarse depths (graphics/raysample.py:285-310), rand_like of the M marched samples' deltas
 * (occgrid_raymarch.py:96-110) and torch.rand([n_hit, nf_i]) for up-sampling stage i (raysample.py:38-61).  Draw k starts at offset
 * base + sum_{j<k} inc(N_j), inc(N) = ((N - 1) / (4 stride) + 1) * 4, stride = 256 min(ceil(N / 256), SMs (maxThreadsPerSM / 256))
 * (torch's ATen/native/cuda/DistributionTemplates.h: calc_execution_policy, distribution_elementwise_grid_stride_kernel; element li is
 * component (li / stride) % 4 of the (li / (4 stride))-th curand_uniform4 of Philox subsequence li % stride, 1 mapped to 0 by uniform_kernel).
 * rng: device int64 {seed, base offset}.  draws_host: n_draws (<= 8) HOST int32 pairs (count slot, multiplier), N_j = counts[slot] * mult, in
 * draw order; the last pair is the entry point's own draw: counts[slot] rows (clamped to the capacity n_rays / n_packs) of n_samples values.
 * next_offset (may be NULL): the offset after the own draw, base + sum of every inc.  No host read: a CUDA graph can capture either call.
 * nsb_coarse_depths_perturbed: t[r, j] = addcmul(near[r], j + u[r, j], (far[r] - near[r]) / n_samples) with torch's fp32 roundings
 *   (the division a product with the fp32 reciprocal, the addcmul one FMA), r below the row count; other rows are not written.
 * nsb_packed_invert_cdf_perturbed: samples[p, j] = nsb_packed_invert_cdf's sample at u = (j + u[p, j]) * (1 / n_samples) (the u of
 *   packed_sample_cdf(perturb=True)), p below the row count; no u buffer. */
int nsb_coarse_depths_perturbed(const float *near, const float *far, int64_t n_rays, int32_t n_samples, const int64_t *rng, const int64_t *counts,
                                const int32_t *draws_host, int32_t n_draws, float *t, int64_t *next_offset, void *stream);
int nsb_packed_invert_cdf_perturbed(const float *bins, const float *cdfs, const int64_t *pack_infos, int64_t n_packs, int32_t n_samples,
                                    const int64_t *rng, const int64_t *counts, const int32_t *draws_host, int32_t n_draws, float *samples,
                                    int64_t *next_offset, void *stream);

/* ---------------------------------------------------------------- error-map importance sampling (csrc/importance.cu)
 * The training batch of one camera as ImpSampler.sample_img_pixel(n) draws it over one ErrorMap (nr3d_lib/models/importance.py:317-336):
 * n_uniform rays from torch.randint(n_images, [n_uniform]) and torch.rand([n_uniform, 2]).clamp_(1e-6, 1 - 1e-6), the other n - n_uniform
 * from torch.rand([n_e]) (the frame, searchsorted on cdf_img) and torch.rand([2, n_e]) (the 2-D inverse cdf), all clamped, drawn in that
 * order from rng = device int64 {seed, offset} (torch_uniform.cuh).  rng_next (may be NULL) := {seed, offset after the four draws}.
 * table: device int64 [n_cameras, NSB_IMP_TABLE_WIDTH], one row per camera: {cdf_img [F], cdf_y [F, res_y], cdf_x [F, res_y, res_x],
 * intrinsics [F, 3, 3] (float32 device pointers), F, W, H, pose_base, appear_base, error_map, last (nsb_error_map_update's), gt_0 ..
 * gt_4 (device pointers of [F, H, W] rows of gt_row_bytes[k] bytes)}; cam: device int64 scalar, the row.  dirs NULL: fidx and xy only (no
 * camera: intrinsics, W, H, the bases and gt are not read).  Per ray r: fidx[r], xy[r] = (x, y) in (0, 1) (unsnapped), pidx[r] =
 * pose_base + fidx, dirs[r] = pinhole_lift(w + 0.5, h + 0.5, 1) of the pixel (w, h) = (xy * WH).long().clamp_(0, WH - 1) (fp32, the
 * reference's operation order, skew included), the n_gt ground-truth rows at (fidx, h, w) into gt_out[k] (HOST array of device
 * pointers, rows of gt_row_bytes[k] (HOST) bytes, copied as stored), and with h_appear the code row appear_table[appear_base + fidx]
 * ([*, n_appear] float32).  No host read.
 * nsb_error_map_update: ErrorMap.update_error_map(fidx, xy, val) (importance.py:87-109) on error_map [n_images, res_y, res_x]: four corner
 * statements in order, each `map[i, h, w] += v` with a cell hit by several rays receiving old + v of the last such ray in batch order.
 * last: int32 [4, n_images, res_y, res_x] scratch, all -1 on entry and on return (the caller fills it once).  With table, error_map, last
 * and the frame count come from row *cam (no host read), n_images then bounds every camera's.  flag |= 1 where a val < 0 (the update still
 * runs).  skip (may be NULL): a device int64; when non-zero the map is left as it is (an overflowed step).  Two launches, deterministic. */
#define NSB_IMP_TABLE_WIDTH 16
#define NSB_IMP_MAX_GT 5
int nsb_imp_sample(const int64_t *table, const int64_t *cam, const int64_t *rng, int64_t n, int64_t n_uniform, int32_t res_y, int32_t res_x,
                   int32_t n_gt, const int64_t *gt_row_bytes, void *const *gt_out, const float *appear_table, int32_t n_appear, float *h_appear,
                   int64_t *fidx, float *xy, int64_t *pidx, float *dirs, int64_t *rng_next, void *stream);
int nsb_error_map_update(float *error_map, int32_t *last, int64_t n_images, const int64_t *table, const int64_t *cam, int32_t res_y, int32_t res_x,
                         const int64_t *fidx, const float *xy, const float *val, int64_t n, int32_t *flag, const int64_t *skip, void *stream);

/* ---------------------------------------------------------------- the LiDAR batch of a frame (csrc/lidar_sample.cu)
 * LidarDataset.sample_merged(frame, n) in the merged_weighted / merged_equal modes (dataio/data_loader/lidar_loader.py:119-204) and the
 * beams' world transform (MultiRaysLidarBundle.get_selected_rays, app/resources/observers/lidars.py:65-78).  table: device int64
 * [n_frames, NSB_LIDAR_TABLE_WIDTH], one row per frame, written by the host once: the frame's first beam in the concatenated arrays
 * (DATA_OFF), its first row of l2w (POSE_BASE: lidar li's transform is row POSE_BASE + li), the generator offsets its draws advance
 * (INC = sum_li inc(num_li)), the lidar count L <= NSB_LIDAR_MAX, the ray segments RAY_START[0 .. L] (lidar li draws the rays
 * [RAY_START[li], RAY_START[li + 1]), RAY_START[L] = n), the cumulative beam counts CUMU[0 .. L] (lidar li's beams are
 * CUMU[li] .. CUMU[li + 1] - 1 of the frame, fewer than 2^32) and each lidar's draw offset DRAW_OFF[li] = sum_{k < li} inc(num_k).
 * frame: device int64 scalar, the row.  rng: device int64 {seed, offset}; lidar li's torch.randint(CUMU[li], CUMU[li + 1], [num_li])
 * starts at offset + DRAW_OFF[li] (torch_uniform.cuh).  Per ray r: the beam b = DATA_OFF + the draw, out_rays_o[r] = R rays_o[b] + t and
 * out_rays_d[r] = R rays_d[b] with (R | t) = l2w[POSE_BASE + li] ([*, 3, 4] float32; a fixed fma order, csrc/lidar_sample.cu),
 * out_ranges[r] = ranges[b], li[r] = li, rays_fidx[r] = *frame.  rng_next (may be NULL) := {seed, offset + INC}.  No host read. */
#define NSB_LIDAR_MAX 8
#define NSB_LIDAR_TABLE_WIDTH 32
#define NSB_LIDAR_ROW_DATA_OFF 0
#define NSB_LIDAR_ROW_POSE_BASE 1
#define NSB_LIDAR_ROW_INC 2
#define NSB_LIDAR_ROW_N_LIDARS 3
#define NSB_LIDAR_ROW_RAY_START 4
#define NSB_LIDAR_ROW_CUMU (NSB_LIDAR_ROW_RAY_START + NSB_LIDAR_MAX + 1)
#define NSB_LIDAR_ROW_DRAW_OFF (NSB_LIDAR_ROW_CUMU + NSB_LIDAR_MAX + 1)
int nsb_lidar_sample(const int64_t *table, const int64_t *frame, const int64_t *rng, int64_t n, const float *rays_o, const float *rays_d,
                     const float *ranges, const float *l2w, float *out_rays_o, float *out_rays_d, float *out_ranges, int64_t *li,
                     int64_t *rays_fidx, int64_t *rng_next, void *stream);

/* ---------------------------------------------------------------- the StreetSurf LiDAR loss (csrc/lidar_loss.cu)
 * LidarLoss.forward with the depth term and the `neus_unisim` line-of-sight term (app/loss/lidar.py:174-210, 254-294) on the renderer's
 * own buffers, and its adjoint: the cotangents of the composite's depth_volume and vw (nsb_composite_backward's g_depth, g_vw).  R rays
 * (the whole-image index; R is the batch, never a device count); blk = {w_depth, w_los, epsilon}: device fp32[3], refreshed by the host
 * before each step.  fn_type: 0 = l1 (recon.py:40-53), 1 = l2_relative (x - y)^2 / (x^2 + 1e-2) (recon.py:119-129).  All sums are
 * deterministic; every fp32 operation rounds as torch's does (no contraction).
 *
 * nsb_lidar_mask_err: mask[r] = (mask_pred[r] > thresh) & (gt[r] > 0), REPLACED by gt[r] <= discard_toofar if has_toofar (lidar.py:264-266:
 *   the reference assigns there); err[r] = |pred[r] - gt[r]| mask[r] (l1_loss(.., reduction='none'), lidar.py:280; loss/utils.py:31-32).
 * nsb_kth_smallest: *out = torch.sort(v).values[k] bit for bit, on the device (lidar.py:281-283 with k = R // 2): an 8-bit-digit radix
 *   select on keys that order like torch.sort (NaN last; a NaN result is returned without its sign).  n <= 65536: one CTA, one launch;
 *   beyond that, four histogram passes over `scratch` (nsb_kth_smallest_scratch_bytes(); zero-filled here).  n < 2^31, 0 <= k < n.
 * nsb_lidar_rows: mask[r] &= !(err[r] > *median * median_factor) (strict >, the product rounded in fp32; median NULL: no discard,
 *   lidar.py:284); depth_row[r] = f(pred[r], gt[r]) mask[r] (may be NULL); los_row[r] = 0 (may be NULL).
 * nsb_lidar_los_rows: one warp per kept ray p < n_packs (count-aware: the rays that keep samples): los_row[rays_inds_hit[p]] =
 *   mask[r] sum_i [|t_i - gt[r]| > epsilon] vw_i^2 over the ray's samples (lidar.py:195-199: the per-ray packed_sum).
 * nsb_lidar_loss_reduce: out[0] = w_depth sum_r depth_row[r] / R (the 'mean' reduction divides by R, loss/utils.py:21-22);
 *   out[1] = w_los sum_r los_row[r] / n_kept, 0 when n_kept == 0 (lidar.py:208-210; count-aware: n_kept).  One CTA, fp64 sums over the
 *   R whole-image rows in one fixed order: the result does not depend on the kept-sample arena or the kept rays' order.  Either row
 *   array may be NULL (that term is 0).
 * nsb_lidar_depth_backward: g_depth[r] = f'(pred, gt) mask[r] g_out[0] w_depth / R (l1: sign with sign(0) = 0; l2_relative: both the
 *   numerator and the denominator differentiated, as autograd does).  The mask is a constant (the reference's `.data`).
 * nsb_lidar_los_backward: g_vw[i] = g_out[1] w_los / n_kept mask[r] [|t_i - gt[r]| > epsilon] 2 vw_i for the samples of the kept rays
 *   (count-aware: n_kept); other rows of g_vw are not written. */
int64_t nsb_kth_smallest_scratch_bytes(void);
int nsb_lidar_mask_err(const float *pred, const float *mask_pred, const float *gt, int64_t n, float mask_pred_thresh, int32_t has_toofar,
                       float discard_toofar, float *mask, float *err, void *stream);
int nsb_kth_smallest(const float *v, int64_t n, int64_t k, float *out, void *scratch, void *stream);
int nsb_lidar_rows(const float *pred, const float *gt, const float *err, const float *median, float median_factor, int32_t fn_type, int64_t n,
                   float *mask, float *depth_row, float *los_row, void *stream);
int nsb_lidar_los_rows(const float *t, const float *vw, const int64_t *pack_infos, const int64_t *rays_inds_hit, int64_t n_packs,
                       const float *gt, const float *mask, const float *blk, float *los_row, void *stream);
int nsb_lidar_loss_reduce(const float *depth_row, const float *los_row, int64_t n, int64_t n_kept, const float *blk, float *out, void *stream);
int nsb_lidar_depth_backward(const float *pred, const float *gt, const float *mask, int64_t n, int32_t fn_type, const float *blk,
                             const float *g_out, float *g_depth, void *stream);
int nsb_lidar_los_backward(const float *t, const float *vw, const int64_t *pack_infos, const int64_t *rays_inds_hit, int64_t n_packs,
                           const float *gt, const float *mask, const float *blk, const float *g_out, float *g_vw, void *stream);

/* ---------------------------------------------------------------- occupancy-grid maintenance (csrc/occ_ema.cu)
 * OccGridEma._step_update_occ (nr3d_lib/models/accelerations/occgrid/ema_single.py:176-190; occgrid/utils.py:63-101) in three small launches:
 * evidence of n points (val = sdf -> normalized_logistic_density on fp16, or val = ready evidence) max-scattered into their voxels
 * ((pts/2+0.5) res, clamped), merged with the non-zero cells of the collected-evidence grid `pcl` (zeroed afterwards; may be NULL), then
 * on every TOUCHED voxel  grid = max(ema_decay grid, evidence);  occ_grid = grid > occ_thre on all voxels; occ_bits (may be NULL) = the
 * bool grid packed 32 cells / word (what nsb_ray_marching_listed takes).  scratch_cells: rx ry rz floats.  Replaces torch_scatter's
 * scatter_max + index_put + nonzero (a host sync) of the reference. */
int nsb_occ_ema_update(const float *pts, const float *val, int64_t n, int32_t val_is_sdf, float inv_s, int32_t rx, int32_t ry, int32_t rz,
                       float *pcl_or_null, float *occ_val_grid, uint8_t *occ_grid, uint32_t *occ_bits_or_null, float ema_decay, float occ_thre,
                       float *scratch_cells, void *stream);
/* nsb_occ_ema_update over the first *n_dev of n_capacity points (a device-resident count); with skip_or_null pointing at a non-zero
 * int64 the update changes nothing (neither grid nor pcl). */
int nsb_occ_ema_update_count(const float *pts, const float *val, const int64_t *n_dev, int64_t n_capacity, int32_t val_is_sdf, float inv_s,
                             int32_t rx, int32_t ry, int32_t rz, float *pcl_or_null, float *occ_val_grid, uint8_t *occ_grid,
                             uint32_t *occ_bits_or_null, float ema_decay, float occ_thre, float *scratch_cells, const int64_t *skip_or_null,
                             void *stream);

/* ---------------------------------------------------------------- the grid's update from the network (csrc/occ_update.cu)
 * OccGridEma._step (ema_single.py:133-175) and sample_pts_in_voxels (occgrid/utils.py:17-41) without a host read.
 * nsb_occ_voxel_lists: the occupied and the empty cells of occ_grid[cells] (bool bytes) as flat indices (row-major, last axis fastest:
 *   nonzero()'s order) in occupied[cells] / empty[cells]; counts[0] = occupied cells, counts[1] = empty cells (device).  flags, first:
 *   int32 [cells] scratch; workspace: nsb_scan_workspace_bytes() of device memory (zeroed here).  One scan (nsb_scan_counts).
 * nsb_occ_draw_pts: the points of one update's num_steps iterations, in the reference's order, drawn from torch's CUDA generator at
 *   (rng[0] seed, rng[1] offset): per iteration, with *warmup != 0, num_pts points in all cells; else num_pts / 2 in all cells,
 *   num_pts / 4 in the empty cells (none if there are none) and num_pts / 4 in the occupied cells (the voxel lists above).  Each part is
 *   sample_pts_in_voxels's torch.randint + torch.rand (n < 2 nv) or torch.rand of nv (n / nv + 1) points, each draw at the offset the
 *   previous one's left, the values and fp32 roundings torch gives.  pts[capacity, 3]; out[0] = the points drawn, out[1] = 1 when the
 *   steady phase found no occupied cell (then nothing is drawn: the reference asserts), else 0.  capacity >= num_steps times the
 *   larger phase's sum over its parts of n + min(cells, n / 2) (a part of n points draws at most that many). */
int nsb_occ_voxel_lists(const uint8_t *occ_grid, int64_t cells, int32_t *flags, int32_t *first, int64_t *occupied, int64_t *empty,
                        int64_t *counts, void *workspace, void *stream);
int nsb_occ_draw_pts(const int64_t *rng, const int32_t *warmup, const int64_t *counts, const int64_t *occupied, const int64_t *empty,
                     int32_t rx, int32_t ry, int32_t rz, int32_t num_steps, int64_t num_pts, int64_t capacity, float *pts, int64_t *out,
                     void *stream);

/* ---------------------------------------------------------------- fused colour / normal query (csrc/color_tc.cu)
 * The whole LoTDNeuS.forward of the reference for packed samples (nr3d_lib/models/fields/neus/lotd_neus.py:141-167 =
 * LoTDSDF.forward_sdf_nablas, lotd_sdf.py:201-257, + RadianceNet.forward, mlp_nerf.py:267-289) as one wgmma kernel, and
 * its backward including the second-order pass through nablas (LoTDFunctionBwdDydx.backward, lotd.py:193-268) as two.
 * All weight pointers are fp16 device images of the fp32 masters (what autocast feeds the GEMMs). */
typedef struct nsb_color_net {
    const void *W1, *b1, *W2, *b2;            /* sdf decoder: [width x 2L], [width], [1 x width], [1] (L levels, 1..24) */
    const void *R1, *rb1, *R2, *rb2, *R3, *rb3; /* radiance net: [rw x rad_in], [rw], [rw x rw], [rw], [3 x rw], [3] */
    int32_t width, rad_width, rad_in, n_appear; /* rad_in = 3 + 16 + 3 + 2L + n_appear ([x, SH4(v), n, h, h_appear]) */
    float beta;                               /* Softplus beta of the decoder                                      */
    float nablas_scale[3];                    /* sdf_scale / radius3d_original                                     */
} nsb_color_net;

/* bytes of ONE saved activation buffer for n points (fp16 tiles of 128 points x 64 columns, core-matrix layout) */
int64_t nsb_color_tile_bytes(int64_t n);
/* bytes of ONE saved activation buffer for n points of an L-level table: nsb_color_tile_bytes(n) for L <= 16; for L = 17..24 the X tile
 * is 80 columns wide (h takes 48), so every buffer is sized n_tiles x 20 KB */
int64_t nsb_color_act_bytes(int64_t n, int32_t n_levels);
/* Points are x[n,3] or rays_o/rays_d[R,3] + ridx[n] (NULL = identity) + t[n]; view_dirs[R,3] and h_appear[R,n_appear] are
 * indexed by ridx (by the point index when ridx is NULL).  Outputs fp32: sdf[n], nablas[n,3], rgb[n,3], x_out[n,3] (optional).
 * act_* : four buffers of nsb_color_act_bytes(n, L) each kept for the backward, or all NULL for inference.
 * collect: NULL or the occupancy-evidence side effect of forward_sdf_nablas (see nsb_occ_collect).
 * rgb == NULL selects the geometry-only form (LoTDSDF.forward_sdf_nablas alone): sdf, nablas, x_out, act_z and the h half of act_x are
 * written exactly as with rgb, nothing of the radiance net is read, view_dirs, h_appear, act_y1 and act_y2 may be NULL (act_z and act_x
 * both or neither), and net_host may have rad_width == 0 with NULL radiance pointers (a model without a radiance net). */
int nsb_fused_color_fwd(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                        const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *view_dirs,
                        const float *h_appear, int64_t n, int32_t max_level, float *sdf, float *nablas, float *rgb, float *x_out,
                        void *act_z, void *act_x, void *act_y1, void *act_y2, const nsb_occ_collect *collect, void *stream);
/* Cotangents g_sdf[n], g_nablas[n,3], g_rgb[n,3] (each may be NULL = zero); dh_scratch[n,32] fp32 workspace ([n,48] for tables of 17..24 levels).
 * All gradient outputs are fp32 and ACCUMULATED into (caller zero-fills); d_R* use the reference's column order.
 * With g_rgb == NULL the radiance backward does not run: act_y1, act_y2, rgb, dh_scratch and d_R* / d_rb* may then be NULL, and net_host
 * may have rad_width == 0 with NULL radiance pointers (the activations of a geometry-only forward are enough). */
int nsb_fused_color_bwd(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                        const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                        const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                        const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1,
                        float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3,
                        float *d_rb3, void *stream);
/* nsb_fused_color_bwd plus the gradient to the appearance codes h_appear[R, n_appear] of the forward (the reference's RadianceNet input
 * columns after h, looked up per ray in single_volume_renderer.py:170-175, so autograd carries it back to the per-image codes):
 * d_h_appear[ray_map[ridx[i]]] += sum over the points i of a ray of dL/dh_appear_i (ray_map NULL: row ridx[i]; ridx NULL: row i).
 * g_rgb is required and the net must have n_appear >= 1.  ha_scratch[n, 8] fp32 workspace (the per-point rows).  The points of a ray
 * must be consecutive (packed samples) for the sum to be deterministic: each ray's points are then summed by one warp in a fixed order
 * and added once onto the caller's zeros.  Rays without a point are not written; with device counts, neither are points or rays past
 * the count.  Everything else as nsb_fused_color_bwd, which computes the same bits in dh_scratch and the other outputs. */
int nsb_fused_color_bwd_appear(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                               const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                               const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                               const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1,
                               float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3,
                               float *d_rb3, float *ha_scratch, const int64_t *ray_map, float *d_h_appear, void *stream);
/* nsb_fused_color_bwd with any of the appearance-code and ray gradients (the shipped configurations train both).  Every output is
 * optional; NULL means not wanted, and with none this is nsb_fused_color_bwd.
 *   d_h_appear: as nsb_fused_color_bwd_appear (needs g_rgb and ha_scratch[n, 8]).
 *   d_rays_o, d_rays_d, d_view_dirs [R, 3]: the gradient to the rays of the points x = rays_o[ridx] + rays_d[ridx] t (x must be NULL) and
 *   to the per-ray view directions view_dirs[R, 3] the forward read (needed with g_rgb).  The depths t are constants.  A point gets
 *     g_x = (1/2) sum over levels of J^T (dh_z + dh_r) + dL/dx of the radiance input      g_v = (dSH4/dv)^T dL/dSH of the radiance input
 *   with dh_z the decoder's and dh_r the radiance net's cotangent of the features (first order: the table-Hessian term of the nablas
 *   backward does not reach x, as the reference's encoding does not form its input Hessian on the hot path); then per ray
 *     d_rays_o[ray_map[r]] += sum of g_x,   d_rays_d[ray_map[r]] += sum of t g_x,   d_view_dirs[ray_map[r]] += sum of g_v
 *   (ray_map NULL: row r).  ray_scratch[n, 36] fp32 workspace.  The caller zero-fills the outputs; the sums are deterministic for packed
 *   samples, as for the codes.  The caller maps d_view_dirs onto its rays (view_dirs = rays_d / |rays_d| with a constant norm).
 * Everything else as nsb_fused_color_bwd, which computes the same bits in the other outputs. */
int nsb_fused_color_bwd_grads(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                              const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                              const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                              const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1,
                              float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3,
                              float *d_rb3, const float *view_dirs, float *ha_scratch, const int64_t *ray_map, float *d_h_appear,
                              float *ray_scratch, float *d_rays_o, float *d_rays_d, float *d_view_dirs, void *stream);

/* ---------------------------------------------------------------- the persistent per-ray kernel (csrc/ray_upsample.cu)
 * The no-grad up-sampling half of neus_ray_query_march_occ_multi_upsample_compressed (neus_ray_query.py:861-905) for every hit ray as ONE
 * persistent kernel: sdf of the marched samples, then per stage cdf -> n_fine[i] inverse-cdf samples -> sdf -> merge, with the ray's samples in
 * shared memory (replaces 11 launches of the stage kernels above, with bit-identical results: the alpha, replay, scan, cdf, inverse-cdf and
 * merge device functions are the ones the stage kernels call, and tests/test_ray_upsample_edges_gpu.py pins the kernel to them).
 * fine_all[n_hit, sum(n_fine)] = cat of the stages' samples; the row of an empty pack or of an overflowing ray is not written.
 * n_fine / inv_s_stage / u_stage are HOST arrays of n_stage entries; u_stage[i] points to DEVICE memory with the n_fine[i] quantiles of stage i (linspace(0,1,n+2)[1:-1]: `perturb=False`).
 * A ray with more marched samples than the shared-memory capacity works in its slice of `scratch` (nsb_upsample_rays_scratch_floats(n_hit
 * capacity, long_cap) floats; long_cap >= max marched samples per ray + sum of the merged stages); overflow[n_hit] (caller zero-fills) is
 * set only for a ray that exceeds long_cap (or the shared-memory capacity when scratch == NULL).  collect: in-kernel sample collection of the
 * training-time SDF queries (may be NULL).  Count-aware (nsb_bind_device_counts: n_hit). */
int nsb_upsample_rays(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *rays_o,
                      const float *rays_d, const float *t_starts, const int64_t *pack_infos, const int64_t *ridx_hit, int64_t n_hit,
                      int32_t max_level, int32_t n_stage, const int32_t *n_fine_host, const float *inv_s_stage_host,
                      const float *const *u_stage_host, int32_t use_estimate_alpha, float early_stop_eps, float alpha_thre, float *fine_all,
                      int32_t *overflow, float *scratch, int32_t long_cap, const nsb_occ_collect *collect, void *stream);
int64_t nsb_upsample_rays_scratch_floats(int64_t n_hit_capacity, int32_t long_cap);
/* the same without scratch / collection (rays beyond the shared-memory capacity are flagged in `overflow`) */
int nsb_upsample_persistent(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *rays_o,
                            const float *rays_d, const float *t_starts, const int64_t *pack_infos, const int64_t *ridx_hit, int64_t n_hit,
                            int32_t max_level, int32_t n_stage, const int32_t *n_fine, const float *inv_s_stage, const float *const *u_stage,
                            int32_t use_estimate_alpha, float early_stop_eps, float alpha_thre, float *fine_all, int32_t *overflow, void *stream);

/* ---------------------------------------------------------------- marching cubes (csrc/mesh.cu)
 * The stages of nr3d_lib.graphics.trianglemesh.extract_mesh (trianglemesh.py:134-254: lattice, SDF volume, skimage marching cubes) on a
 * lattice of n0 x n1 x n2 points (point (i, j, k) at flat index (i n1 + j) n2 + k, k fastest: meshgrid(indexing="ij")) streamed in slabs of
 * whole planes along axis 0.  A slab owns planes [p0, p1): the vertices on the edges (+x, +y, +z) their points own and the cells
 * (p0 - 1 .. p1 - 2).  Slot l in [0, (p1 - p0) n1 n2) of every per-slab array is point (p0 + l / (n1 n2), j, k) and cell (p0 - 1 + l / (n1 n2), j, k).
 * sdf_win: fp32 planes [w0, w0 + n_win) of the volume, holding at least planes [p0 - 1, p1 + 1) (count) / [p0 - 1, p1 + 2) (vertices), clipped
 * to [0, n0).  A point is inside when sdf < level.  The case table (csrc/mc_table.cuh) is generated by oracle/mc_table.py.
 *
 * nsb_mc_lattice_points: x[n, 3] = (lin0[i], lin1[j], lin2[k]) of the flat indices start .. start + n - 1 (the query points).
 * nsb_mc_count: flags[l] = bits (x, y, z) of the owned edges whose ends differ in sign, vcount[l] = their number; cases[l] = case index of
 *   the cell of slot l (0 if it does not exist), tcount[l] = its triangle count.  Scan both counts (nsb_scan_counts) for vfirst / tfirst.
 * nsb_mc_vertices: the vertices of slot l at vfirst[l] + 0, 1, 2 in axis order: position bmin + spacing (idx + t), t = (level - s0) / (s1 - s0),
 *   normal = normalise(g0 + t (g1 - g0)) of the lattice gradients g (central differences, one-sided at the volume border, over the spacing);
 *   fp64 arithmetic, fp32 outputs verts[., 3], normals[., 3].  bmin3_host / spacing3_host: HOST arrays of 3 doubles.
 * nsb_mc_triangles: faces[tfirst[l] + q] (int32 [., 3]) = triangle q of the cell of slot l, as global vertex ids: vbase + vfirst + rank of the
 *   edge among its owner's flags, or, for an owner on plane p0 - 1, carry_base + carry_first[jk] + rank among carry_flags[jk] (that plane's
 *   flags and scanned offsets, kept from the previous slab; may be NULL when p0 == 0).  The caller makes sure the ids fit in int32. */
int nsb_mc_lattice_points(const float *lin0, const float *lin1, const float *lin2, int32_t n1, int32_t n2, int64_t start, int64_t n, float *x,
                          void *stream);
int nsb_mc_count(const float *sdf_win, int32_t w0, int32_t n_win, int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1, double level,
                 uint8_t *flags, int32_t *vcount, uint8_t *cases, int32_t *tcount, void *stream);
int nsb_mc_vertices(const float *sdf_win, int32_t w0, int32_t n_win, int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1, double level,
                    const double *bmin3_host, const double *spacing3_host, const uint8_t *flags, const int32_t *vfirst, float *verts, float *normals,
                    void *stream);
int nsb_mc_triangles(int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1, const uint8_t *cases, const int32_t *tcount, const int32_t *tfirst,
                     const uint8_t *flags, const int32_t *vfirst, int64_t vbase, const uint8_t *carry_flags, const int32_t *carry_first,
                     int64_t carry_base, int32_t *faces, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NEURALSIM_B200_H */
