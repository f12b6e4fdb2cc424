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
/* Self-check / A-B switches: key "sdf_simt" (0|1) routes nsb_fused_sdf* through the CUDA-core cross-check kernel; "color_tma" (0|1|2) the
 * TMA fetch of the saved activation tiles in the colour backward; "asm_chunk" (1|8) rays per search of the hit list in nsb_assemble_boundary. */
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
/* packed_sort_qsort: ascending, in place on vals; idx (may be NULL) receives global gather indices. */
int nsb_packed_sort(float *vals, const int64_t *pack_infos, int64_t n_packs, int64_t *idx, void *stream);
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
typedef struct nsb_sdf_decoder {       /* LoTDSDF decoder 32->W->1, Softplus(beta)  (lotd_sdf.py:176-200) */
    const void *W1;                    /* fp16 [W, F]   (fp32 master rounded by the caller) */
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

/* forward_sdf on N points: x in network space [-1,1]^3 (not yet /2+0.5).  sdf fp32 (fp16-valued). */
int nsb_fused_sdf(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host,
                  const float *x, int64_t n, int32_t max_level, float *sdf, void *h_out_half, void *stream);
/* the three queries below with the occupancy-evidence side effect (collect may be NULL = the plain query) */
int nsb_fused_sdf_collect(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_sdf_decoder *dec_host, const float *x,
                          const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n,
                          const int64_t *pack_infos, const int64_t *pack_ray, int64_t n_packs, int32_t mode, int32_t max_level, float *sdf,
                          const nsb_occ_collect *collect, void *stream);

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

/* ---------------------------------------------------------------- device-resident sizes (a step without host reads)
 * The reference reads every data-dependent size back to the host (`.item()`, `nonzero()`: ~25 syncs per ray_query, SURVEY.md §8a a9).
 * Here a size may stay in device memory: nsb_bind_device_counts(c0, c1) binds one or two device int64 to the calling thread; the NEXT
 * count-aware entry point of that thread consumes (and clears) the binding and its kernel processes min(n_arg, *c0) items -- n_arg
 * (the `n` / `n_packs` / `n_rays` / `n_list` argument) then is the CAPACITY the buffers and the grid were sized for.  c1 is the second
 * count of nsb_assemble_boundary (n_hit).  Count-aware: nsb_gather_rays, nsb_ray_marching_listed (first round: num_steps of the rays
 * in [*c0, n_rays) is written as 0; second round: the listed rays), nsb_ray_marching_record / nsb_march_compact (the same), nsb_fused_sdf_collect / _rays / _packs, nsb_fused_sdf_bwd(_indexed),
 * nsb_neus_upsample_cdf, nsb_packed_invert_cdf_shared_u, nsb_merge_sorted_vals, nsb_assemble_boundary, nsb_neus_alpha_forward
 * (num_steps of the packs in [*c0, n_packs) is written as 0) / _backward, nsb_compact_samples, nsb_scatter_f32, nsb_flag_nonzero,
 * nsb_fused_color_fwd / _bwd, nsb_composite_forward / _backward.  With every size on the device a whole fwd+bwd step has no host
 * read and can be captured in a CUDA graph (neuralsim_b200/graphics/neus_static.py). */
int nsb_bind_device_counts(const int64_t *count0, const int64_t *count1);
/* flag[i] = (v[i] != 0) for i < live count, 0 up to n (count-aware). */
int nsb_flag_nonzero(const float *v, int64_t n, int32_t *flag, void *stream);
/* Derived sizes of one NeuS query in a device block `counts` of >= 32 int64 (zero-filled once per query):
 *   written by nsb_scan_counts (totals = counts + 0 / + 3 / + 6 / + 9):
 *     [0] rays that pass the box test  [2] coherent neighbour pairs   [3] M marched samples  [4] n_hit rays with samples
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
 * (what packed_sample_cdf(perturb=False) feeds it, graphics/raysample.py:38-61). */
int nsb_packed_invert_cdf_shared_u(const float *bins, const float *cdfs, const float *u, const int64_t *pack_infos, int64_t n_packs,
                                   int32_t n_samples, float *samples, void *stream);
/* alpha[S] = neus_packed_sdf_to_alpha(sdf, *inv_s_dev) and, in the same pass, the compression selector / kept-count per pack
 * of packed_volume_render_compression (pack_ops.py:286-291).  inv_s is read from device memory (no host sync). */
int nsb_neus_alpha_forward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, float early_stop_eps,
                           float alpha_thre, float *alpha, uint8_t *selector, int32_t *num_steps, void *stream);
/* adjoint of the above: d_sdf[S] (written), d_inv_s[1] (accumulated; caller zero-fills). */
int nsb_neus_alpha_backward(const float *sdf, const int64_t *pack_infos, int64_t n_packs, const float *inv_s_dev, const float *d_alpha,
                            float *d_sdf, float *d_inv_s, void *stream);
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
 * (neus_ray_query.py:907-976): coarse[n_rays, n_coarse] sorted rows; fine[n_hit, n_fine] rows of the rays ridx_hit (sorted,
 * unique), each a concatenation of n_runs sorted runs of run_len_host[q] samples (one per up-sampling stage; HOST array, <= 8 runs).
 * -> d1, mid [S], ridx_all [S], pack_infos [n_rays, 2], S = n_rays n_coarse + n_hit n_fine. */
int nsb_assemble_boundary(const float *coarse, int64_t n_rays, int32_t n_coarse, const int64_t *ridx_hit, int64_t n_hit, const float *fine,
                          int32_t n_fine, const int32_t *run_len_host, int32_t n_runs, float *d1, float *mid, int64_t *ridx_all,
                          int64_t *pack_infos, void *stream);
/* gather of the samples packed_volume_render_compression keeps (pack_ops.py:286-291): slot = first_out[p] + rank inside the pack. */
int nsb_compact_samples(const uint8_t *selector, const int64_t *pack_infos, const int32_t *first_out, const int32_t *kept, int64_t n_packs,
                        const int64_t *ridx_all, const float *t, const float *alpha, int64_t *pidx, int64_t *ridx_c, float *t_c,
                        float *alpha_c, void *stream);
/* dst[idx[j]] = src[j] (unique idx; adjoint of the gather above). */
int nsb_scatter_f32(const float *src, const int64_t *idx, int64_t n, float *dst, void *stream);
/* AABBSpace.ray_test (nr3d_lib/models/spatial/aabb.py:71-99): normalised rays o_n, d_n [n,3], clamped slab interval near / far [n]
 * and flag[n] = the reference's validity mask.  center3 / radius3 are HOST pointers to 3 floats.  coherent_pairs (device, may be
 * NULL) is incremented by the number of rays i whose origin and direction are within 3 % of ray i-1's (image-ordered rays). */
int nsb_ray_test_aabb(const float *rays_o, const float *rays_d, int64_t n, const float *center3, const float *radius3, int has_near,
                      float near_clip, int has_far, float far_clip, float *o_n, float *d_n, float *near, float *far, int32_t *flag,
                      int64_t *coherent_pairs, void *stream);
/* rows idx[j] of (o_n, d_n, near, far) and of one optional per-ray fp32 payload extra[., extra_cols] (rays_h_appear) -> row j of
 * the compacted outputs. */
int nsb_gather_rays(const int64_t *idx, int64_t n, const float *o_n, const float *d_n, const float *near, const float *far, float *o_c,
                    float *d_c, float *near_c, float *far_c, const float *extra, float *extra_c, int32_t extra_cols, void *stream);

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

/* ---------------------------------------------------------------- fused colour / normal query (csrc/color_tc.cu)
 * The whole LoTDNeuS.forward of the reference for packed samples (nr3d_lib/models/fields/neus/lotd_neus.py:141-167 =
 * LoTDSDF.forward_sdf_nablas, lotd_sdf.py:201-257, + RadianceNet.forward, mlp_nerf.py:267-289) as one wgmma kernel, and
 * its backward including the second-order pass through nablas (LoTDFunctionBwdDydx.backward, lotd.py:193-268) as two.
 * All weight pointers are fp16 device images of the fp32 masters (what autocast feeds the GEMMs). */
typedef struct nsb_color_net {
    const void *W1, *b1, *W2, *b2;            /* sdf decoder: [width x 32], [width], [1 x width], [1]              */
    const void *R1, *rb1, *R2, *rb2, *R3, *rb3; /* radiance net: [rw x rad_in], [rw], [rw x rw], [rw], [3 x rw], [3] */
    int32_t width, rad_width, rad_in, n_appear; /* rad_in = 3 + 16 + 3 + 32 + n_appear ([x, SH4(v), n, h, h_appear]) */
    float beta;                               /* Softplus beta of the decoder                                      */
    float nablas_scale[3];                    /* sdf_scale / radius3d_original                                     */
} nsb_color_net;

/* bytes of ONE saved activation buffer for n points (fp16 tiles of 128 points x 64 columns, core-matrix layout) */
int64_t nsb_color_tile_bytes(int64_t n);
/* Points are x[n,3] or rays_o/rays_d[R,3] + ridx[n] (NULL = identity) + t[n]; view_dirs[R,3] and h_appear[R,n_appear] are
 * indexed by ridx (by the point index when ridx is NULL).  Outputs fp32: sdf[n], nablas[n,3], rgb[n,3], x_out[n,3] (optional).
 * act_* : four buffers of nsb_color_tile_bytes(n) each kept for the backward, or all NULL for inference.
 * collect: NULL or the occupancy-evidence side effect of forward_sdf_nablas (see nsb_occ_collect). */
int nsb_fused_color_fwd(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                        const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, const float *view_dirs,
                        const float *h_appear, int64_t n, int32_t max_level, float *sdf, float *nablas, float *rgb, float *x_out,
                        void *act_z, void *act_x, void *act_y1, void *act_y2, const nsb_occ_collect *collect, void *stream);
/* Cotangents g_sdf[n], g_nablas[n,3], g_rgb[n,3] (each may be NULL = zero); dh_scratch[n,32] fp32 workspace.
 * All gradient outputs are fp32 and ACCUMULATED into (caller zero-fills); d_R* use the reference's column order. */
int nsb_fused_color_bwd(const nsb_lotd_meta *meta_host, const void *params_half, const nsb_color_net *net_host, const float *x,
                        const float *rays_o, const float *rays_d, const int64_t *ridx, const float *t, int64_t n, int32_t max_level,
                        const void *act_z, const void *act_x, const void *act_y1, const void *act_y2, const float *rgb,
                        const float *g_sdf, const float *g_nablas, const float *g_rgb, float *dh_scratch, float *d_grid, float *d_W1,
                        float *d_b1, float *d_W2, float *d_b2, float *d_R1, float *d_rb1, float *d_R2, float *d_rb2, float *d_R3,
                        float *d_rb3, void *stream);

/* ---------------------------------------------------------------- the persistent per-ray kernel (csrc/ray_upsample.cu)
 * The no-grad up-sampling half of neus_ray_query_march_occ_multi_upsample_compressed (neus_ray_query.py:861-905) for every hit ray as ONE
 * persistent kernel: sdf of the marched samples, then per stage cdf -> n_fine[i] inverse-cdf samples -> sdf -> merge, with the ray's samples in
 * shared memory (replaces 11 launches of the stage kernels above; bit-identical results: same device functions).
 * fine_all[n_hit, sum(n_fine)] = cat of the stages' samples.  n_fine / inv_s_stage / u_stage are HOST arrays of n_stage entries; u_stage[i]
 * points to DEVICE memory with the n_fine[i] quantiles of stage i (linspace(0,1,n+2)[1:-1]: `perturb=False`).
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

#ifdef __cplusplus
}
#endif
#endif /* NEURALSIM_B200_H */
