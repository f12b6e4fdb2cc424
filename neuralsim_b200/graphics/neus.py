"""NeuS maths and the per-ray query -- API of `nr3d_lib.graphics.neus`
(reference: nr3d_lib/nr3d_lib/graphics/neus/neus_utils.py, neus_ray_query.py:732-1104).

`neus_ray_query_march_occ_multi_upsample_compressed(model, ray_tested, ...)` is the hot path's entry point: the
function `NeusRendererMixin.ray_query` dispatches to for `query_mode: march_occ_multi_upsample_compressed`
(renderer_mixin.py:346-350).  It returns the same packed `volume_buffer` dict (renderer_mixin.py:263-303).
Duck-typed `model` interface: forward_sdf(x)->{'sdf'}, forward(x, v=, h_appear=, nablas_has_grad=, with_rgb=,
with_normal=)->{'sdf','nablas','rgb','h'}, forward_inv_s(), accel.ray_march(rays_o, rays_d, near=, far=, perturb=, **march_cfg).

Two implementations of the same function live here: the op-by-op chain in the reference's own formulation (every call a
`nr3d_lib`-named wrapper of this package), and `_query_fused`, one launch per stage (csrc/neus_glue.cu, neus_fused.cu, fused_tc.cu,
color_tc.cu), taken when the model offers `forward_sdf_on_rays` and the occupancy grid is a single 3-D grid.  FUSED_STAGES = False
forces the chain; tests/test_neus_fused_gpu.py renders with both and compares samples, images and gradients.
"""
from __future__ import annotations

from operator import itemgetter

import torch

from .nerf import packed_alpha_to_vw, packed_volume_render_compression, ray_alpha_to_vw
from .pack_ops import (get_pack_infos_from_batch, merge_two_batch_a_includes_b, merge_two_packs_sorted_aligned,
                       packed_cumsum, packed_diff, packed_div)
from .raysample import batch_sample_step_linear, packed_sample_cdf
from . import neus_fused

# True: the per-ray stages run as the fused kernels of csrc/neus_fused.cu; False: as the reference's chain of
# pack_ops / elementwise calls (same maths; kept for the parity tests and as documentation of what is fused).
FUSED_STAGES = True
import os as _os
# The no-grad half of the fused query (sdf of the marched samples + the up-sampling stages) as ONE persistent per-ray kernel
# (csrc/ray_upsample.cu) or as one launch per stage -- same values either way (tests/test_ray_upsample_gpu.py).  The persistent kernel saves
# launches on small batches (25 instead of 35 for 4096 random rays) and loses on large ones (its 128-point tiles are filled by 4 rays' 9-sample
# stages to 28 %), so: True / False force it, "auto" (default) takes it below PERSISTENT_MAX_RAYS tested rays.  perturb=True always runs the stage kernels.
_pu = _os.environ.get("NSB_PERSISTENT_UPSAMPLE", "auto")
PERSISTENT_UPSAMPLE = "auto" if _pu == "auto" else (_pu != "0")
PERSISTENT_MAX_RAYS = 8192


def use_persistent_upsample(n_rays: int) -> bool:
    return (n_rays < PERSISTENT_MAX_RAYS) if PERSISTENT_UPSAMPLE == "auto" else bool(PERSISTENT_UPSAMPLE)
MARCHED_TILED = _os.environ.get("NSB_MARCHED_TILED", "0") != "0"     # ray-tiled traversal of the marched samples (off: ray-major was the faster order)

__all__ = ["neus_cdf", "neus_ray_cdf_to_alpha", "neus_ray_sdf_to_alpha", "neus_ray_sdf_to_vw", "neus_packed_cdf_to_alpha",
           "neus_packed_sdf_to_alpha", "neus_packed_sdf_to_upsample_alpha", "neus_ray_sdf_to_upsample_alpha",
           "neus_ray_query_march_occ_multi_upsample_compressed"]


def neus_cdf(x, inv_s):
    return torch.sigmoid(x * inv_s)


# ---- batched rays [..., n+1] boundary values -> [..., n] interval alphas
def neus_ray_cdf_to_alpha(cdf, append_cdf_1=False):
    if append_cdf_1:
        d = cdf.diff(append=cdf.new_full((*cdf.shape[:-1], 1), 1.))
        return (-d / (cdf + 1e-5)).clamp_min(0)
    return (-cdf.diff() / (cdf[..., :-1] + 1e-5)).clamp_min(0)


def neus_ray_sdf_to_alpha(sdf, inv_s, append_cdf_1=False):
    return neus_ray_cdf_to_alpha(torch.sigmoid(sdf * inv_s), append_cdf_1)


def neus_ray_sdf_to_vw(sdf, inv_s, append_cdf_1=False):
    return ray_alpha_to_vw(neus_ray_sdf_to_alpha(sdf, inv_s, append_cdf_1))


# ---- packed rays: one alpha per boundary point, the last of every pack is 0 (or uses the appended cdf)
def neus_packed_cdf_to_alpha(cdf, pack_infos, append_cdf_1=False, pack_cdf_appends=None):
    if append_cdf_1:
        pack_cdf_appends = cdf.new_full((pack_infos.shape[0],), 1.)
    drop = -1 * packed_diff(cdf, pack_infos, pack_appends=pack_cdf_appends)
    return (drop / (cdf + 1e-5)).clamp_min(0)


def neus_packed_sdf_to_alpha(sdf, inv_s, pack_infos, append_cdf_1=False, pack_sdf_appends=None):
    app = None if pack_sdf_appends is None else torch.sigmoid(pack_sdf_appends * inv_s)
    return neus_packed_cdf_to_alpha(torch.sigmoid(sdf * inv_s), pack_infos, append_cdf_1, app)


@torch.no_grad()
def neus_packed_sdf_to_upsample_alpha(sdf, depth_samples, inv_s, pack_infos):
    """Up-sampling alpha of the original NeuS: re-estimate the sdf at both ends of an interval from the mid value
    and the (clamped, non-increasing) slope, then take the cdf drop (neus_utils.py:164-188)."""
    d_sdf = packed_diff(sdf, pack_infos)
    d_t = packed_diff(depth_samples, pack_infos)
    mid = sdf + d_sdf * 0.5
    slope = d_sdf / (d_t + 1e-5)
    prev = slope.roll(1).index_fill_(0, pack_infos[:, 0], 0)
    slope = torch.minimum(prev, slope).clamp_(-10, 0)
    ends = torch.addcmul(mid.unsqueeze(-1).to(depth_samples.dtype), slope.unsqueeze(-1),
                         d_t.unsqueeze(-1) * d_t.new_tensor([-0.5, 0.5]))
    cdf = torch.sigmoid(ends * inv_s)
    return ((cdf[..., 0] - cdf[..., 1]) / (cdf[..., 0] + 1e-5)).clamp_min_(0)


@torch.no_grad()
def neus_ray_sdf_to_upsample_alpha(sdf, depth_samples, inv_s):
    d_sdf, d_t = sdf.diff(dim=-1), depth_samples.diff(dim=-1)
    mid = (sdf[..., :-1] + sdf[..., 1:]) * 0.5
    slope = d_sdf / (d_t + 1e-5)
    prev = torch.cat([slope.new_zeros([*slope.shape[:-1], 1]), slope[..., :-1]], -1)
    slope = torch.minimum(prev, slope).clamp_(-10.0, 0.0)
    ends = torch.addcmul(mid.unsqueeze(-1), slope.unsqueeze(-1), d_t.unsqueeze(-1) * d_t.new_tensor([-0.5, 0.5]))
    cdf = torch.sigmoid(ends * inv_s)
    return ((cdf[..., 0] - cdf[..., 1]) / (cdf[..., 0] + 1e-5)).clamp_min_(0)


# ---------------------------------------------------------------------------------------------------------------------
def _query_fused(model, ray_tested, view_dirs, rays_h_appear, *, perturb=False, with_rgb, with_normal, nablas_has_grad, forward_inv_s, num_coarse, march_cfg, num_fine,
                 upsample_inv_s, factors, use_estimate_alpha):
    """The query below with every stage between the big kernels as ONE launch (csrc/neus_glue.cu, csrc/neus_fused.cu) and three host
    reads in total (march size, compression size, + the ray test's): same samples, same values as the chain it replaces (with `perturb`,
    the same random stream too) -- the chain
    stays in this file as the specification (tests/test_neus_fused_gpu.py runs both).  None -> no ray marched into an occupied voxel
    (the caller falls back to the general path for that rare case)."""
    rays_o, rays_d, near, far, rays_inds = itemgetter("rays_o", "rays_d", "near", "far", "rays_inds")(ray_tested)
    dtype, n_stage = rays_o.dtype, len(factors)
    mc = dict(march_cfg)
    fac = mc.pop("step_size_factor", 1.0)
    mc["step_size"] = mc.get("step_size", 1e-3) * fac
    mc["dt_gamma"] = mc.get("dt_gamma", 0.0) * fac
    mc.setdefault("max_steps", 512)
    rays_o, rays_d = rays_o.contiguous(), rays_d.contiguous()
    depths_coarse_1 = batch_sample_step_linear(near, far, num_coarse + 1, prefix_shape=[rays_o.shape[0]], perturb=perturb)
    marched = neus_fused.march_lean(model.accel.occ.occ_grid, rays_o, rays_d, near.contiguous(), far.contiguous(), **mc)
    if marched is None:
        return None
    ridx_hit, pinfo_march, depth_samples, ridx = marched
    if perturb:
        # the single-grid marcher jitters only `deltas` (occgrid_raymarch.py:96-110), which this query never reads; the draw is made
        # anyway so that the random stream -- and therefore every later sample -- is the one the op-by-op chain consumes
        torch.rand(depth_samples.shape, dtype=depth_samples.dtype, device=depth_samples.device)
    pack_infos = pinfo_march
    coherent = bool(ray_tested.get("rays_coherent", False))      # image-ordered rays: ray-tiled traversal inside the SDF kernel
    surf = getattr(model, "implicit_surface", None)
    if use_persistent_upsample(rays_o.shape[0]) and not perturb and surf is not None and getattr(surf, "_fusable", lambda: False)():
        # the whole no-grad half in ONE persistent per-ray kernel (csrc/ray_upsample.cu); same values as the stage kernels below
        grid16, dec = surf._fused_state()
        accel = getattr(model, "accel", None)
        collect = accel.occ.collect_struct() if (model.training and accel is not None) else None
        fine_all, _overflow = neus_fused.upsample_rays(surf.encoding.meta, grid16, dec, ridx_hit, pack_infos, depth_samples, rays_o, rays_d,
                                                       [upsample_inv_s * f for f in factors], num_fine, max_level=surf._ml(getattr(model, "max_level", None)),
                                                       max_steps=mc["max_steps"], use_estimate_alpha=use_estimate_alpha, collect=collect)
        with torch.no_grad():
            d1, mid, ridx_all, pinfo = neus_fused.assemble_boundary(depths_coarse_1.contiguous(), ridx_hit, fine_all, run_len=list(num_fine))
        return _query_fused_tail(model, ray_tested, view_dirs, rays_h_appear, rays_o, rays_d, rays_inds, d1, mid, ridx_all, pinfo, pinfo_march, coherent, dtype,
                                 with_rgb=with_rgb, with_normal=with_normal, nablas_has_grad=nablas_has_grad, forward_inv_s=forward_inv_s)
    with torch.no_grad():
        # marched packs are ragged (20-100 samples per ray): tiles of 32 rays are padded to the longest and the samples of one ray are
        # already close together, so the ray-major order wins here (A/B switch MARCHED_TILED); the boundary and fine queries have
        # uniform packs and are ray-tiled whenever the rays are image-ordered
        tiled_m = coherent and MARCHED_TILED
        sdf = model.forward_sdf_on_rays(ridx, depth_samples, rays_o, rays_d, packs=(pack_infos, ridx_hit) if tiled_m else None)["sdf"].to(dtype)
        fine_stages = []
        for i, factor in enumerate(factors):
            cdf = neus_fused.upsample_cdf(sdf, depth_samples, pack_infos, upsample_inv_s * factor, use_estimate_alpha)
            if perturb:                  # one stratified u per pack and sample (raysample.py:38-61)
                fine = packed_sample_cdf(depth_samples, cdf, pack_infos, num_fine[i], perturb=True)[0]
            else:
                fine = neus_fused.sample_cdf_uniform(depth_samples, cdf, pack_infos, num_fine[i])
            fine_stages.append(fine)
            if i < n_stage - 1:         # (the reference also merges after the last stage; nothing reads that result)
                packs = (get_pack_infos_from_batch(ridx_hit.shape[0], fine.shape[1], device=fine.device), ridx_hit) if coherent else None
                sdf_fine = model.forward_sdf_on_rays(ridx_hit, fine, rays_o, rays_d, packs=packs)["sdf"].to(dtype).contiguous()
                depth_samples, sdf, pack_infos = neus_fused.merge_sorted_vals(depth_samples, sdf, pack_infos, fine, sdf_fine)
        fine_all = torch.cat(fine_stages, dim=-1) if n_stage > 1 else fine_stages[0]
        d1, mid, ridx_all, pinfo = neus_fused.assemble_boundary(depths_coarse_1.contiguous(), ridx_hit, fine_all.contiguous(), run_len=[f.shape[1] for f in fine_stages])
    return _query_fused_tail(model, ray_tested, view_dirs, rays_h_appear, rays_o, rays_d, rays_inds, d1, mid, ridx_all, pinfo, pinfo_march, coherent, dtype,
                             with_rgb=with_rgb, with_normal=with_normal, nablas_has_grad=nablas_has_grad, forward_inv_s=forward_inv_s)


def _query_fused_tail(model, ray_tested, view_dirs, rays_h_appear, rays_o, rays_d, rays_inds, d1, mid, ridx_all, pinfo, pinfo_march, coherent, dtype, *,
                      with_rgb, with_normal, nablas_has_grad, forward_inv_s):
    """boundary SDF (grad) -> alpha -> compression -> colour / normal query: the second half of `_query_fused`"""
    sdf_b = model.forward_sdf_on_rays(ridx_all, d1, rays_o, rays_d, packs=(pinfo, None) if coherent else None)["sdf"].to(dtype)
    comp = neus_fused.neus_alpha_compact(sdf_b, forward_inv_s, pinfo, ridx_all, mid, rays_inds)
    if comp is None:
        return dict(type="empty", rays_inds_hit=[]), {}
    volume_buffer = dict(type="packed", rays_inds_hit=comp["rays_inds_hit"], pack_infos_hit=comp["pack_infos"], t=comp["t"].to(dtype),
                         opacity_alpha=comp["alpha"].to(dtype))
    if with_rgb or with_normal:
        _net_forward_into(volume_buffer, model, rays_o, rays_d, view_dirs, rays_h_appear, comp["ridx"], comp["t"], nablas_has_grad=nablas_has_grad,
                          with_rgb=with_rgb, with_normal=with_normal, dtype=dtype)
    details = {"march.num_per_ray": pinfo_march[:, 1], "render.num_per_ray0": pinfo[:, 1], "render.num_per_ray": comp["pack_infos"][:, 1]}
    return volume_buffer, details


def _net_forward_into(volume_buffer, model, rays_o, rays_d, view_dirs, rays_h_appear, ridx_all, depths, *, nablas_has_grad,
                      with_rgb, with_normal, dtype, cond_kw=None):
    if view_dirs is None and cond_kw is None and not with_rgb and with_normal and FUSED_STAGES and getattr(model, "use_view_dirs", False) and not rays_d.requires_grad:
        # LiDAR-style rays (with_rgb=False, with_normal=True: code_single/tools/train.py:900): sdf + second-order nablas are what is needed; the
        # fused op computes them (its radiance head runs too and is dropped; no gradient reaches the radiance net)
        view_dirs = rays_d / rays_d.detach().norm(dim=-1).clamp_min(1.0e-10).unsqueeze(-1)
        if rays_h_appear is None and getattr(model, "use_h_appear", False):
            rays_h_appear = rays_d.new_zeros(rays_d.shape[0], model.radiance_net.blocks.layers[0].in_features - 54)
    if (FUSED_STAGES and cond_kw is None and (with_rgb or with_normal) and view_dirs is not None and getattr(model, "_color_fusable", lambda: False)()
            and not (rays_h_appear is not None and rays_h_appear.requires_grad) and not depths.requires_grad
            # learnable rays (pose refinement): the reference's model.forward(x = o + d t) carries d(loss)/d(rays); the fused op detaches them
            and not (rays_o.requires_grad or rays_d.requires_grad or view_dirs.requires_grad)):
        out = model.forward_on_rays(ridx_all, depths, rays_o, rays_d, view_dirs, rays_h_appear, nablas_has_grad=nablas_has_grad)
        volume_buffer["net_x"] = out["x"]
        volume_buffer["nablas"] = out["nablas"].to(dtype)
        if with_rgb:
            volume_buffer["rgb"] = out["rgb"].to(dtype)
        return
    x = torch.addcmul(rays_o[ridx_all], rays_d[ridx_all], depths.unsqueeze(-1))
    kw = dict(x=x, nablas_has_grad=nablas_has_grad, with_rgb=with_rgb, with_normal=with_normal)
    if rays_h_appear is not None:
        kw["h_appear"] = rays_h_appear[ridx_all]
    if view_dirs is not None:
        kw["v"] = view_dirs[ridx_all]
    if cond_kw is not None:
        kw.update(cond_kw(ridx_all))
    out = model.forward(**kw)
    volume_buffer["net_x"] = x
    if "nablas" in out:
        volume_buffer["nablas"] = out["nablas"].to(dtype)
    if "rgb" in out:
        volume_buffer["rgb"] = out["rgb"].to(dtype)


def neus_ray_query_march_occ_multi_upsample_compressed(
        model, ray_tested, with_rgb=True, with_normal=True, perturb=False, nablas_has_grad=False, forward_inv_s=None,
        num_coarse=0, coarse_step_cfg=dict(step_mode="linear"), chunksize_query=2 ** 24, march_cfg=dict(), num_fine=8,
        upsample_inv_s=64., upsample_s_divisor=1.0, upsample_inv_s_factors=(1, 4, 16), upsample_use_estimate_alpha=False):
    """Occupancy-grid march -> multi-stage NeuS up-sampling -> (optional coarse samples) -> SDF with grad -> alpha ->
    sample compression -> colour / normal query.  See the module docstring for the contract."""
    empty = dict(type="empty", rays_inds_hit=[])
    if ray_tested["num_rays"] == 0:
        return empty, {}
    use_h_appear = getattr(model, "use_h_appear", False) and with_rgb
    use_view_dirs = getattr(model, "use_view_dirs", False) and with_rgb
    n_stage = len(upsample_inv_s_factors)
    if isinstance(num_fine, int):
        num_fine = [num_fine] * n_stage
    assert len(num_fine) == n_stage, f"num_fine should be of the same length={n_stage} with upsample"
    num_fine = [n // 2 * 2 + 1 for n in num_fine]
    upsample_inv_s = upsample_inv_s / upsample_s_divisor
    forward_inv_s = model.forward_inv_s() if forward_inv_s is None else forward_inv_s
    step_mode = coarse_step_cfg.get("step_mode", "linear")
    if num_coarse > 0 and step_mode != "linear":
        raise RuntimeError(f"coarse step_mode={step_mode!r} is not built (CFG uses 'linear')")

    rays_o, rays_d, near, far, rays_inds = itemgetter("rays_o", "rays_d", "near", "far", "rays_inds")(ray_tested)
    rays_h_appear = ray_tested["rays_h_appear"] if use_h_appear else None
    device, dtype = rays_o.device, rays_o.dtype
    R = rays_o.shape[0]
    dir_scale = rays_d.detach().norm(dim=-1)
    view_dirs = rays_d / dir_scale.clamp_min(1.0e-10).unsqueeze(-1) if use_view_dirs else None

    # conditioned field families (dynamic / generative models) take per-ray ts / fidx / bidx / pix with every network query
    # (neus_ray_query.py:776-790, 846-866); they run the op-by-op chain below, the values gathered per sample
    cond = {k: ray_tested[f"rays_{k}"] for k in ("ts", "fidx", "bidx", "pix") if getattr(model, f"use_{k}", False) and ray_tested.get(f"rays_{k}") is not None}
    cond_kw = (lambda ridx_: {k: v[ridx_] for k, v in cond.items()}) if cond else (lambda ridx_: {})

    def sdf_on_rays(ridx_, t_):
        if not cond:
            return model.forward_sdf_on_rays(ridx_, t_, rays_o, rays_d)["sdf"]
        r2 = ridx_.unsqueeze(-1).expand(t_.shape) if t_.dim() == 2 else ridx_
        x_ = torch.addcmul(rays_o[r2], rays_d[r2], t_.unsqueeze(-1))
        return model.forward_sdf(x_.flatten(0, -2), **cond_kw(r2.reshape(-1)))["sdf"].view(t_.shape)

    if (FUSED_STAGES and not cond and num_coarse > 0 and rays_o.is_cuda and dtype == torch.float32 and hasattr(model, "forward_sdf_on_rays")
            and getattr(getattr(model.accel, "occ", None), "occ_grid", None) is not None and model.accel.occ.occ_grid.dim() == 3
            and not (rays_o.requires_grad or rays_d.requires_grad or near.requires_grad or far.requires_grad)
            and set(march_cfg) <= {"step_size", "max_steps", "max_step_size", "dt_gamma", "step_size_factor"}):
        ret = _query_fused(model, ray_tested, view_dirs, rays_h_appear, perturb=perturb, with_rgb=with_rgb, with_normal=with_normal, nablas_has_grad=nablas_has_grad,
                           forward_inv_s=forward_inv_s, num_coarse=num_coarse, march_cfg=march_cfg, num_fine=num_fine, upsample_inv_s=upsample_inv_s,
                           factors=upsample_inv_s_factors, use_estimate_alpha=upsample_use_estimate_alpha)
        if ret is not None:
            return ret

    if num_coarse > 0:
        depths_coarse_1, deltas_coarse_1 = batch_sample_step_linear(near, far, num_coarse + 1, perturb=perturb, return_dt=True)
    marched = model.accel.ray_march(rays_o, rays_d, near=near, far=far, perturb=perturb, **march_cfg)
    net_kw = dict(nablas_has_grad=nablas_has_grad, with_rgb=with_rgb, with_normal=with_normal, dtype=dtype, cond_kw=cond_kw if cond else None)

    if marched.ridx_hit is not None:
        # ---------------- up-sample on the marched samples (no grad)
        pack_infos = marched.pack_infos.clone()
        depth_samples = marched.depth_samples
        n_hit = marched.num_hit_rays
        rays_inds_hit = rays_inds[marched.ridx_hit]
        with torch.no_grad():
            sdf = model.forward_sdf(marched.samples, **cond_kw(marched.ridx))["sdf"].to(dtype)
            fine_stages = []
            for i, factor in enumerate(upsample_inv_s_factors):
                if FUSED_STAGES:
                    cdf = neus_fused.upsample_cdf(sdf, depth_samples, pack_infos, upsample_inv_s * factor, upsample_use_estimate_alpha)
                else:
                    if upsample_use_estimate_alpha:
                        alpha = neus_packed_sdf_to_upsample_alpha(sdf, depth_samples, upsample_inv_s * factor, pack_infos)
                    else:
                        alpha = neus_packed_sdf_to_alpha(sdf, upsample_inv_s * factor, pack_infos)
                    vw = packed_alpha_to_vw(alpha, pack_infos)
                    cdf = packed_cumsum(vw, pack_infos, exclusive=True)
                    norm = cdf[pack_infos[:, 0] + pack_infos[:, 1] - 1].clamp_min(1e-5)
                    cdf = packed_div(cdf, norm, pack_infos)
                if FUSED_STAGES and not perturb:
                    fine = neus_fused.sample_cdf_uniform(depth_samples, cdf, pack_infos, num_fine[i])
                else:
                    fine = packed_sample_cdf(depth_samples, cdf, pack_infos, num_fine[i], perturb=perturb)[0]
                fine_stages.append(fine)
                if n_stage > 1:
                    pinfo_fine = get_pack_infos_from_batch(n_hit, num_fine[i], device=device)
                    pidx0, pidx1, pack_infos = merge_two_packs_sorted_aligned(depth_samples, pack_infos, fine.flatten(), pinfo_fine, b_sorted=True)
                    n_old = depth_samples.numel()
                    merged = depth_samples.new_empty([n_old + fine.numel()])
                    merged[pidx0], merged[pidx1] = depth_samples, fine.flatten()
                    depth_samples = merged
                    if i < n_stage - 1:
                        sdf_fine = sdf_on_rays(marched.ridx_hit, fine).to(dtype)
                        sdf_new = sdf.new_empty([n_old + fine.numel()])
                        sdf_new[pidx0], sdf_new[pidx1] = sdf, sdf_fine.flatten()
                        sdf = sdf_new
            depths_1 = torch.cat(fine_stages, dim=-1).sort(dim=-1).values if n_stage > 1 else fine_stages[0]

        # ---------------- boundary points with grad, alpha, compression
        if num_coarse == 0:
            x = torch.addcmul(rays_o[marched.ridx_hit].unsqueeze(-2), rays_d[marched.ridx_hit].unsqueeze(-2), depths_1.unsqueeze(-1))
            alpha = neus_ray_sdf_to_alpha(sdf_on_rays(marched.ridx_hit, depths_1).to(dtype) if cond else
                                          model.forward_sdf(x.flatten(0, -2))["sdf"].to(dtype).view(depths_1.shape), forward_inv_s)
            depths = depths_1[..., :-1] + depths_1.diff(dim=-1) / 2.
            pack_infos = get_pack_infos_from_batch(n_hit, depths.size(-1), device=device)
            nidx_useful, pack_infos_useful, pidx_useful = packed_volume_render_compression(alpha.flatten(), pack_infos)
            if nidx_useful.numel() == 0:
                return empty, {}
            depths_packed, alpha_packed = depths.flatten()[pidx_useful], alpha.flatten()[pidx_useful]
            volume_buffer = dict(type="packed", rays_inds_hit=rays_inds_hit[nidx_useful], pack_infos_hit=pack_infos_useful,
                                 t=depths_packed.to(dtype), opacity_alpha=alpha_packed.to(dtype))
            if with_rgb or with_normal:
                ridx_all = marched.ridx_hit.unsqueeze(-1).expand(n_hit, depths.size(-1)).flatten()[pidx_useful]
                _net_forward_into(volume_buffer, model, rays_o, rays_d, view_dirs, rays_h_appear, ridx_all, depths_packed, **net_kw)
            details = {"march.num_per_ray": marched.pack_infos[:, 1], "render.num_per_ray0": depths.size(-1),
                       "render.num_per_ray": pack_infos_useful[:, 1]}
            return volume_buffer, details

        ridx_coarse = torch.arange(R, device=device)
        pidx0, pidx1, pack_infos = merge_two_batch_a_includes_b(depths_coarse_1, ridx_coarse, depths_1, marched.ridx_hit, a_sorted=True)
        S = depths_1.numel() + depths_coarse_1.numel()
        depths_1_packed = depths_1.new_zeros([S])
        ridx_all = marched.ridx_hit.new_zeros([S])
        ridx_all[pidx0], ridx_all[pidx1] = ridx_coarse.unsqueeze(-1), marched.ridx_hit.unsqueeze(-1)
        depths_1_packed[pidx0], depths_1_packed[pidx1] = depths_coarse_1, depths_1
        depths_packed = depths_1_packed + packed_diff(depths_1_packed, pack_infos) / 2.
        sdf_b = sdf_on_rays(ridx_all, depths_1_packed).to(dtype)
        if FUSED_STAGES:
            alpha_packed, nidx_useful, pack_infos_useful, pidx_useful = neus_fused.neus_alpha_compress(sdf_b, forward_inv_s, pack_infos)
        else:
            alpha_packed = neus_packed_sdf_to_alpha(sdf_b, forward_inv_s, pack_infos)
            nidx_useful, pack_infos_useful, pidx_useful = packed_volume_render_compression(alpha_packed, pack_infos)
        if nidx_useful.numel() == 0:
            return empty, {}
        ridx_all, depths_packed, alpha_packed = ridx_all[pidx_useful], depths_packed[pidx_useful], alpha_packed[pidx_useful]
        volume_buffer = dict(type="packed", rays_inds_hit=rays_inds[nidx_useful], pack_infos_hit=pack_infos_useful,
                             t=depths_packed.to(dtype), opacity_alpha=alpha_packed.to(dtype))
        if with_rgb or with_normal:
            _net_forward_into(volume_buffer, model, rays_o, rays_d, view_dirs, rays_h_appear, ridx_all, depths_packed, **net_kw)
        details = {"march.num_per_ray": marched.pack_infos[:, 1], "render.num_per_ray0": pack_infos[:, 1],
                   "render.num_per_ray": pack_infos_useful[:, 1]}
        return volume_buffer, details

    # ---------------- no ray hit the occupancy grid
    if num_coarse == 0:
        return empty, {}
    x = torch.addcmul(rays_o.unsqueeze(-2), rays_d.unsqueeze(-2), depths_coarse_1.unsqueeze(-1))
    sdf_c = (sdf_on_rays(torch.arange(R, device=device), depths_coarse_1) if cond else model.forward_sdf(x.flatten(0, -2))["sdf"].view(depths_coarse_1.shape)).to(dtype)
    alpha_coarse = neus_ray_sdf_to_alpha(sdf_c, forward_inv_s)
    depths_coarse = depths_coarse_1[..., :num_coarse] + deltas_coarse_1[..., :num_coarse] / 2.
    pack_infos_coarse = get_pack_infos_from_batch(R, num_coarse, device=device)
    nidx_useful, pack_infos_useful, pidx_useful = packed_volume_render_compression(alpha_coarse.flatten(), pack_infos_coarse)
    if nidx_useful.numel() == 0:
        return empty, {}
    depths_packed, alpha_packed = depths_coarse.flatten()[pidx_useful], alpha_coarse.flatten()[pidx_useful]
    volume_buffer = dict(type="packed", rays_inds_hit=rays_inds[nidx_useful], pack_infos_hit=pack_infos_useful,
                         t=depths_packed.to(dtype), opacity_alpha=alpha_packed.to(dtype))
    if with_rgb or with_normal:
        ridx_all = torch.arange(R, device=device).unsqueeze(-1).expand_as(depths_coarse).flatten()[pidx_useful]
        _net_forward_into(volume_buffer, model, rays_o, rays_d, view_dirs, rays_h_appear, ridx_all, depths_packed, **net_kw)
    return volume_buffer, {"render.num_per_ray0": depths_coarse.size(-1), "render.num_per_ray": pack_infos_useful[:, 1]}
