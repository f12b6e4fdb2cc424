"""CPU restatement of the per-ray NeuS rendering path (Python/PyTorch layer of the reference).
TEST INFRASTRUCTURE.

Follows (paths relative to the reference project):
  ray test          nr3d_lib/nr3d_lib/models/spatial/aabb.py:85-99, graphics/raytest.py:162-167
  coarse sampling   nr3d_lib/nr3d_lib/graphics/raysample.py:285-310 (batch_sample_step_linear)
  fine sampling     nr3d_lib/nr3d_lib/graphics/raysample.py:38-61 (packed_sample_cdf)
  march wrapper     nr3d_lib/nr3d_lib/graphics/raymarch/occgrid_raymarch.py:25-112
  NeuS maths        nr3d_lib/nr3d_lib/graphics/neus/neus_utils.py:88-111,164-188
  pack helpers      nr3d_lib/nr3d_lib/graphics/pack_ops/pack_ops.py:97-291,529-747
  orchestration     nr3d_lib/nr3d_lib/graphics/neus/neus_ray_query.py:732-1104
  integration       app/renderers/single_volume_renderer.py:73-102

Float ops are differentiable torch (fp32); integer/index ops come from oracle.pack_ops / oracle.march.
"""
from __future__ import annotations

import torch

from . import pack_ops as opk
from . import march as omarch
from . import nets as onets


# ------------------------------------------------------------------ pack_infos helpers (pack_ops.py:725-747)
def get_pack_infos_from_n(n):
    return torch.stack([n.cumsum(0) - n, n], 1)


def get_pack_infos_from_batch(num, size):
    return torch.stack([torch.arange(0, num * size, size, dtype=torch.long), torch.full([num], size, dtype=torch.long)], 1)


def _pack_index(pack_infos):
    return torch.repeat_interleave(torch.arange(pack_infos.shape[0]), pack_infos[:, 1])


# ------------------------------------------------------------------ differentiable pack ops (pack_ops.py:97-392)
def packed_sum(feats, pack_infos):
    out = feats.new_zeros((pack_infos.shape[0],) + feats.shape[1:])
    return out.index_add(0, _pack_index(pack_infos), feats)


def packed_div(feats, other, pack_infos):
    o = torch.repeat_interleave(other, pack_infos[:, 1], dim=0)
    return feats / o


def packed_diff(feats, pack_infos, pack_appends=None):
    """out[i] = f[i+1]-f[i]; pack tail = append - f[last] or 0 (pack_ops.py:189-224, kernel :1099-1142)."""
    last = pack_infos[:, 0] + pack_infos[:, 1] - 1
    nxt = torch.roll(feats, -1, 0)
    if pack_appends is not None:
        nxt = nxt.index_copy(0, last, pack_appends)
        return nxt - feats
    is_last = torch.zeros(feats.shape[0], dtype=torch.bool)
    is_last[last] = True
    d = nxt - feats
    return torch.where(is_last.view(-1, *([1] * (feats.dim() - 1))), torch.zeros_like(d), d)


def packed_cumsum_exclusive(feats, pack_infos):
    return opk.packed_cumsum(feats, pack_infos, True, False)


class _PackedAlphaToVW(torch.autograd.Function):
    """pack_ops.py:254-279 over the nerfacc-derived kernels."""

    @staticmethod
    def forward(ctx, alphas, pack_infos, eps, thre):
        w = opk.packed_alpha_to_vw_forward(alphas.detach(), pack_infos, eps, thre, False)[0]
        ctx.save_for_backward(alphas.detach(), pack_infos, w)
        ctx.cfg = (eps, thre)
        return w

    @staticmethod
    def backward(ctx, gw):
        alphas, pack_infos, w = ctx.saved_tensors
        ga = opk.packed_alpha_to_vw_backward(w, gw.contiguous(), alphas, pack_infos, *ctx.cfg)
        return ga, None, None, None


def packed_alpha_to_vw(alpha, pack_infos, early_stop_eps=1e-4, alpha_thre=0.0):
    if alpha.requires_grad:
        return _PackedAlphaToVW.apply(alpha, pack_infos, early_stop_eps, alpha_thre)
    return opk.packed_alpha_to_vw_forward(alpha, pack_infos, early_stop_eps, alpha_thre, False)[0]


def packed_volume_render_compression(alpha, pack_infos, early_stop_eps=1e-4, alpha_thre=0.0):
    """pack_ops.py:286-291."""
    _, info, sel = opk.packed_alpha_to_vw_forward(alpha.detach(), pack_infos, early_stop_eps, alpha_thre, True)
    pidx = sel.nonzero()[:, 0]
    nidx = (info[:, 1] > 0).nonzero()[:, 0]
    return nidx, info[nidx].long(), pidx


def merge_two_batch_a_includes_b(vals_a, nidx_a, vals_b, nidx_b):
    """pack_ops.py:669-720 (a_sorted=True, return_val=False)."""
    n_a, bds_a, bds_b = nidx_a.numel(), vals_a.shape[-1], vals_b.shape[-1]
    if n_a == nidx_b.numel() and torch.equal(nidx_a, nidx_b):
        order = torch.cat([vals_a, vals_b], -1).sort(dim=-1, stable=True).indices
        rank = order.argsort(-1)
        pack_infos = get_pack_infos_from_n(torch.full([n_a], bds_a + bds_b, dtype=torch.long))
        first = pack_infos[:, 0:1]
        return first + rank[:, :bds_a], first + rank[:, bds_a:], pack_infos
    where_b = torch.searchsorted(nidx_a, nidx_b)
    n_per = torch.full([n_a], bds_a, dtype=torch.long)
    n_per[where_b] = bds_a + bds_b
    pack_infos = get_pack_infos_from_n(n_per)
    first = pack_infos[:, 0:1]
    pidx_a = first + torch.arange(bds_a)[None, :]
    rank = torch.cat([vals_a[where_b], vals_b], 1).sort(dim=-1, stable=True).indices.argsort(-1)
    pidx_a[where_b] = first[where_b] + rank[:, :bds_a]
    pidx_b = first[where_b] + rank[:, bds_a:]
    return pidx_a, pidx_b, pack_infos


# ------------------------------------------------------------------ samplers
def batch_sample_step_linear(near, far, num, perturb=False, generator=None):
    """raysample.py:285-310 -> (t [R,num], deltas [R,num])."""
    near, far = near.view(-1, 1), far.view(-1, 1)
    if not perturb:
        dt = (far - near) / (num - 1)
        t = torch.addcmul(near, torch.arange(num).to(near.dtype), dt)
        return t, dt.expand(-1, num)
    idx = torch.arange(num) + torch.rand([near.shape[0], num], generator=generator, dtype=near.dtype)
    dt = (far - near) / num
    t = torch.addcmul(near, idx.to(near.dtype), dt)
    deltas = torch.zeros_like(t)
    deltas[:, :-1], deltas[:, -1] = t.diff(dim=-1), (far[:, 0] - near[:, 0]) / num
    return t, deltas


def packed_sample_cdf(bins, cdfs, pack_infos, num, perturb=False, generator=None):
    """raysample.py:38-61."""
    P = pack_infos.shape[0]
    if not perturb:
        u = torch.linspace(0., 1., num + 2, dtype=bins.dtype)[1:-1].expand(P, num)
    else:
        u = batch_sample_step_linear(bins.new_zeros(P), bins.new_ones(P), num, True, generator)[0]
    return opk.packed_invert_cdf(bins, cdfs.to(bins.dtype), u.contiguous(), pack_infos)


# ------------------------------------------------------------------ ray test (aabb.py:85-99)
def ray_test(rays_o, rays_d, near=None, far=None):
    with torch.no_grad():
        t0 = (-1. - rays_o) / rays_d
        t1 = (1. - rays_o) / rays_d
        near_ = torch.minimum(t0, t1).max(-1).values
        far_ = torch.maximum(t0, t1).min(-1).values
        if near is not None:
            near_.clamp_min_(near)
        if far is not None:
            far_.clamp_max_(far)
        mask = (far_ > near_) & (far_ > (0 if near is None else near))
        if far is not None:
            mask &= near_ < far
        ridx = mask.nonzero()[:, 0]
    return dict(num_rays=ridx.shape[0], rays_inds=ridx, near=near_[ridx], far=far_[ridx],
                rays_o=rays_o[ridx], rays_d=rays_d[ridx])


# ------------------------------------------------------------------ NeuS maths (neus_utils.py)
def neus_packed_sdf_to_alpha(sdf, inv_s, pack_infos):
    """neus_utils.py:88-111: cdf=sigmoid(sdf*inv_s); alpha_i = max(0, (cdf_i - cdf_{i+1}) / (cdf_i + 1e-5)), tail 0."""
    cdf = torch.sigmoid(sdf * inv_s)
    return ((-1 * packed_diff(cdf, pack_infos)) / (cdf + 1e-5)).clamp_min(0)


@torch.no_grad()
def neus_packed_sdf_to_upsample_alpha(sdf, depth, inv_s, pack_infos):
    """neus_utils.py:164-188."""
    sdf_diff = packed_diff(sdf, pack_infos)
    deltas = packed_diff(depth, pack_infos)
    mid = sdf + sdf_diff * 0.5
    dot = sdf_diff / (deltas + 1e-5)
    prev = dot.roll(1).index_fill_(0, pack_infos[:, 0], 0)
    dot = torch.minimum(prev, dot).clamp_(-10, 0)
    est = torch.addcmul(mid.unsqueeze(-1).to(depth.dtype), dot.unsqueeze(-1),
                        deltas.unsqueeze(-1) * deltas.new_tensor([-0.5, 0.5]))
    cdf = torch.sigmoid(est * inv_s)
    return ((cdf[..., 0] - cdf[..., 1]) / (cdf[..., 0] + 1e-5)).clamp_min_(0)


# ------------------------------------------------------------------ march wrapper (occgrid_raymarch.py:25-112)
class Marched:
    pass


def occgrid_raymarch(occ_grid, rays_o, rays_d, near, far, step_size, max_steps, perturb=False, generator=None,
                     max_step_size=1e10, dt_gamma=0.0):
    roi = torch.tensor([-1., -1, -1, 1, 1, 1])
    info, t0, t1, ridx, gidx = omarch.ray_marching(rays_o, rays_d, near, far, roi, occ_grid, step_size,
                                                   max_step_size, dt_gamma, max_steps)
    m = Marched()
    hit = info[:, 1].nonzero()[:, 0]
    m.num_hit_rays = hit.numel()
    if hit.numel() == 0:
        m.ridx_hit = None
        return m
    m.ridx_hit = hit
    m.pack_infos = info[hit].long()
    m.ridx, m.gidx = ridx.long(), gidx.long()
    deltas = t1 - t0
    if perturb:   # only `deltas` are perturbed for the single-grid variant (:96-106, depth stays t_starts)
        noise = torch.rand(deltas.shape, generator=generator, dtype=deltas.dtype)
        deltas = packed_diff(torch.addcmul(t0, noise, deltas), m.pack_infos)
    m.deltas = deltas
    m.depth_samples = t0
    m.samples = torch.addcmul(rays_o[m.ridx], rays_d[m.ridx], t0.unsqueeze(-1))
    return m


# ------------------------------------------------------------------ orchestration (neus_ray_query.py:732-1104)
def neus_ray_query(P: onets.LoTDNeuSParams, occ_grid, ray_tested, *, with_rgb=True, with_normal=True, perturb=False,
                   nablas_has_grad=True, forward_inv_s=None, num_coarse=64, num_fine=(8, 8, 32), step_size=0.005,
                   max_steps=4096, upsample_inv_s=64., upsample_s_divisor=1.0, upsample_inv_s_factors=(1, 4, 16),
                   upsample_use_estimate_alpha=True, rays_h_appear=None, generator=None):
    """`neus_ray_query_march_occ_multi_upsample_compressed` for the num_coarse>0 configuration of CFG."""
    empty = dict(type="empty", rays_inds_hit=[])
    if ray_tested["num_rays"] == 0:
        return empty, {}
    assert num_coarse > 0, "oracle restates the num_coarse>0 branches (CFG: num_coarse=64)"
    num_fine = [n // 2 * 2 + 1 for n in num_fine]
    upsample_inv_s = upsample_inv_s / upsample_s_divisor
    inv_s = P.forward_inv_s() if forward_inv_s is None else forward_inv_s
    rays_o, rays_d, near, far, rays_inds = (ray_tested[k] for k in ("rays_o", "rays_d", "near", "far", "rays_inds"))
    R = rays_o.shape[0]
    dir_scale = rays_d.detach().norm(dim=-1)
    view_dirs = rays_d / dir_scale.clamp_min(1.0e-10).unsqueeze(-1)

    depths_coarse_1, _ = batch_sample_step_linear(near, far, num_coarse + 1, perturb, generator)
    marched = occgrid_raymarch(occ_grid, rays_o, rays_d, near, far, step_size, max_steps, perturb, generator)
    ridx_coarse = torch.arange(R)

    if marched.ridx_hit is not None:
        pack_infos = marched.pack_infos.clone()
        depth_samples = marched.depth_samples
        o_hit = rays_o[marched.ridx_hit].unsqueeze(-2)
        d_hit = rays_d[marched.ridx_hit].unsqueeze(-2)
        with torch.no_grad():
            sdf = onets.forward_sdf(P, marched.samples)["sdf"]
            depths_1 = []
            for i, factor in enumerate(upsample_inv_s_factors):
                pinfo_fine = get_pack_infos_from_batch(marched.num_hit_rays, num_fine[i])
                if upsample_use_estimate_alpha:
                    alpha = neus_packed_sdf_to_upsample_alpha(sdf, depth_samples, upsample_inv_s * factor, pack_infos)
                else:
                    alpha = neus_packed_sdf_to_alpha(sdf, upsample_inv_s * factor, pack_infos)
                vw = packed_alpha_to_vw(alpha, pack_infos)
                cdf = packed_cumsum_exclusive(vw, pack_infos)
                last = cdf[pack_infos[:, 0] + pack_infos[:, 1] - 1]
                cdf = packed_div(cdf, last.clamp_min(1e-5), pack_infos)
                fine = packed_sample_cdf(depth_samples, cdf.to(depth_samples.dtype), pack_infos, num_fine[i], perturb, generator)[0]
                depths_1.append(fine)
                if len(upsample_inv_s_factors) > 1:
                    pidx0, pidx1, pack_infos = opk.try_merge_two_packs_sorted_aligned(
                        depth_samples, pack_infos, fine.flatten(), pinfo_fine, True)
                    n_old = depth_samples.numel()
                    merged = depth_samples.new_empty([n_old + fine.numel()])
                    merged[pidx0], merged[pidx1] = depth_samples, fine.flatten()
                    depth_samples = merged
                    if i < len(upsample_inv_s_factors) - 1:
                        x_fine = torch.addcmul(o_hit, d_hit, fine.unsqueeze(-1))
                        sdf_new = sdf.new_empty([n_old + fine.numel()])
                        sdf_new[pidx0], sdf_new[pidx1] = sdf, onets.forward_sdf(P, x_fine.flatten(0, -2))["sdf"]
                        sdf = sdf_new
            depths_1 = torch.cat(depths_1, -1).sort(-1).values if len(upsample_inv_s_factors) > 1 else depths_1[0]

        pidx0, pidx1, pack_infos = merge_two_batch_a_includes_b(depths_coarse_1, ridx_coarse, depths_1, marched.ridx_hit)
        S = depths_1.numel() + depths_coarse_1.numel()
        depths_1_packed = depths_1.new_zeros([S])
        ridx_all = torch.zeros([S], dtype=torch.long)
        ridx_all[pidx0], ridx_all[pidx1] = ridx_coarse.unsqueeze(-1).expand_as(pidx0), marched.ridx_hit.unsqueeze(-1).expand_as(pidx1)
        depths_1_packed[pidx0], depths_1_packed[pidx1] = depths_coarse_1, depths_1
        details = {"march.num_per_ray": marched.pack_infos[:, 1]}
    else:
        pack_infos = get_pack_infos_from_batch(R, num_coarse + 1)
        depths_1_packed = depths_coarse_1.flatten()
        ridx_all = ridx_coarse.unsqueeze(-1).expand(R, num_coarse + 1).flatten()
        details = {}
        # NOTE neus_ray_query.py:1048-1104 composes this branch with batched ops (alpha over [R,65], mid depths
        # from the first 64 boundaries); the packed formulation here is the same arithmetic.

    depths_packed = depths_1_packed + packed_diff(depths_1_packed, pack_infos) / 2.
    x_bound = torch.addcmul(rays_o[ridx_all], rays_d[ridx_all], depths_1_packed.unsqueeze(-1))
    sdf_bound = onets.forward_sdf(P, x_bound)["sdf"]
    alpha_packed = neus_packed_sdf_to_alpha(sdf_bound, inv_s, pack_infos)
    nidx_useful, pack_infos_useful, pidx_useful = packed_volume_render_compression(alpha_packed, pack_infos)
    details["render.num_per_ray0"] = pack_infos[:, 1]
    if nidx_useful.numel() == 0:
        return empty, {}
    ridx_all, depths_packed, alpha_packed = ridx_all[pidx_useful], depths_packed[pidx_useful], alpha_packed[pidx_useful]
    vb = dict(type="packed", rays_inds_hit=rays_inds[nidx_useful], pack_infos_hit=pack_infos_useful,
              t=depths_packed, opacity_alpha=alpha_packed, ridx=ridx_all)
    if with_rgb or with_normal:
        x = torch.addcmul(rays_o[ridx_all], rays_d[ridx_all], depths_packed.unsqueeze(-1))
        ha = None if rays_h_appear is None else rays_h_appear[ridx_all]
        out = onets.forward(P, x, view_dirs[ridx_all], ha, nablas_has_grad=nablas_has_grad)
        vb["net_x"] = x
        vb["nablas"] = out["nablas"]
        vb["sdf"] = out["sdf"]
        if with_rgb:
            vb["rgb"] = out["rgb"]
    details["render.num_per_ray"] = pack_infos_useful[:, 1]
    return vb, details


# ------------------------------------------------------------------ volume integration (single_volume_renderer.py:73-102)
def volume_integration(vb, num_rays, training=True, depth_use_normalized_vw=True):
    out = dict(mask_volume=torch.zeros(num_rays), depth_volume=torch.zeros(num_rays),
               rgb_volume=torch.zeros(num_rays, 3), normals_volume=torch.zeros(num_rays, 3))
    if vb["type"] == "empty":
        return out
    pi, hit = vb["pack_infos_hit"], vb["rays_inds_hit"]
    vw = packed_alpha_to_vw(vb["opacity_alpha"], pi)
    vb["vw"] = vw
    vw_sum = packed_sum(vw, pi)
    depth_w = packed_div(vw, vw_sum + 1e-10, pi) if depth_use_normalized_vw else vw
    out["mask_volume"] = out["mask_volume"].index_put((hit,), vw_sum)
    out["depth_volume"] = out["depth_volume"].index_put((hit,), packed_sum(depth_w * vb["t"], pi))
    if "rgb" in vb:
        out["rgb_volume"] = out["rgb_volume"].index_put((hit,), packed_sum(vw[:, None] * vb["rgb"], pi))
    if "nablas" in vb:
        nab = vb["nablas"] if training else torch.nn.functional.normalize(vb["nablas"].clamp(-1, 1), dim=-1)
        out["normals_volume"] = out["normals_volume"].index_put((hit,), packed_sum(vw[:, None] * nab, pi))
    return out
