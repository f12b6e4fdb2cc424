"""LoTDNeuS field + NeuS renderer mixin -- API of `nr3d_lib.models.fields.neus.LoTDNeuS / LoTDNeuSModel`
(reference: nr3d_lib/nr3d_lib/models/fields/neus/lotd_neus.py:27-232, renderer_mixin.py:40-440).

State-dict names follow the reference so checkpoints keep loading (SURVEY.md §9):
  implicit_surface.encoding.flattened_params, implicit_surface.decoder.layers.{0,1}.{weight,bias},
  radiance_net.blocks.layers.{0,1,2}.{weight,bias}, ctrl_var.ln_inv_s, accel.occ.{is_initialized,occ_grid,occ_val_grid}.
A geometry-only model (`radiance_cfg=False`, the reference's `radiance_cfg: null`) has no `radiance_net.*` keys.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..graphics import neus as neus_graphics, neus_fused
from ..graphics.neus import neus_ray_query_march_occ_multi_upsample_compressed
from ..graphics.nerf import packed_alpha_to_vw, ray_alpha_to_vw
from ..graphics.pack_ops import packed_div, packed_sum
from .accel import OccGridAccel
from .fused_color import color_net_c, fused_color
from .networks import LoTDSDF, RadianceNet, VarSingleMixLinear
from .space import AABBSpace


class _Cfg(dict):
    """dict with attribute access (the reference passes addict/ConfigDict objects)."""
    __getattr__ = dict.get


class LoTDNeuS(nn.Module):
    """radiance_cfg: a dict of RadianceNet arguments over the defaults; None builds the default radiance net; False builds none -- a
    geometry-only model (the reference's `radiance_cfg: null`, lotd_neus.py:71-85, e.g. the LiDAR-only StreetSurf configuration): then
    `radiance_net` is None, use_view_dirs = use_nablas = use_h_appear = False, and only sdf / nablas can be queried."""

    def __init__(self, surface_cfg: dict = None, radiance_cfg=None, var_ctrl_cfg: dict = None, dtype=torch.half, device=None,
                 generator=None, n_appear_embedding: int = None):
        super().__init__()
        self.dtype = dtype
        sc = dict(surface_cfg or {})
        bounding_size = sc.pop("bounding_size", 2.0)
        aabb = sc.pop("aabb", None)                      # a cuboid space (street scenes: LoTDNeuSStreet, `lotd_use_cuboid`)
        self.space = AABBSpace(bounding_size, aabb=aabb, device=device)
        self.implicit_surface = LoTDSDF(encoding_cfg=sc.get("encoding_cfg"), decoder_cfg=sc.get("decoder_cfg"), dtype=dtype, device=device,
                                        generator=generator, sdf_scale=sc.get("sdf_scale", 1.0), aabb=self.space.aabb.cpu(),
                                        radius3d_original=(self.space.radius3d_original.cpu() if aabb is not None else bounding_size / 2.),
                                        max_fused_levels=sc.get("max_fused_levels", 16))
        if radiance_cfg is False:
            self.radiance_net = None
        else:
            rc = dict(use_pos=True, use_view_dirs=True, use_nablas=True, D=2, W=64)
            rc.update(radiance_cfg or {})
            if n_appear_embedding is not None:
                rc["n_appear_embedding"] = n_appear_embedding
            self.radiance_net = RadianceNet(n_extra_feat=self.implicit_surface.encoding.out_features, dtype=dtype, device=device, generator=generator, **rc)
        vc = dict(ln_inv_s_init=0.3, ln_inv_s_factor=10.0, stop_it=1, start_it=0, final_inv_s=2048.)
        vc.update({k: v for k, v in (var_ctrl_cfg or {}).items() if k != "ctrl_type"})
        self.ctrl_var = VarSingleMixLinear(**vc, device=device)
        r = self.radiance_net
        self.use_view_dirs = r is not None and r.use_view_dirs
        self.use_nablas = r is not None and r.use_nablas
        self.use_h_appear = r is not None and r.use_h_appear
        self.max_level = None

    @property
    def device(self):
        return self.implicit_surface.encoding.flattened_params.device

    def forward_inv_s(self):
        return self.ctrl_var()

    def forward_sdf(self, x, *, return_h=False):
        if return_h:
            return self.implicit_surface(x, return_h=True, max_level=self.max_level)
        return self.implicit_surface.forward_sdf(x, max_level=self.max_level)

    def forward_sdf_on_rays(self, ridx, t, rays_o, rays_d, packs=None, collect=None):
        """sdf at o[ridx] + d[ridx]*t.  No-grad calls never materialise the points (fused kernel).
        packs = (pack_infos [P,2], ray of every pack [P] | None): the samples are the packs of coherent (image-ordered) rays -> the
        fused kernel walks them ray-tiled; same values.  collect = nsb_occ_collect | None: the accel's sample collection, done by the kernel."""
        if self.implicit_surface._fusable():
            if not torch.is_grad_enabled():
                return dict(sdf=self.implicit_surface.fused_sdf_rays(ridx, t, rays_o, rays_d, max_level=self.max_level, packs=packs, collect=collect))
            if not t.requires_grad:                              # learnable rays get their gradient from the fused op
                return dict(sdf=self.implicit_surface.fused_sdf_rays_autograd(ridx, t, rays_o, rays_d, max_level=self.max_level, packs=packs,
                                                                              collect=collect))
        if t.dim() == 2:
            x = torch.addcmul(rays_o[ridx].unsqueeze(-2), rays_d[ridx].unsqueeze(-2), t.unsqueeze(-1)).flatten(0, -2)
            return dict(sdf=self.forward_sdf(x)["sdf"].view(t.shape))
        return self.forward_sdf(torch.addcmul(rays_o[ridx], rays_d[ridx], t.unsqueeze(-1)))

    # ---- fused colour query (csrc/color_tc.cu)
    def _geometry_fusable(self):
        """the preconditions of the geometry-only colour op (sdf + nablas, csrc/color_tc.cu k_color_fwd<false>): those of the fused SDF query"""
        return self.implicit_surface._fusable()

    def _color_fusable(self):
        from .networks import SHEncoder
        if self.radiance_net is None:
            return False
        r, b = self.radiance_net, self.radiance_net.blocks
        return (self.implicit_surface._fusable() and r.use_pos and r.use_view_dirs and r.use_nablas and r.use_extra_feat
                and isinstance(r.embed_fn_view, SHEncoder) and r.embed_fn_view.degree == 4 and b.D == 2 and not b.skips and b.dtype == torch.half
                and all(isinstance(l.activation, nn.ReLU) for l in b.layers[:2]) and isinstance(b.layers[2].activation, nn.Sigmoid)
                and b.layers[0].out_features <= 64 and b.layers[1].out_features <= 64 and b.layers[1].in_features == b.layers[0].out_features
                and 0 <= b.layers[0].in_features - self.implicit_surface.encoding.out_features - 22 <= 8
                and all(l.bias is not None for l in b.layers))

    def _fused_color_state(self):
        """(fp16 table, nsb_color_net, the fp16 tensors it points at) -- rebuilt when a master changed."""
        s, b = self.implicit_surface, self.radiance_net.blocks.layers
        grid16, _dec = s._fused_state()
        ps = [s.decoder.layers[0].weight, s.decoder.layers[0].bias, s.decoder.layers[1].weight, s.decoder.layers[1].bias,
              b[0].weight, b[0].bias, b[1].weight, b[1].bias, b[2].weight, b[2].bias]
        key = tuple((p.data_ptr(), p._version) for p in ps)
        cache = getattr(self, "_color_cache", None)
        if cache is None or cache[0] != key:
            t = [p.detach().to(torch.half).contiguous() for p in ps]
            cache = self._color_cache = (key, t, color_net_c(t, s.decoder.layers, b, self._nablas_fac()))
        return grid16, cache[2], cache[1]

    def _nablas_fac(self):
        """sdf_scale / radius3d_original per axis as host floats"""
        s = self.implicit_surface
        r3 = s.radius3d_original                          # a buffer: read back once, not at every parameter update (a host sync)
        fk = (r3.data_ptr(), r3._version, float(s.sdf_scale))
        if getattr(self, "_fac_cache", (None,))[0] != fk:
            self._fac_cache = (fk, (s.sdf_scale / r3).float().tolist())
        return self._fac_cache[1]

    def _fused_geometry_state(self):
        """(fp16 table, nsb_color_net with rad_width = 0, the fp16 tensors it points at) for the geometry-only op; the fp16 images are
        the fused SDF query's (LoTDSDF._fused_state)"""
        s = self.implicit_surface
        grid16, _dec = s._fused_state()
        t, fac = s._fused_cache[1], self._nablas_fac()
        cache = getattr(self, "_geo_cache", None)
        if cache is None or cache[0] is not t or cache[1] != fac:
            cache = self._geo_cache = (t, list(fac), color_net_c(t[1:], s.decoder.layers, None, fac))
        return grid16, cache[2], t

    def forward_on_rays(self, ridx, t, rays_o, rays_d, view_dirs=None, rays_h_appear=None, *, nablas_has_grad=True, with_rgb=True):
        """LoTDNeuS.forward at x = o[ridx] + d[ridx] t with per-ray view_dirs / h_appear, as one fused op (fields/fused_color.py).
        with_rgb=False: sdf and nablas only (no view_dirs / h_appear; any model, with or without a radiance net)."""
        accel = getattr(self, "accel", None)
        collect = accel.occ.collect_struct() if (self.training and accel is not None) else None
        return fused_color(self, ridx, t, rays_o, rays_d, view_dirs, rays_h_appear if self.use_h_appear else None,
                           nablas_has_grad=nablas_has_grad, collect=collect, with_rgb=with_rgb)

    @torch.no_grad()
    def query_sdf(self, x):
        return self.forward_sdf(x)["sdf"]

    def forward_sdf_nablas(self, x, *, has_grad: bool = None, nablas_has_grad: bool = None, grad_guard=None):
        return self.implicit_surface.forward_sdf_nablas(x, has_grad=has_grad, nablas_has_grad=nablas_has_grad, max_level=self.max_level,
                                                        grad_guard=grad_guard)

    def forward(self, x, *, v=None, h_appear=None, has_grad: bool = None, nablas_has_grad: bool = None, with_rgb=True, with_normal=True):
        if with_rgb and self.radiance_net is None:
            raise RuntimeError("LoTDNeuS.forward(with_rgb=True): this model has no radiance net (radiance_cfg=False); query it with with_rgb=False")
        prefix = x.shape[:-1]
        if with_normal or (with_rgb and self.use_nablas):
            ret = self.forward_sdf_nablas(x, has_grad=has_grad, nablas_has_grad=nablas_has_grad)
        else:
            ret = self.forward_sdf(x, return_h=True)
        if with_rgb:
            ret.update(self.radiance_net(
                x, v=v.expand(*prefix, 3) if self.use_view_dirs else None,
                n=ret["nablas"].detach().clamp(-1, 1) if self.use_nablas else None,   # clamp: no salt-and-pepper from large dy/dx
                h_extra=ret["h"], h_appear=h_appear.expand(*prefix, -1) if (h_appear is not None and self.use_h_appear) else None))
        return ret


class LoTDNeuSModel(LoTDNeuS):
    """LoTDNeuS + the NeuS renderer mixin: occupancy accel, ray_test, ray_query (renderer_mixin.py:40-440)."""

    def __init__(self, *args, accel_cfg: dict = None, ray_query_cfg: dict = None, **kw):
        device = kw.get("device")
        super().__init__(*args, **kw)
        self.accel = OccGridAccel(space=self.space, device=device, **(accel_cfg or {})) if accel_cfg is not None else None
        self.ray_query_cfg = _Cfg(ray_query_cfg or dict(query_mode="march_occ_multi_upsample_compressed", query_param={}))
        self.upsample_s_divisor = 1.0
        self.it = 0

    # ---- sampling helpers the losses use (renderer_mixin.py:137-152)
    def sample_pts_uniform(self, num_samples: int):
        x = self.space.sample_pts_uniform(num_samples)
        ret = {k: v.to(x.dtype) for k, v in LoTDNeuS.forward_sdf_nablas(self, x).items()}
        ret["net_x"] = x
        return ret

    def sample_pts_in_occupied(self, num_samples: int):
        x = self.accel.sample_pts_in_occupied(num_samples)
        ret = {k: v.to(x.dtype) for k, v in LoTDNeuS.forward_sdf_nablas(self, x).items()}
        ret["net_x"] = x
        return ret

    @torch.no_grad()
    def query_sdf(self, x):
        # the base model's query: no sample collection (renderer_mixin.py:166-168 -> super().query_sdf); this is what the accel's own
        # init / EMA update evaluate
        return LoTDNeuS.forward_sdf(self, x)["sdf"]

    # ---- the accel watches every training-time SDF query (renderer_mixin.py:154-164)
    def forward_sdf(self, x, skip_accel=False, **kw):
        collect = self.accel.occ.collect_struct() if (self.training and not skip_accel and self.accel is not None) else None
        if collect is not None and not kw.get("return_h", False) and self.implicit_surface._fusable() and not x.requires_grad:
            s = self.implicit_surface                               # the fused query collects in-kernel
            fn = s.fused_sdf_autograd if torch.is_grad_enabled() else s.fused_sdf
            return dict(sdf=fn(x, max_level=self.max_level, collect=collect))
        ret = super().forward_sdf(x, **kw)
        if self.training and not skip_accel and self.accel is not None:
            self.accel.collect_samples(x, val=ret["sdf"].detach())
        return ret

    def forward_sdf_on_rays(self, ridx, t, rays_o, rays_d, packs=None):
        # training: the accel watches every SDF query (renderer_mixin.py:154-164).  The fused kernels do the collection themselves
        # (nsb_occ_collect); the unfused fall-back went through self.forward_sdf, which collected already.
        collect = self.accel.occ.collect_struct() if (self.training and self.accel is not None) else None
        return super().forward_sdf_on_rays(ridx, t, rays_o, rays_d, packs=packs, collect=collect)

    def forward_sdf_nablas(self, x, skip_accel=False, **kw):
        ret = super().forward_sdf_nablas(x, **kw)
        if self.training and not skip_accel and self.accel is not None:
            self.accel.collect_samples(x, val=ret["sdf"].detach())
        return ret

    def training_initialize(self, logger=None):
        return self.accel.init(self.query_sdf, logger=logger) if self.accel is not None else False

    def training_before_per_step(self, cur_it: int, logger=None):
        # lotd_neus.py:116-121 then renderer_mixin.py:176-182: the level schedule is set before the accel queries the field
        self.it = cur_it
        self.ctrl_var.set_iter(cur_it)
        self.implicit_surface.training_before_per_step(cur_it, logger=logger)
        if self.accel is not None:
            self.upsample_s_divisor = 2 ** self.accel.training_granularity
            if self.training:
                self.accel.step(cur_it, self.query_sdf, logger)

    def ray_test(self, rays_o, rays_d, near=None, far=None, return_rays=True, **extra_ray_data):
        return self.space.ray_test(rays_o, rays_d, near=near, far=far, return_rays=return_rays, **extra_ray_data)

    def ray_query(self, ray_input=None, ray_tested=None, config=dict(), return_buffer=False, return_details=False,
                  render_per_obj_individual=False):
        """-> {'volume_buffer', 'details', 'rendered'} as NeusRendererMixin.ray_query (renderer_mixin.py:234-440)."""
        if ray_tested is None:
            assert ray_input is not None
            ray_tested = self.ray_test(**ray_input)
        config = _Cfg(config)
        device, dtype = self.device, torch.float
        query_mode = config.get("query_mode", self.ray_query_cfg.query_mode)
        with_rgb, with_normal = config.get("with_rgb", True), config.get("with_normal", True)
        forward_inv_s = config.get("forward_inv_s", None)
        if forward_inv_s is None:
            forward_inv_s = self.forward_inv_s()
        raw = dict()
        if return_buffer:
            raw["volume_buffer"] = dict(type="empty", rays_inds_hit=[])
        if return_details:
            details = raw["details"] = {}
        if render_per_obj_individual:
            prefix = ray_input["rays_o"].shape[:-1]
            rendered = raw["rendered"] = dict(depth_volume=torch.zeros(prefix, dtype=dtype, device=device),
                                              mask_volume=torch.zeros(prefix, dtype=dtype, device=device))
            if with_rgb:
                rendered["rgb_volume"] = torch.zeros([*prefix, 3], dtype=dtype, device=device)
            if with_normal:
                rendered["normals_volume"] = torch.zeros([*prefix, 3], dtype=dtype, device=device)
        if ray_tested["num_rays"] == 0:
            return raw
        if query_mode != "march_occ_multi_upsample_compressed":
            raise RuntimeError(f"query_mode={query_mode!r} is not built; the shipped configs use 'march_occ_multi_upsample_compressed'")
        qp = dict(config.get("query_param", None) or self.ray_query_cfg.get("query_param", {}))
        volume_buffer, qd = neus_ray_query_march_occ_multi_upsample_compressed(
            self, ray_tested, with_rgb=with_rgb, with_normal=with_normal, upsample_s_divisor=self.upsample_s_divisor,
            perturb=config.get("perturb", False), forward_inv_s=forward_inv_s, **qp)
        if return_buffer:
            raw["volume_buffer"] = volume_buffer
        if return_details:
            details.update(qd)
        if render_per_obj_individual and volume_buffer["type"] != "empty":
            volume_integration(volume_buffer, rendered, training=self.training,
                               depth_use_normalized_vw=config.get("depth_use_normalized_vw", True), nablas_key="nablas", fresh=True)
        return raw


def volume_integration(volume_buffer, rendered, training=True, depth_use_normalized_vw=True, nablas_key="nablas", fresh=False):
    """vw = alpha_to_vw(alpha); mask = sum vw; depth = sum vw/(mask+1e-10) t; rgb = sum vw rgb; normals = sum vw nablas
    (single_volume_renderer.py:73-102 / renderer_mixin.py:396-439).  Writes into `rendered` at rays_inds_hit."""
    hit = volume_buffer["rays_inds_hit"]
    if volume_buffer["type"] == "packed" and neus_graphics.FUSED_STAGES:
        # one kernel: weights + the four per-ray sums (+ one adjoint kernel), csrc/neus_fused.cu
        nab = volume_buffer.get(nablas_key) if "normals_volume" in rendered else None
        if nab is not None and not training:
            nab = F.normalize(nab.clamp(-1, 1), dim=-1)
        rgb = volume_buffer.get("rgb") if "rgb_volume" in rendered else None
        n_img = getattr(rendered, "_n", None)               # renderer._LazyZeros: nothing allocated yet
        if fresh and n_img is None and rendered["mask_volume"].dim() == 1:
            n_img = rendered["mask_volume"].shape[0]
        if fresh and n_img is not None:
            # `rendered` holds nothing yet (all zeros): the kernel writes whole-image buffers at rays_inds_hit directly
            vw, m, d, c, nn_ = neus_fused.composite(volume_buffer["opacity_alpha"], volume_buffer["t"], volume_buffer["pack_infos_hit"], rgb=rgb,
                                                     nablas=nab, normalize_depth=depth_use_normalized_vw, ray_index=hit, n_rays=n_img)
            volume_buffer["vw"] = vw
            rendered["mask_volume"], rendered["depth_volume"] = m, d
            if c is not None:
                rendered["rgb_volume"] = c
            if nn_ is not None:
                rendered["normals_volume"] = nn_
            return rendered
        vw, m, d, c, nn_ = neus_fused.composite(volume_buffer["opacity_alpha"], volume_buffer["t"], volume_buffer["pack_infos_hit"],
                                                 rgb=rgb, nablas=nab, normalize_depth=depth_use_normalized_vw)
        volume_buffer["vw"] = vw
        rendered["mask_volume"] = rendered["mask_volume"].index_put((hit,), m)
        rendered["depth_volume"] = rendered["depth_volume"].index_put((hit,), d)
        if c is not None:
            rendered["rgb_volume"] = rendered["rgb_volume"].index_put((hit,), c)
        if nn_ is not None:
            rendered["normals_volume"] = rendered["normals_volume"].index_put((hit,), nn_)
        return rendered
    if volume_buffer["type"] == "batched":
        vw = ray_alpha_to_vw(volume_buffer["opacity_alpha"])
        vw_sum = vw.sum(-1)
        depth_w = vw / (vw_sum.unsqueeze(-1) + 1e-10) if depth_use_normalized_vw else vw
        red = lambda a: a.sum(-1 if a.dim() == vw.dim() else -2)
        expand = lambda a: a.unsqueeze(-1)
    else:
        pi = volume_buffer["pack_infos_hit"]
        vw = packed_alpha_to_vw(volume_buffer["opacity_alpha"], pi)
        vw_sum = packed_sum(vw.view(-1), pi)
        depth_w = packed_div(vw, vw_sum + 1e-10, pi) if depth_use_normalized_vw else vw
        red = lambda a: packed_sum(a, pi)
        expand = lambda a: a.view(-1, 1)
    volume_buffer["vw"] = vw
    rendered["mask_volume"] = rendered["mask_volume"].index_put((hit,), vw_sum)
    rendered["depth_volume"] = rendered["depth_volume"].index_put((hit,), red(depth_w * volume_buffer["t"]))
    if "rgb_volume" in rendered and "rgb" in volume_buffer:
        rendered["rgb_volume"] = rendered["rgb_volume"].index_put((hit,), red(expand(vw) * volume_buffer["rgb"]))
    if "normals_volume" in rendered and nablas_key in volume_buffer:
        nab = volume_buffer[nablas_key]
        if not training:
            nab = F.normalize(nab.clamp(-1, 1), dim=-1)
        rendered["normals_volume"] = rendered["normals_volume"].index_put((hit,), red(expand(vw) * nab))
    return rendered
