"""Putting the fused / static NeuS path UNDER a model object of the reference (INTEGRATION.md §3).

`accelerate(ref_model)` takes a `LoTDNeuS`-family model of an unmodified neuralsim checkout (app/models/single: `LoTDNeuSObj`,
`LoTDNeuSStreet` = `NeusRendererMixin` + `LoTDNeuS`, nr3d_lib/models/fields/neus/lotd_neus.py:27-232, renderer_mixin.py:40-440), builds the
`neuralsim_b200.fields.LoTDNeuSModel` with the same architecture AROUND THE REFERENCE'S OWN PARAMETER AND BUFFER OBJECTS (no copy: the table
`implicit_surface.encoding.flattened_params`, the decoder / radiance `layers.{i}.{weight,bias}`, `ctrl_var.ln_inv_s`, `accel.occ.occ_grid /
occ_val_grid`, `space.aabb` are shared, so the reference's optimisers, checkpoints and EMA keep working on them), and re-binds the three methods
the renderers call (`ray_test`, `ray_query`, `forward_sdf_nablas` stays the reference's) to it:

    import neuralsim_b200.bindings as nsb;  nsb.install_as_nr3d_lib_bindings()
    ...                                         # the reference builds its scene / asset bank as usual
    from neuralsim_b200.adapter import accelerate
    accelerate(scene.get_drawable_groups_by_class_name('Street')[0].model)       # app/renderers/single_volume_renderer.py:238-246 now lands in _query_fused

Only attribute names are used (duck typing), because the reference's model classes cannot be imported in the build container (addict, kornia, ...
are not installable there, SURVEY.md §8c); tests/test_adapter_gpu.py drives it with a stand-in that exposes exactly the reference's attributes.
Anything outside the built envelope raises instead of silently keeping the slow path.  A reference model without a radiance net
(`radiance_cfg: null`, e.g. the LiDAR-only StreetSurf configuration: `radiance_net is None`) becomes a geometry-only LoTDNeuSModel
(`radiance_cfg=False`) that shares the table, the decoder, `ln_inv_s`, the occupancy buffers and `radius3d_original`.
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn

from .fields.neus import LoTDNeuSModel

__all__ = ["accelerate", "describe"]


def _lotd_cfg_of(enc):
    cfg = getattr(enc, "lotd_cfg", None)
    if cfg is None:
        raise RuntimeError("adapter: the encoding has no `lotd_cfg` (lotd_encoding.py:86)")
    cfg = dict(cfg)
    keep = {k: cfg[k] for k in ("lod_res", "lod_n_feats", "lod_types") if k in cfg}
    keep["hashmap_size"] = cfg.get("hashmap_size", cfg.get("size"))
    return keep


def _mlp_shape(mlp):
    layers = list(mlp.layers)
    return dict(D=len(layers) - 1, W=[l.out_features for l in layers[:-1]])


def describe(ref_model) -> dict:
    """the constructor arguments of the equivalent LoTDNeuSModel, read off a reference model's attributes"""
    surf, rad = ref_model.implicit_surface, ref_model.radiance_net
    enc, dec = surf.encoding, surf.decoder
    act = dec.layers[0].activation
    if not isinstance(act, nn.Softplus):
        raise RuntimeError(f"adapter: decoder activation {type(act).__name__} is outside the built envelope (Softplus)")
    space = getattr(ref_model, "space", None) or enc.space
    aabb = space.aabb.detach().cpu().tolist()
    if rad is None:                                          # geometry only (lotd_neus.py:71-85)
        radiance_cfg = False
    else:
        blocks = rad.blocks
        in_rad = blocks.layers[0].in_features
        n_appear = in_rad - (3 + 16 + 3 + enc.out_features)
        if n_appear < 0:
            raise RuntimeError("adapter: radiance net input width does not match [x, SH4(v), n, h, h_appear]")
        radiance_cfg = dict(n_appear_embedding=int(n_appear), dir_embed_cfg=dict(type="spherical", degree=4), **_mlp_shape(blocks))
    occ = ref_model.accel.occ
    rq = ref_model.ray_query_cfg
    return dict(
        surface_cfg=dict(aabb=aabb, sdf_scale=float(getattr(surf, "sdf_scale", 1.0)), encoding_cfg=dict(lotd_cfg=_lotd_cfg_of(enc)),
                         decoder_cfg=dict(**_mlp_shape(dec), activation=dict(type="softplus", beta=float(act.beta)))),
        radiance_cfg=radiance_cfg,
        var_ctrl_cfg=dict(ln_inv_s_init=float(ref_model.ctrl_var.ln_inv_s.detach().reshape(-1)[0]),
                          ln_inv_s_factor=float(getattr(ref_model.ctrl_var, "ln_inv_s_factor", 10.0)),
                          start_it=getattr(ref_model.ctrl_var, "start_it", 0), stop_it=getattr(ref_model.ctrl_var, "stop_it", 1),
                          final_inv_s=float(getattr(ref_model.ctrl_var, "final_inv_s", 2048.))),
        accel_cfg=dict(resolution=list(occ.occ_grid.shape), occ_val_fn_cfg=dict(type="sdf", inv_s=float(getattr(occ, "occ_inv_s", 256.0))),
                       occ_thre=float(occ.occ_thre), ema_decay=float(occ.ema_decay),
                       update_from_samples_cfg=dict() if getattr(occ, "should_collect_samples", False) else None),
        ray_query_cfg=dict(query_mode=rq["query_mode"] if isinstance(rq, dict) else rq.query_mode,
                           query_param=dict(rq["query_param"] if isinstance(rq, dict) else rq.query_param)))


def _share(dst: nn.Module, name: str, src):
    """make `dst.<name>` BE the tensor object `src` (parameter or buffer)"""
    if isinstance(src, nn.Parameter):
        dst._parameters[name] = src
    else:
        dst._buffers[name] = src


def accelerate(ref_model, *, patch=True, max_fused_levels: int = 16) -> LoTDNeuSModel:
    """-> the LoTDNeuSModel that now backs `ref_model` (also stored as `ref_model._nsb`).  See the module docstring.
    max_fused_levels = 24 runs tables of 17..24 levels (the shipped StreetSurf camera models) on the fused kernels too."""
    cfg = describe(ref_model)
    cfg["surface_cfg"]["max_fused_levels"] = max_fused_levels
    dev = ref_model.implicit_surface.encoding.flattened_params.device
    ours = LoTDNeuSModel(device=dev, **cfg)
    rs, os_ = ref_model.implicit_surface, ours.implicit_surface
    if os_.encoding.flattened_params.shape != rs.encoding.flattened_params.shape:
        raise RuntimeError(f"adapter: table sizes differ ({tuple(os_.encoding.flattened_params.shape)} here, {tuple(rs.encoding.flattened_params.shape)} in the "
                           "reference): level types outside Dense / Hash?")
    _share(os_.encoding, "flattened_params", rs.encoding.flattened_params)
    pairs = [(os_.decoder.layers, rs.decoder.layers)]
    if ours.radiance_net is not None:
        pairs.append((ours.radiance_net.blocks.layers, ref_model.radiance_net.blocks.layers))
    for mine, theirs in pairs:
        for a, b in zip(mine, theirs):
            if a.weight.shape != b.weight.shape:
                raise RuntimeError(f"adapter: layer shapes differ ({tuple(a.weight.shape)} vs {tuple(b.weight.shape)})")
            _share(a, "weight", b.weight)
            if b.bias is None:
                raise RuntimeError("adapter: layers without bias are outside the built envelope")
            _share(a, "bias", b.bias)
    _share(ours.ctrl_var, "ln_inv_s", ref_model.ctrl_var.ln_inv_s)
    for k in ("occ_grid", "occ_val_grid", "is_initialized"):
        if hasattr(ref_model.accel.occ, k):
            _share(ours.accel.occ, k, getattr(ref_model.accel.occ, k))
    if hasattr(rs, "radius3d_original"):
        _share(os_, "radius3d_original", rs.radius3d_original)
    ours.train(ref_model.training)
    ref_model._nsb = ours
    if patch:
        def _sync(self):
            o = self._nsb
            o.train(self.training)
            # the level the reference's queries use: `max_level or encoding.max_level` (lotd_neus.py:127, lotd_encoding.py:162); the
            # model's own max_level stays None, the annealer sets the encoding's (lotd_encoding.py:146-148)
            o.max_level = getattr(self, "max_level", None)
            o.implicit_surface.encoding.max_level = getattr(self.implicit_surface.encoding, "max_level", None)
            o.upsample_s_divisor = getattr(self, "upsample_s_divisor", 1.0)
            o.ctrl_var.set_iter(getattr(self.ctrl_var, "it", getattr(self, "it", 0)))
            occ_r, occ_o = self.accel.occ, o.accel.occ
            if occ_o.occ_grid is not occ_r.occ_grid:             # the reference re-assigns `occ_grid` on every update (ema_single.py:190)
                occ_o._buffers["occ_grid"] = occ_r.occ_grid
            return o

        def ray_test(self, rays_o, rays_d, near=None, far=None, return_rays=True, **extra):
            return _sync(self).ray_test(rays_o, rays_d, near=near, far=far, return_rays=return_rays, **extra)

        def ray_query(self, ray_input=None, ray_tested=None, config=dict(), return_buffer=False, return_details=False, render_per_obj_individual=False):
            return _sync(self).ray_query(ray_input=ray_input, ray_tested=ray_tested, config=dict(config), return_buffer=return_buffer,
                                         return_details=return_details, render_per_obj_individual=render_per_obj_individual)

        ref_model.ray_test = types.MethodType(ray_test, ref_model)
        ref_model.ray_query = types.MethodType(ray_query, ref_model)
    return ours
