"""Tiny networks of the NeuS field -- API of `nr3d_lib.models.layers.DenseLayer`, `blocks.MLP`, `fields.sdf.LoTDSDF`,
`fields.nerf.RadianceNet`, `embedders.SHEncoder`, `fields.neus.variance`
(reference files: nr3d_lib/nr3d_lib/models/layers.py:228-312, blocks/mlp.py:26-125, fields/sdf/lotd_sdf.py:40-257,
fields/nerf/mlp_nerf.py:188-289, embedders/spherical_harmonics/sphere_harmonics.py:14-82, fields/neus/variance.py:122-142).

fp32 master weights, fp16 autocast evaluation -- the numerics contract of the reference.  The modules below are the
reference's layers (torch autocast, cuBLAS) and remain the specification; the hot path replaces them by fused wgmma
kernels with the same rounding points: SDF queries (with or without grad) by `nsb_fused_sdf*` + `nsb_fused_sdf_bwd`
(`_FusedSDF`, csrc/fused_tc.cu), the colour / normal query by `nsb_fused_color_*` (fields/fused_color.py, csrc/color_tc.cu).
"""
from __future__ import annotations

import ctypes
import math
from typing import List, Union

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import autograd

from .. import _lib as L
from ..bindings import _shencoder
from .encoding import LoTDEncoding


def _act(cfg):
    if cfg is None or cfg == "none":
        return None
    if isinstance(cfg, dict):
        cfg = dict(cfg)
        name = cfg.pop("type")
    else:
        name, cfg = cfg, {}
    name = name.lower()
    if name == "relu":
        return nn.ReLU(inplace=False)
    if name == "softplus":
        return nn.Softplus(beta=cfg.get("beta", 1.0))
    if name == "sigmoid":
        return nn.Sigmoid()
    raise RuntimeError(f"Invalid nonlinearity={name}")


class DenseLayer(nn.Module):
    """Linear layer evaluated under autocast(dtype) with fp32 parameters (layers.py:228-312)."""

    def __init__(self, in_features, out_features, *, bias=True, activation=None, dtype=torch.float, device=None, generator=None):
        super().__init__()
        self.dtype = dtype
        self.in_features, self.out_features = in_features, out_features
        bound = 1.0 / math.sqrt(in_features)       # == kaiming_uniform_(a=sqrt(5)) of nn.Linear
        w = torch.empty((out_features, in_features), device=device, dtype=torch.float).uniform_(-bound, bound, generator=generator)
        self.weight = nn.Parameter(w)
        if bias:
            self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=torch.float).uniform_(-bound, bound, generator=generator))
        else:
            self.register_parameter("bias", None)
        self.activation = _act(activation) if not isinstance(activation, nn.Module) else activation

    def forward(self, x, max_channel: int = None):
        with torch.autocast(device_type="cuda", dtype=self.dtype, enabled=self.dtype != torch.float):
            w = self.weight[:, :max_channel] if max_channel is not None else self.weight
            out = F.linear(x, w, self.bias)
            return self.activation(out) if self.activation is not None else out


class MLP(nn.Module):
    """D hidden layers of width W (blocks/mlp.py:26-125); state-dict keys `layers.{i}.{weight,bias}`."""

    def __init__(self, in_features, out_features, *, D=4, W: Union[int, List[int]] = 128, skips: List[int] = [], activation="relu",
                 output_activation=None, bias=True, dtype=None, device=None, generator=None):
        super().__init__()
        self.dtype = dtype or torch.float
        self.D, self.skips, self.in_features = D, list(skips), in_features
        Ws = [W] * D if isinstance(W, int) else list(W)
        layers = []
        for l in range(D + 1):
            o = out_features if l == D else Ws[l]
            i = in_features if l == 0 else (in_features + Ws[l - 1] if l in self.skips else Ws[l - 1])
            layers.append(DenseLayer(i, o, activation=(output_activation if l == D else activation), bias=bias, dtype=self.dtype,
                                     device=device, generator=generator))
        self.layers = nn.ModuleList(layers)

    def forward(self, x, return_last=False):
        h = x
        last = None
        for i, layer in enumerate(self.layers):
            if i == 0:
                h = layer(x)
            elif i in self.skips:
                h = layer(torch.cat([h, x], dim=-1))
            else:
                if i == self.D:
                    last = h
                h = layer(h)
        return (h, last) if return_last else h


class _sh_encoder(autograd.Function):
    @staticmethod
    def forward(ctx, inputs, degree, calc_grad_inputs=False):
        inputs = inputs.contiguous().float()
        B = inputs.shape[0]
        out = torch.empty(B, degree ** 2, dtype=inputs.dtype, device=inputs.device)
        dy_dx = torch.empty(B, 3 * degree ** 2, dtype=inputs.dtype, device=inputs.device) if calc_grad_inputs else torch.empty(1, dtype=inputs.dtype, device=inputs.device)
        _shencoder.sh_encode_forward(inputs, out, B, 3, degree, calc_grad_inputs, dy_dx)
        if calc_grad_inputs:
            ctx.save_for_backward(inputs, dy_dx)
            ctx.dims = (B, degree)
        ctx.calc = calc_grad_inputs
        return out

    @staticmethod
    def backward(ctx, grad):
        if not ctx.calc:
            return None, None, None
        inputs, dy_dx = ctx.saved_tensors
        B, degree = ctx.dims
        gi = torch.zeros_like(inputs)
        _shencoder.sh_encode_backward(grad.contiguous().float(), inputs, B, 3, degree, dy_dx, gi)
        return gi, None, None


class SHEncoder(nn.Module):
    def __init__(self, input_dim=3, degree=4):
        super().__init__()
        assert input_dim == 3, "SH encoder only support input dim == 3"
        assert 0 < degree <= 4, "this build's SH encoder supports degree in [1, 4]"
        self.degree, self.in_features, self.out_features = degree, 3, degree ** 2

    def forward(self, inputs, size=1):
        prefix = inputs.shape[:-1]
        flat = (inputs / size).flatten(0, -2)
        return _sh_encoder.apply(flat, self.degree, flat.requires_grad).unflatten(0, prefix)


class _FusedSDF(autograd.Function):
    """sdf = decoder(LoTD(x)) as ONE op with a hand-written backward (csrc/fused_tc.cu): forward keeps nothing but its
    inputs, backward recomputes features / pre-activations and accumulates straight into fp32 gradients of the table and
    the four decoder tensors.  `x` is either points [N,3] or a (ridx, t, rays_o, rays_d) tuple (x = o[ridx] + d[ridx] t)."""

    @staticmethod
    def forward(ctx, owner, pts, max_level, grid, W1, b1, W2, b2):
        grid16, dec = owner._fused_state()
        with L.KERNEL_TIMER.time("fused_sdf_fwd", (pts[1] if isinstance(pts, tuple) else pts).shape[0]):
            sdf = owner._launch_sdf(grid16, dec, pts, max_level)
        n = sdf.shape[0]
        ctx.owner, ctx.pts, ctx.max_level, ctx.n = owner, pts[:5] if isinstance(pts, tuple) else pts, max_level, n
        ctx.held = (grid16, dec, owner._fused_cache[1])          # the fp16 images the forward used (the tensors `dec` points into stay alive)
        ctx.shapes = (grid.shape, W1.shape, b1.shape, W2.shape, b2.shape)
        return sdf

    @staticmethod
    @autograd.function.once_differentiable
    def backward(ctx, d_sdf):
        grid16, dec, _alive = ctx.held
        meta, dev = ctx.owner.encoding.meta, d_sdf.device
        gs, w1s, b1s, w2s, b2s = ctx.shapes
        d_grid = torch.zeros(gs, dtype=torch.float32, device=dev)
        ks = [int(torch.Size(x).numel()) for x in (w1s, b1s, w2s, b2s)]
        small = torch.zeros(sum(ks), dtype=torch.float32, device=dev)         # one zero-fill for the four decoder gradients
        d_W1, d_b1 = small[:ks[0]].view(w1s), small[ks[0]:ks[0] + ks[1]].view(b1s)
        d_W2, d_b2 = small[ks[0] + ks[1]:ks[0] + ks[1] + ks[2]].view(w2s), small[ks[0] + ks[1] + ks[2]:].view(b2s)
        d_sdf = d_sdf.contiguous().float()
        # Most boundary points of a NeuS ray carry an exactly-zero cotangent (saturated sigmoid far from the surface, samples
        # behind the early-stop): only the others are recomputed (the reference's scatter kernel skips them one by one).
        from ..graphics.neus_fused import scan_counts      # compaction without a driver-level sync (the size is polled from pinned memory)
        keep = scan_counts(d_sdf.ne(0).to(torch.int32), want_index=True)["index"]
        n = keep.numel()
        if n == 0:
            return None, None, None, d_grid, d_W1, d_b1, d_W2, d_b2
        sparse = n < 0.9 * ctx.n
        if sparse:
            d_sdf = d_sdf[keep]
        if isinstance(ctx.pts, tuple):
            ridx, t, rays_o, rays_d, _packs = ctx.pts[:5]
            if sparse:
                ridx, t = ridx[keep], t[keep]
            args = (None, L.ptr(rays_o, "f32"), L.ptr(rays_d, "f32"), L.ptr(ridx, "i64"), L.ptr(t, "f32"))
        else:
            pts = ctx.pts[keep] if sparse else ctx.pts
            args = (L.ptr(pts, "f32"), None, None, None, None)
        n = n if sparse else ctx.n
        with L.KERNEL_TIMER.time("fused_sdf_bwd", n):
            L.check(L.lib().nsb_fused_sdf_bwd(meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), *args, L.ptr(d_sdf, "f32"), L.c_i64(n),
                                              L.c_i32(ctx.max_level), L.ptr(d_grid), L.ptr(d_W1), L.ptr(d_b1), L.ptr(d_W2), L.ptr(d_b2),
                                              L.stream_ptr()), "fused_sdf_bwd")
        return None, None, None, d_grid, d_W1, d_b1, d_W2, d_b2


class LoTDSDF(nn.Module):
    """LoTD encoding + MLP decoder -> sdf (and nablas by analytic back-propagation through decoder and table)."""

    def __init__(self, encoding_cfg: dict = None, decoder_cfg: dict = None, dtype=torch.half, device=None, generator=None,
                 sdf_scale=1.0, radius3d_original=1.0, aabb=None):
        super().__init__()
        self.dtype = dtype
        self.encoding = LoTDEncoding(3, **(encoding_cfg or {}), dtype=dtype, device=device, generator=generator, aabb=aabb)
        dc = dict(D=1, W=64, activation=dict(type="softplus", beta=100.0))
        dc.update(decoder_cfg or {})
        dc.pop("type", None)
        self.decoder = MLP(self.encoding.out_features, 1, **dc, dtype=dtype, device=device, generator=generator)
        self.sdf_scale = sdf_scale
        r3 = torch.as_tensor(radius3d_original, dtype=torch.float, device=device)
        self.register_buffer("radius3d_original", r3.expand(3).clone() if r3.numel() == 1 else r3.reshape(3).clone(), persistent=True)
        self.register_buffer("is_pretrained", torch.tensor([False], dtype=torch.bool, device=device), persistent=True)
        self._fused_cache = None

    # ---- reference API
    def forward(self, x, *, return_h=False, max_level: int = None):
        h = self.encoding(x, max_level=max_level)
        sdf = self.decoder(h)[..., 0]
        return dict(sdf=sdf, h=h) if return_h else dict(sdf=sdf)

    def forward_sdf(self, x, *, max_level: int = None):
        if self._fusable():
            if not torch.is_grad_enabled():
                return dict(sdf=self.fused_sdf(x, max_level=max_level))
            if not x.requires_grad:
                return dict(sdf=self.fused_sdf_autograd(x, max_level=max_level))
        return self.forward(x, return_h=False, max_level=max_level)

    def _ml(self, max_level):
        ml = max_level or self.encoding.max_level
        return self.encoding.meta.n_levels if ml is None else int(ml)

    def _launch_sdf(self, grid16, dec, pts, max_level):
        """one launch of the fused query.  pts: x [n,3]  |  (ridx, t, rays_o, rays_d, packs | None[, collect | None])"""
        meta = self.encoding.meta
        if isinstance(pts, tuple):
            ridx, t, rays_o, rays_d, packs = pts[:5]
            collect = pts[5] if len(pts) > 5 else None
            sdf = torch.empty(t.numel(), dtype=torch.float32, device=t.device)
            mode = 2 if packs is not None else 1
            L.check(L.lib().nsb_fused_sdf_collect(
                meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), None, L.ptr(rays_o, "f32"), L.ptr(rays_d, "f32"),
                L.ptr(ridx, "i64", allow_none=(mode == 2)) if mode == 1 else None, L.ptr(t, "f32"), L.c_i64(t.numel()),
                L.ptr(packs[0], "i64") if mode == 2 else None, L.ptr(packs[1], "i64", allow_none=True) if mode == 2 else None,
                L.c_i64(packs[0].shape[0] if mode == 2 else 0), L.c_i32(mode), L.c_i32(max_level), L.ptr(sdf),
                ctypes.byref(collect) if collect is not None else None, L.stream_ptr()), "fused_sdf")
            return sdf
        sdf = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
        L.check(L.lib().nsb_fused_sdf_collect(meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), L.ptr(pts, "f32"), None, None, None, None,
                                              L.c_i64(pts.shape[0]), None, None, L.c_i64(0), L.c_i32(0), L.c_i32(max_level), L.ptr(sdf),
                                              ctypes.byref(self._collect) if getattr(self, "_collect", None) is not None else None, L.stream_ptr()),
                "fused_sdf")
        return sdf

    def fused_sdf_autograd(self, x, max_level: int = None, collect=None):
        """differentiable (wrt. table + decoder) fused query on points [...,3]"""
        d = self.decoder.layers
        prefix = x.shape[:-1]
        self._collect = collect
        try:
            sdf = _FusedSDF.apply(self, x.detach().reshape(-1, 3).contiguous().float(), self._ml(max_level), self.encoding.flattened_params,
                                  d[0].weight, d[0].bias, d[1].weight, d[1].bias)
        finally:
            self._collect = None
        return sdf.view(prefix)

    def fused_sdf_rays_autograd(self, ridx, t, rays_o, rays_d, max_level: int = None, packs=None, collect=None):
        d = self.decoder.layers
        shape = t.shape
        if t.dim() == 2:
            ridx = ridx.unsqueeze(-1).expand(shape)
        pts = (ridx.reshape(-1).contiguous().long(), t.detach().reshape(-1).contiguous().float(), rays_o.detach().contiguous(),
               rays_d.detach().contiguous(), packs, collect)
        sdf = _FusedSDF.apply(self, pts, self._ml(max_level), self.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias)
        return sdf.view(shape)

    def forward_sdf_nablas(self, x, *, has_grad: bool = None, nablas_has_grad: bool = None, max_level: int = None, grad_guard=None):
        has_grad = torch.is_grad_enabled() if has_grad is None else has_grad
        nablas_has_grad = has_grad if nablas_has_grad is None else (nablas_has_grad and has_grad)
        need_dL_dinput = has_grad and x.requires_grad
        x = x.requires_grad_(True)
        with torch.enable_grad():
            h, dy_dx = self.encoding.forward_dydx(x, max_level=max_level, need_dL_dinput=need_dL_dinput)
            sdf = self.decoder(h)[..., 0]
        dL_dh = autograd.grad(sdf, h, sdf.new_ones(sdf.shape), retain_graph=has_grad, create_graph=nablas_has_grad, only_inputs=True)[0]
        nablas = self.encoding.backward_dydx(dL_dh, dy_dx, x, max_level=max_level, grad_guard=grad_guard)
        if not nablas_has_grad:
            nablas = nablas.detach()
        if not has_grad:
            sdf, h = sdf.detach(), h.detach()
        x.requires_grad_(need_dL_dinput)
        return dict(sdf=sdf, h=h, nablas=nablas * (self.sdf_scale / self.radius3d_original))

    # ---- fused no-grad query (csrc/fused.cu)
    def _fusable(self):
        """the preconditions of the fused kernels (csrc/fused_tc.cu: `n_pseudo == 16 && F == 2 && plmeta_two_feature_cells`, width <= 64, both
        biases, CUDA parameters); any other valid LoTD / decoder configuration takes the generic encoding -> decoder path of forward()"""
        e, d = self.encoding, self.decoder
        m = e.meta
        return (self.dtype == torch.half and e.window is None and d.D == 1 and e.out_features == 32 and e.in_features == 3
                and m.n_pseudo_levels == 16 and m.n_feat_per_pseudo_lvl == 2 and all(f == 2 for f in m.level_n_feats)
                and d.layers[0].out_features <= 64 and isinstance(d.layers[0].activation, nn.Softplus)
                and d.layers[0].bias is not None and d.layers[1].bias is not None and e.flattened_params.is_cuda)

    def _fused_state(self):
        """fp16 images of the masters, rebuilt when any master changed (version counters)."""
        ps = [self.encoding.flattened_params, self.decoder.layers[0].weight, self.decoder.layers[0].bias,
              self.decoder.layers[1].weight, self.decoder.layers[1].bias]
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if self._fused_cache is None or self._fused_cache[0] != key:
            t = [p.detach().to(torch.half).contiguous() for p in ps]
            dec = L.SdfDecoderC(t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), self.decoder.layers[0].out_features,
                                float(self.decoder.layers[0].activation.beta))
            self._fused_cache = (key, t, dec)
        return self._fused_cache[1][0], self._fused_cache[2]

    @torch.no_grad()
    def fused_sdf(self, x, max_level: int = None, collect=None):
        grid16, dec = self._fused_state()
        prefix = x.shape[:-1]
        xf = x.reshape(-1, 3).contiguous().float()
        self._collect = collect
        try:
            with L.KERNEL_TIMER.time("lotd_gather", xf.shape[0]):
                sdf = self._launch_sdf(grid16, dec, xf, self._ml(max_level))
        finally:
            self._collect = None
        return sdf.view(prefix)

    @torch.no_grad()
    def fused_sdf_rays(self, ridx, t, rays_o, rays_d, max_level: int = None, packs=None, collect=None):
        grid16, dec = self._fused_state()
        shape = t.shape
        if packs is not None or collect is not None:
            if packs is None and t.dim() == 2:
                ridx = ridx.unsqueeze(-1).expand(shape)
            tf = t.reshape(-1).contiguous().float()
            pts = (ridx.reshape(-1).contiguous().long() if packs is None else None, tf, rays_o.contiguous(), rays_d.contiguous(), packs, collect)
            with L.KERNEL_TIMER.time("lotd_gather", tf.shape[0]):
                sdf = self._launch_sdf(grid16, dec, pts, self._ml(max_level))
            return sdf.view(shape)
        if t.dim() == 2:
            ridx = ridx.unsqueeze(-1).expand(shape)
        ridx, tf = ridx.reshape(-1).contiguous().long(), t.reshape(-1).contiguous().float()
        sdf = torch.empty(tf.shape[0], dtype=torch.float32, device=tf.device)
        ml = self.encoding.meta.n_levels if (max_level or self.encoding.max_level) is None else int(max_level or self.encoding.max_level)
        with L.KERNEL_TIMER.time("lotd_gather", tf.shape[0]):
          L.check(L.lib().nsb_fused_sdf_rays(self.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), L.ptr(rays_o.contiguous(), "f32"),
                                           L.ptr(rays_d.contiguous(), "f32"), L.ptr(ridx, "i64"), L.ptr(tf, "f32"), L.c_i64(tf.shape[0]),
                                           L.c_i32(ml), L.ptr(sdf), L.stream_ptr()), "fused_sdf_rays")
        return sdf.view(shape)


class RadianceNet(nn.Module):
    """rgb = sigmoid(MLP([x, SH(v), n, h_extra, h_appear]))  (mlp_nerf.py:188-289); state-dict keys `blocks.layers.*`."""

    def __init__(self, use_pos=True, use_view_dirs=True, use_nablas=True, dir_embed_cfg=dict(type="spherical", degree=4), n_extra_feat=32,
                 n_appear_embedding=0, D=2, W=64, activation="relu", output_activation="sigmoid", dtype=torch.half, device=None, generator=None):
        super().__init__()
        self.use_pos, self.use_view_dirs, self.use_nablas = use_pos, use_view_dirs, use_nablas
        self.use_extra_feat, self.use_h_appear = n_extra_feat > 0, n_appear_embedding > 0
        ch = 3 if use_pos else 0
        if use_view_dirs:
            kind = dir_embed_cfg.get("type", "identity")
            if kind == "spherical":
                self.embed_fn_view = SHEncoder(3, dir_embed_cfg.get("degree", 4))
                ch += self.embed_fn_view.out_features
            elif kind == "identity":
                self.embed_fn_view = nn.Identity()
                ch += 3
            else:
                raise RuntimeError(f"dir_embed_cfg type={kind!r} is not built")
        ch += (3 if use_nablas else 0) + n_extra_feat + n_appear_embedding
        self.in_features = ch
        self.blocks = MLP(ch, 3, D=D, W=W, activation=activation, output_activation=output_activation, dtype=dtype, device=device,
                          generator=generator)

    def forward(self, x, *, v=None, n=None, h_extra=None, h_appear=None):
        parts = []
        if self.use_pos:
            parts.append(x)
        if self.use_view_dirs:
            parts.append(self.embed_fn_view(v))
        if self.use_nablas:
            parts.append(n)
        if self.use_extra_feat:
            parts.append(h_extra)
        if self.use_h_appear:
            parts.append(h_appear)
        return dict(rgb=self.blocks(torch.cat(parts, dim=-1)))


class VarSingleMixLinear(nn.Module):
    """inv_s = (1-w) * exp(ln_inv_s * factor) + w * final_inv_s with w annealed linearly (variance.py:122-142)."""

    def __init__(self, ln_inv_s_init, ln_inv_s_factor=10.0, stop_it=1, start_it=0, final_inv_s=2048., device=None):
        super().__init__()
        self.ln_inv_s_factor, self.final_inv_s = ln_inv_s_factor, final_inv_s
        self.start_it, self.stop_it, self.it = start_it, stop_it, 0
        self.ln_inv_s = nn.Parameter(torch.tensor([ln_inv_s_init], device=device, dtype=torch.float))

    def set_iter(self, it):
        self.it = it

    def mix_weight(self) -> float:
        return min(max((self.it - self.start_it) / max(self.stop_it - self.start_it, 1), 0.), 1.)

    def forward(self, it: int = None):
        if it is not None:
            self.set_iter(it)
        # the annealing weight is a host number in the reference; a captured CUDA graph would freeze it, so the static step
        # (graphics/neus_static.py) reads it from a device scalar that it refreshes before every replay
        w = self._w_dev if getattr(self, "_use_w_dev", False) else self.mix_weight()
        return (1 - w) * torch.exp(self.ln_inv_s * self.ln_inv_s_factor) + w * self.final_inv_s
