"""The colour / normal query of LoTDNeuS as ONE differentiable op over the wgmma kernels of csrc/color_tc.cu.

`fused_color(model, ridx, t, rays_o, rays_d, view_dirs, h_appear)` computes, for the packed samples x = o[ridx] + d[ridx] t,
what `LoTDNeuS.forward(x, v=, h_appear=, nablas_has_grad=True)` computes in the reference
(nr3d_lib/models/fields/neus/lotd_neus.py:141-167): sdf, nablas (analytic, differentiable -> second-order table / decoder
gradients) and rgb.  The unfused module path (`LoTDNeuS.forward`) stays the specification the tests compare against.
"""
from __future__ import annotations

import ctypes

import torch
from torch import autograd

from .. import _lib as L


class _FusedColor(autograd.Function):
    @staticmethod
    def forward(ctx, model, pts, view_dirs, h_appear, max_level, keep, collect, *params):
        grid16, net, _held = model._fused_color_state()
        ridx, t, rays_o, rays_d = pts
        n, dev = t.numel(), t.device
        meta = model.implicit_surface.encoding.meta
        sdf = torch.empty(n, dtype=torch.float32, device=dev)
        nab = torch.empty(n, 3, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
        x = torch.empty(n, 3, dtype=torch.float32, device=dev)
        acts = None
        if keep:
            acts = torch.empty(4, int(L.lib().nsb_color_tile_bytes(L.c_i64(n))), dtype=torch.uint8, device=dev)
        ap = [L.ptr(acts[k]) if keep else None for k in range(4)]
        with L.KERNEL_TIMER.time("fused_color_fwd", n):
            L.check(L.lib().nsb_fused_color_fwd(meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(net), None, L.ptr(rays_o, "f32"), L.ptr(rays_d, "f32"),
                                                L.ptr(ridx, "i64"), L.ptr(t, "f32"), L.ptr(view_dirs, "f32"), L.ptr(h_appear, "f32", allow_none=True),
                                                L.c_i64(n), L.c_i32(max_level), L.ptr(sdf), L.ptr(nab), L.ptr(rgb), L.ptr(x), *ap,
                                                ctypes.byref(collect) if collect is not None else None, L.stream_ptr()),
                    "fused_color_fwd")
        ctx.model, ctx.pts, ctx.max_level, ctx.n = model, pts, max_level, n
        ctx.held = (grid16, net, _held, acts, rgb)
        ctx.shapes = [p.shape for p in params]
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(x)
        return sdf, nab, rgb, x

    @staticmethod
    @autograd.function.once_differentiable
    def backward(ctx, g_sdf, g_nab, g_rgb, _gx):
        grid16, net, _held, acts, rgb = ctx.held
        if acts is None:
            raise RuntimeError("fused_color: backward through a forward that ran without grad")
        dev, n = rgb.device, ctx.n
        meta = ctx.model.implicit_surface.encoding.meta
        # one zero-fill for the table gradient, one for the ten small tensors (views of a flat buffer)
        sizes = [int(torch.Size(s).numel()) for s in ctx.shapes[1:]]
        small = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        grads, o = [torch.zeros(ctx.shapes[0], dtype=torch.float32, device=dev)], 0
        for sh, k in zip(ctx.shapes[1:], sizes):
            grads.append(small[o:o + k].view(sh))
            o += k
        if g_sdf is None and g_nab is None and g_rgb is None:
            return (None,) * 7 + tuple(grads)
        ridx, t, rays_o, rays_d = ctx.pts
        c = lambda g: None if g is None else g.contiguous().float()
        g_sdf, g_nab, g_rgb = c(g_sdf), c(g_nab), c(g_rgb)
        dh = torch.empty(n, 32, dtype=torch.float32, device=dev)
        with L.KERNEL_TIMER.time("fused_color_bwd", n):
            L.check(L.lib().nsb_fused_color_bwd(meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(net), None, L.ptr(rays_o, "f32"), L.ptr(rays_d, "f32"),
                                                L.ptr(ridx, "i64"), L.ptr(t, "f32"), L.c_i64(n), L.c_i32(ctx.max_level), L.ptr(acts[0]), L.ptr(acts[1]),
                                                L.ptr(acts[2]), L.ptr(acts[3]), L.ptr(rgb), L.ptr(g_sdf, allow_none=True), L.ptr(g_nab, allow_none=True),
                                                L.ptr(g_rgb, allow_none=True), L.ptr(dh), *[L.ptr(g) for g in grads], L.stream_ptr()),
                    "fused_color_bwd")
        return (None,) * 7 + tuple(grads)


def fused_color(model, ridx, t, rays_o, rays_d, view_dirs, h_appear=None, *, nablas_has_grad=True, collect=None):
    """-> dict(sdf [n], nablas [n,3], rgb [n,3], x [n,3]).  Gradients flow to the table, the decoder and the radiance net."""
    s, r = model.implicit_surface, model.radiance_net.blocks.layers
    d = s.decoder.layers
    params = (s.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias, r[0].weight, r[0].bias, r[1].weight, r[1].bias,
              r[2].weight, r[2].bias)
    pts = (ridx.reshape(-1).contiguous().long(), t.detach().reshape(-1).contiguous().float(), rays_o.detach().contiguous().float(),
           rays_d.detach().contiguous().float())
    keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    ha = None if h_appear is None else h_appear.detach().contiguous().float()
    sdf, nab, rgb, x = _FusedColor.apply(model, pts, view_dirs.detach().contiguous().float(), ha, s._ml(model.max_level), keep, collect, *params)
    if not nablas_has_grad:
        nab = nab.detach()
    return dict(sdf=sdf, nablas=nab, rgb=rgb, x=x)
