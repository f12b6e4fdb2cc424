"""The colour / normal query of LoTDNeuS as ONE differentiable op over the wgmma kernels of csrc/color_tc.cu.

`fused_color(model, ridx, t, rays_o, rays_d, view_dirs, h_appear)` computes, for the packed samples x = o[ridx] + d[ridx] t,
what `LoTDNeuS.forward(x, v=, h_appear=, nablas_has_grad=True)` computes in the reference
(nr3d_lib/models/fields/neus/lotd_neus.py:141-167): sdf, nablas (analytic, differentiable -> second-order table / decoder
gradients) and rgb; appearance codes, rays and view directions that require grad get their gradient (summed over each ray's samples).  The unfused module path (`LoTDNeuS.forward`) stays the specification the tests compare against.
With `with_rgb=False` it is `forward_sdf_nablas` alone (k_color_fwd<false>: no radiance head runs, two activation tiles are kept instead of
four, and only the table and the decoder are inputs of the op), for models without a radiance net and for rays that render no rgb.
"""
from __future__ import annotations

import ctypes

import torch
from torch import autograd

from .. import _lib as L


def h_tile_cols(n_levels):
    """the width of the kernels' feature tile for an n_levels-level table (csrc/fused_tc_common.cuh feature_cols): the columns of dh_scratch"""
    return 32 if n_levels <= 16 else 48


def color_net_c(t16, dec, rad, fac):
    """nsb_color_net over the fp16 images t16 = (W1, b1, W2, b2[, R1, rb1, R2, rb2, R3, rb3]) of the decoder layers `dec` and the radiance
    layers `rad` (None: the geometry-only net, rad_width = 0); fac: sdf_scale / radius3d_original per axis"""
    ptrs = [x.data_ptr() for x in t16] + [None] * (10 - len(t16))
    # the radiance input is [x(3), SH4(v) (16), n(3), h(2L), h_appear(n_appear)]; the decoder's input is h
    rw, ri, na = (rad[0].out_features, rad[0].in_features, rad[0].in_features - 22 - dec[0].in_features) if rad is not None else (0, 0, 0)
    return L.ColorNetC(*ptrs, dec[0].out_features, rw, ri, na, float(dec[0].activation.beta), (ctypes.c_float * 3)(*fac))


class SharedTableGrad:
    """One zero-filled fp32 table gradient that several backward nodes of a step scatter into, instead of a buffer each that autograd
    then adds up.  The nodes take the table through `route(table)`, an identity node created before them: each node's backward adds its
    part into `take()` and returns None for the table, and the identity node -- which autograd runs only after every node that consumes
    its output -- hands the finished buffer on and empties the holder.  So autograd sees the buffer only once all parts are in it,
    whatever else contributes to the table's gradient, and the next backward pass (a retained graph) starts from a fresh zeroed buffer."""
    __slots__ = ("buf",)

    def __init__(self):
        self.buf = None

    def route(self, table, anchor=None):
        """-> the table as the input of the nodes that scatter into this holder.  anchor (optional): a tensor that requires grad, an input
        of the identity node too, so that the nodes' outputs require grad -- and their backward passes run -- even when the table does not
        (a step that returns only gradients to its inputs); its node's backward runs after this one's, so after all the nodes'"""
        return _TableGradSink.apply(self, table, anchor)

    def take(self, shape, device):
        """(inside a backward) -> the buffer, zero-filled by the first caller of this backward pass"""
        if self.buf is None:
            self.buf = torch.zeros(shape, dtype=torch.float32, device=device)
        return self.buf


class _TableGradSink(autograd.Function):
    """identity on the table; its backward passes the holder's buffer on (see SharedTableGrad)"""

    @staticmethod
    def forward(ctx, holder, table, anchor=None):
        ctx.holder = holder
        ctx.set_materialize_grads(False)
        return table.view_as(table)

    @staticmethod
    @autograd.function.once_differentiable
    def backward(ctx, g):
        buf, ctx.holder.buf = ctx.holder.buf, None
        if g is not None:                          # a consumer that returned its own table gradient
            buf = g if buf is None else buf.add_(g)
        return None, buf, None


class ColorQuery:
    """what the forward and backward launches of one colour query share: the table's meta and fp16 image, the net struct and the fp16
    tensors it points at, the rays, max level (a host int, or a device int32 scalar: _lib.call's level=), the occupancy collection, the device count (_lib.call's count=, None: host-sized),
    the step's shared table gradient (a SharedTableGrad, None: the backward fills its own) and the step's appearance-code gradient
    (None, or (d_h_appear, ray_map): the backward adds the code gradient of ray r into d_h_appear[ray_map[r]], which the caller
    zero-fills -- for codes that are not an autograd input of the op, as in the one-launch step) and the step's ray gradient (None, or
    (d_rays_o, d_rays_d, d_view_dirs | None, ray_map): the backward adds ray r's gradient to its rays and view direction at row
    ray_map[r] of the caller's zero-filled buffers; the entry point takes one ray map, so with both it must be the codes' one)"""
    __slots__ = ("meta", "grid16", "net", "held", "rays_o", "rays_d", "ml", "collect", "count", "table_grad", "appear_grad", "ray_grad")

    def __init__(self, meta, grid16, net, held, rays_o, rays_d, ml, collect, count, table_grad=None, appear_grad=None, ray_grad=None):
        self.meta, self.grid16, self.net, self.held = meta, grid16, net, held
        self.rays_o, self.rays_d, self.ml, self.collect, self.count = rays_o, rays_d, ml, collect, count
        self.table_grad, self.appear_grad, self.ray_grad = table_grad, appear_grad, ray_grad
        if appear_grad is not None and ray_grad is not None and appear_grad[1] is not ray_grad[3]:
            raise RuntimeError("ColorQuery: the code and ray gradients must share one ray map")


class _FusedColor(autograd.Function):
    """q: ColorQuery; params: the five SDF parameters (table, W1, b1, W2, b2), then the six radiance parameters when rgb is computed.
    rays_o / rays_d (or None): the rays q holds detached copies of, as inputs of the op, so that learnable rays get their gradient."""

    @staticmethod
    def forward(ctx, q, ridx, t, view_dirs, h_appear, rays_o, rays_d, keep, *params):
        rad = len(params) > 5
        n, dev = t.numel(), t.device
        sdf = torch.empty(n, dtype=torch.float32, device=dev)
        nab = torch.empty(n, 3, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev) if rad else None
        x = torch.empty(n, 3, dtype=torch.float32, device=dev)
        n_act = 4 if rad else 2                                  # Z, X (+ Y1, Y2)
        acts = None
        if keep:
            acts = torch.empty(n_act, int(L.lib().nsb_color_act_bytes(n, q.meta.n_pseudo_levels)), dtype=torch.uint8, device=dev)
        ap = [L.ptr(acts[k]) if keep and k < n_act else None for k in range(4)]
        P = L.ptr
        with L.KERNEL_TIMER.time("fused_color_fwd", n):
            L.call(L.lib().nsb_fused_color_fwd, "fused_color_fwd", q.meta.c_ref, P(q.grid16, "f16"), ctypes.byref(q.net), None, P(q.rays_o, "f32"),
                   P(q.rays_d, "f32"), P(ridx, "i64"), P(t, "f32"), P(view_dirs, "f32", allow_none=not rad), P(h_appear, "f32", allow_none=True),
                   L.c_i64(n), L.c_level(q.ml), P(sdf), P(nab), P(rgb, allow_none=not rad), P(x), *ap,
                   ctypes.byref(q.collect) if q.collect is not None else None, L.stream_ptr(), count=q.count, level=q.ml)
        ctx.q, ctx.ridx, ctx.t, ctx.n, ctx.rad = q, ridx, t, n, rad
        ctx.ha_shape = h_appear.shape if h_appear is not None else None
        ctx.vd = view_dirs
        ctx.held = (acts, rgb)
        ctx.shapes = [p.shape for p in params]
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(x)
        return (sdf, nab, rgb, x) if rad else (sdf, nab, x)

    @staticmethod
    @autograd.function.once_differentiable
    def backward(ctx, *g_out):
        acts, rgb = ctx.held
        if acts is None:
            raise RuntimeError("fused_color: backward through a forward that ran without grad")
        q, dev, n = ctx.q, acts.device, ctx.n
        g_sdf, g_nab, g_rgb = g_out[0], g_out[1], (g_out[2] if ctx.rad else None)
        # one zero-fill for the table gradient (or the step's shared one), one for the small tensors (views of a flat buffer)
        sizes = [int(torch.Size(s).numel()) for s in ctx.shapes[1:]]
        small = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        if q.table_grad is None:
            d_grid = torch.zeros(ctx.shapes[0], dtype=torch.float32, device=dev)
        else:
            d_grid = q.table_grad.take(ctx.shapes[0], dev)            # handed on by the table's SharedTableGrad.route node
        grads, o = [d_grid], 0
        for sh, k in zip(ctx.shapes[1:], sizes):
            grads.append(small[o:o + k].view(sh))
            o += k
        # the code gradient: of the op's h_appear input, or into the step's buffer (ColorQuery.appear_grad)
        ng = ctx.needs_input_grad
        d_ha = torch.zeros(ctx.ha_shape, dtype=torch.float32, device=dev) if ng[4] else None
        appear = (d_ha, None) if d_ha is not None else q.appear_grad
        # the gradients of learnable rays and view directions (summed per ray in the call)
        zeros3 = lambda want, like: torch.zeros(like.shape, dtype=torch.float32, device=dev) if want else None
        d_vd, d_ro, d_rd = zeros3(ng[3] and ctx.rad, ctx.vd), zeros3(ng[5], q.rays_o), zeros3(ng[6], q.rays_d)
        ret = (None,) * 3 + (d_vd, d_ha, d_ro, d_rd, None, (d_grid if q.table_grad is None else None)) + tuple(grads[1:])
        if g_sdf is None and g_nab is None and g_rgb is None:
            return ret
        c = lambda g: None if g is None else g.contiguous().float()
        g_sdf, g_nab, g_rgb = c(g_sdf), c(g_nab), c(g_rgb)
        dh = torch.empty(n, h_tile_cols(q.meta.n_pseudo_levels), dtype=torch.float32, device=dev) if g_rgb is not None else None
        P = L.ptr
        ag = [P(g) for g in grads] + [None] * (11 - len(grads))          # d_R* / d_rb*: NULL without the radiance net's parameters
        args = (q.meta.c_ref, P(q.grid16, "f16"), ctypes.byref(q.net), None, P(q.rays_o, "f32"), P(q.rays_d, "f32"), P(ctx.ridx, "i64"), P(ctx.t, "f32"),
                L.c_i64(n), L.c_level(q.ml), P(acts[0]), P(acts[1]), *([P(acts[2]), P(acts[3])] if ctx.rad else [None, None]), P(rgb, allow_none=True),
                P(g_sdf, allow_none=True), P(g_nab, allow_none=True), P(g_rgb, allow_none=True), P(dh, allow_none=True), *ag)
        # the ray targets: the op's ray inputs (rows in ray order), or the step's buffers (ColorQuery.ray_grad, through its ray map)
        ro_t, rd_t, vd_t, ray_map = (d_ro, d_rd, d_vd, None) if q.ray_grad is None else q.ray_grad
        rays = ro_t is not None or rd_t is not None or (vd_t is not None and g_rgb is not None)
        with L.KERNEL_TIMER.time("fused_color_bwd", n):
            if rays:
                ha = appear if (appear is not None and g_rgb is not None) else (None, None)
                ha_rows = torch.empty(n, 8, dtype=torch.float32, device=dev) if ha[0] is not None else None
                ray_rows = torch.empty(n, 36, dtype=torch.float32, device=dev)      # per-sample ray rows and radiance input gradients
                ray_map = ha[1] if ray_map is None else ray_map
                L.call(L.lib().nsb_fused_color_bwd_grads, "fused_color_bwd_grads", *args, P(ctx.vd, "f32", allow_none=True),
                       P(ha_rows, allow_none=True), P(ray_map, "i64", allow_none=True), P(ha[0], "f32", allow_none=True), P(ray_rows),
                       P(ro_t, allow_none=True), P(rd_t, allow_none=True), P(vd_t if g_rgb is not None else None, allow_none=True), L.stream_ptr(),
                       count=q.count, level=q.ml)
            elif appear is not None and g_rgb is not None:
                ha_rows = torch.empty(n, 8, dtype=torch.float32, device=dev)        # per-sample code gradients, summed per ray in the call
                L.call(L.lib().nsb_fused_color_bwd_appear, "fused_color_bwd_appear", *args, P(ha_rows), P(appear[1], "i64", allow_none=True),
                       P(appear[0], "f32"), L.stream_ptr(), count=q.count, level=q.ml)
            else:
                L.call(L.lib().nsb_fused_color_bwd, "fused_color_bwd", *args, L.stream_ptr(), count=q.count, level=q.ml)
        return ret


def fused_color(model, ridx, t, rays_o, rays_d, view_dirs=None, h_appear=None, *, nablas_has_grad=True, collect=None, with_rgb=True):
    """-> dict(sdf [n], nablas [n,3], rgb [n,3] (with_rgb only), x [n,3]).  Gradients flow to the table and the decoder, and with rgb to the
    radiance net, and to h_appear [R, n_appear], rays_o, rays_d [R, 3] and view_dirs [R, 3] if they require grad (the samples of a ray must
    then be consecutive, as packed samples are, for the per-ray sums to be deterministic; the depths t are constants)."""
    s = model.implicit_surface
    d = s.decoder.layers
    params = (s.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias)
    if with_rgb:
        r = model.radiance_net.blocks.layers
        params += (r[0].weight, r[0].bias, r[1].weight, r[1].bias, r[2].weight, r[2].bias)
    grid16, net, held = model._fused_color_state() if with_rgb else model._fused_geometry_state()
    q = ColorQuery(s.encoding.meta, grid16, net, held, rays_o.detach().contiguous().float(), rays_d.detach().contiguous().float(), s._ml(model.max_level),
                   collect, None)
    ha = None if (h_appear is None or not with_rgb) else h_appear.contiguous().float()
    vd = view_dirs.contiguous().float() if with_rgb else None
    ro, rd = (rays_o, rays_d) if (rays_o.requires_grad or rays_d.requires_grad) else (None, None)
    keep = torch.is_grad_enabled() and (any(p.requires_grad for p in params) or any(v is not None and v.requires_grad for v in (ha, vd, ro, rd)))
    out = _FusedColor.apply(q, ridx.reshape(-1).contiguous().long(), t.detach().reshape(-1).contiguous().float(), vd, ha, ro, rd, keep, *params)
    sdf, nab, x = out[0], out[1], out[-1]
    if not nablas_has_grad:
        nab = nab.detach()
    ret = dict(sdf=sdf, nablas=nab, x=x)
    if with_rgb:
        ret["rgb"] = out[2]
    return ret
