"""The NeuS step with every data-dependent size kept ON THE DEVICE: no host read, no `.item()`, no `nonzero()` -- so a whole
fwd+bwd step can be captured in ONE CUDA graph and replayed with a single launch (`StaticFrame`).

Same kernels, same values as `graphics.neus._query_fused` + `fields.neus.volume_integration` (reference:
nr3d_lib/graphics/neus/neus_ray_query.py:732-1104, app/renderers/single_volume_renderer.py:73-102,136-460): the only difference
is where the sizes live; the settings (`graphics.neus.query_config`) and the up-sampling (`graphics.neus.upsample_boundary`) are
shared code.  The reference reads ~25 sizes back per `ray_query` (SURVEY.md §8a a9); `_query_fused` reads three (+ one in the
backward); here the three scans leave their totals in a device block `cnt` (layout: include/neuralsim_b200.h, nsb_query_counts),
every buffer is allocated at a fixed CAPACITY and every kernel processes `min(capacity, *count)` items (nsb_bind_device_counts).
Capacities: rays -> R (the chunk), boundary samples -> R (n_coarse + 1 + sum n_fine), marched / merged samples -> `march_cap`,
samples kept by the compression -> `kept_cap`.  If a frame needs more than a capacity the step renders nothing and raises bit 0 / 1 of
cnt[20]; `StaticFrame.check()` reads that flag (one D2H, whenever the caller wants it) and `StaticFrame` re-captures with larger arenas.

tests/test_static_gpu.py: images bit-equal to the host-sized path, gradients equal up to the order of the fp32 atomics.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn.functional as F

from .. import _lib as L
from ..fields.fused_color import ColorQuery, SharedTableGrad, _FusedColor, color_net_c
from ..fields.networks import sdf_bwd, sdf_decoder_c, sdf_fwd
from .neus import query_config, upsample_boundary
from .raysample import batch_sample_step_linear
from . import neus_fused as NF
from . import perturb as PT
from .pose import FramePose
from .. import torch_rng as TR

__all__ = ["render_static", "StaticFrame", "CNT_SLOTS", "static_volume_buffer"]

CNT_SLOTS = dict(n_rays=0, pairs=2, marched_raw=3, hit_raw=4, kept_raw=6, kept_rays_raw=7, nonzero=9, marched=12, hit=13, fine0=14,
                 boundary=18, kept=19, overflow=20, kept_rays=21, merged0=22, rays_if_kept_fits=26, row_len=27)
# "auto": small batches march once and copy (nsb_ray_marching_record + nsb_march_compact) when the per-ray record fits this many bytes;
# "0": always the two-round march; "1": always the recorded march.  Same samples bit for bit either way.
MARCH_ONEPASS = "auto"
MARCH_ONEPASS_MAX_BYTES = 64 << 20


def march_onepass(n_rays, max_steps):
    if MARCH_ONEPASS == "0":
        return False
    return MARCH_ONEPASS == "1" or 4 * int(n_rays) * int(max_steps) <= MARCH_ONEPASS_MAX_BYTES


_slot = L.slot


def _call(fn, what, cnt, k0, k1, *args):
    """one launch with the counts cnt[k0] (and cnt[k1]) of the step's count block (_lib.call)"""
    L.call(fn, what, *args, count=(cnt, k0) if k1 is None else (cnt, k0, k1))


def _scan(counts, cnt, slot, *, first=None, info2=None, index=None, pack=None, src=None, nz_src=None, ws=None):
    """neus_fused.scan_launch with the totals left in cnt[slot], cnt[slot + 1] (no host hand-off)"""
    NF.scan_launch(counts, _slot(cnt, slot), first=first, info2=info2, index=index, pack=pack, src=src, nz_src=nz_src, ws=ws)


def _block_order(rays_inds, via, n_rays, cnt, slot):
    """the 8 x 4 pixel-block order of the cnt[slot] live packs on pixels rays_inds[via[p]] (neus_fused.ray_block_order; the row length and
    the coherence test are the ray test's, in cnt)"""
    return NF.ray_block_order(rays_inds, via, n_rays, _slot(cnt, CNT_SLOTS["pairs"]), _slot(cnt, CNT_SLOTS["row_len"]), count=(cnt, slot))


def _query_counts(cnt, phase, n_coarse1, num_fine, march_cap, kept_cap):
    nf = (ctypes.c_int32 * max(len(num_fine), 1))(*[int(n) for n in num_fine])
    L.check(L.lib().nsb_query_counts(ctypes.c_void_p(cnt.data_ptr()), L.c_i32(phase), L.c_i32(n_coarse1), nf, L.c_i32(len(num_fine)),
                                     L.c_i64(march_cap), L.c_i64(kept_cap), L.stream_ptr()), "query_counts")


# ---------------------------------------------------------------------------------------------------------------- autograd pieces
class _StaticBoundary(torch.autograd.Function):
    """boundary SDF query -> alpha -> compression -> gather of the kept samples (fields/networks.py:_FusedSDF + graphics/neus_fused.py:
    neus_alpha_compact with device-resident sizes).  -> alpha of the K kept samples (differentiable in inv_s and the SDF parameters) and
    their depth, ray, the kept packs and their pixels.  The backward runs over the kept samples only: d_alpha is zero everywhere else, so
    the kept-interval adjoint (nsb_neus_alpha_backward_kept) lists the boundary samples with a non-zero d_sdf -- per-ray counts, a scan
    over the rays, the list -- and k_sdf_bwd_tc walks that list; nothing boundary-wide is filled, scattered, flagged or scanned."""

    @staticmethod
    def forward(ctx, st, d1, pinfo, ridx_all, order_b, rays_inds, kept_cap, qc, inv_s, grid, W1, b1, W2, b2):
        """ridx_all None: coherent rays, the query walks the packs in the 8 x 4 pixel-block order order_b; else sample by sample"""
        R, dev, cnt = pinfo.shape[0], d1.device, st.cnt
        sdf = torch.empty(d1.numel(), dtype=torch.float32, device=dev)
        with L.KERNEL_TIMER.time("fused_sdf_fwd", d1.numel()):
            if ridx_all is None:
                sdf_fwd(st.meta, st.grid16, st.dec, sdf, st.ml, rays_o=st.rays_o, rays_d=st.rays_d, t=d1, packs=(pinfo, None, order_b), collect=st.collect,
                        count=(cnt, CNT_SLOTS["n_rays"]))
            else:
                sdf_fwd(st.meta, st.grid16, st.dec, sdf, st.ml, rays_o=st.rays_o, rays_d=st.rays_d, t=d1, ridx=ridx_all, collect=st.collect,
                        count=(cnt, CNT_SLOTS["boundary"]))
        inv_c = inv_s.detach().contiguous().float().reshape(1)
        alpha, sel, steps = NF.alpha_forward(sdf, pinfo, inv_c, 1e-4, 0.0, count=(cnt, CNT_SLOTS["n_rays"]))
        first = torch.empty(R, dtype=torch.int32, device=dev)
        nidx = torch.empty(R, dtype=torch.int64, device=dev)
        pinfo_kept = torch.empty(R, 2, dtype=torch.int64, device=dev)
        rays_inds_hit = torch.empty(R, dtype=torch.int64, device=dev)
        _scan(steps, cnt, CNT_SLOTS["kept_raw"], first=first, index=nidx, pack=pinfo_kept, src=rays_inds, nz_src=rays_inds_hit, ws=st.ws[2])
        _query_counts(cnt, 1, *qc)
        pidx, ridx_k, t_k, alpha_k = NF.compact_samples(sel, pinfo, first, steps, alpha, kept_cap, d1=d1, count=(cnt, CNT_SLOTS["rays_if_kept_fits"]))
        ctx.st, ctx.saved = st, (d1, sdf, inv_c, pinfo, nidx, pinfo_kept, pidx)
        ctx.shapes = (inv_s.shape, grid.shape, W1.shape, b1.shape, W2.shape, b2.shape)
        ctx.mark_non_differentiable(t_k, ridx_k, pinfo_kept, rays_inds_hit)
        return alpha_k, t_k, ridx_k, pinfo_kept, rays_inds_hit

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_alpha, _gt, _gr, _gp, _gi):
        st, (d1, sdf, inv_c, pinfo, nidx, pinfo_kept, pidx) = ctx.st, ctx.saved
        dev, R, S, K = sdf.device, pinfo.shape[0], sdf.numel(), pidx.numel()
        inv_shape, gs, w1s, b1s, w2s, b2s = ctx.shapes
        d_grid = st.table_grad.take(gs, dev)           # shared with the colour query's backward, handed on by SharedTableGrad.route
        ks = [int(torch.Size(x).numel()) for x in (w1s, b1s, w2s, b2s)]
        small = torch.zeros(1 + sum(ks), dtype=torch.float32, device=dev)
        d_inv, o = small[:1], 1
        d_W1, d_b1 = small[o:o + ks[0]].view(w1s), small[o + ks[0]:o + ks[0] + ks[1]].view(b1s)
        o += ks[0] + ks[1]
        d_W2, d_b2 = small[o:o + ks[2]].view(w2s), small[o + ks[2]:].view(b2s)
        P, cnt, lib = L.ptr, st.cnt, L.lib()
        if g_alpha is not None:
            g = g_alpha.contiguous().float()
            d_sdf = torch.empty(S, dtype=torch.float32, device=dev)            # written at the listed samples only
            ray = torch.empty(S, dtype=torch.int64, device=dev)                # (the same)
            counts = torch.empty(R, dtype=torch.int32, device=dev)
            a = (P(pinfo, "i64"), P(nidx, "i64"), P(pinfo_kept, "i64"), P(pidx, "i64"))
            _call(lib.nsb_neus_alpha_backward_kept, "neus_alpha_backward_kept", cnt, CNT_SLOTS["kept_rays"], None, P(sdf, "f32"), *a, L.c_i64(R),
                  P(inv_c, "f32"), P(g, "f32"), P(d_sdf), P(counts), P(d_inv), L.stream_ptr())
            offs = torch.empty(R, dtype=torch.int32, device=dev)
            _scan(counts, cnt, CNT_SLOTS["nonzero"], first=offs, ws=st.ws[3])
            n_list = min(S, 2 * K)                         # at most a kept sample and the one after it per kept sample
            keep = torch.empty(n_list, dtype=torch.int64, device=dev)
            _call(lib.nsb_neus_alpha_backward_kept_list, "neus_alpha_backward_kept_list", cnt, CNT_SLOTS["kept_rays"], None, *a, P(g, "f32"),
                  P(d_sdf, "f32"), P(offs, "i32"), L.c_i64(R), P(keep), P(ray), L.stream_ptr())
            # with the ray gradient, the listed samples' rows (one per list slot: the scratch is sized n_list) are summed per ray -- a ray's
            # listed samples are consecutive, so the sums are deterministic -- into the step's accumulators (st.ray_grads)
            with L.KERNEL_TIMER.time("fused_sdf_bwd", n_list):
                sdf_bwd(st.meta, st.grid16, st.dec, d_sdf, n_list, st.ml, (d_grid, d_W1, d_b1, d_W2, d_b2), rays=(st.rays_o, st.rays_d, ray, d1), keep=keep,
                        count=(cnt, CNT_SLOTS["nonzero"]), ray_grads=st.ray_grads)
        return (None,) * 8 + (d_inv.reshape(inv_shape), None, d_W1, d_b1, d_W2, d_b2)


class _RayGradAdjoint(torch.autograd.Function):
    """identity on a scalar leaf that requires grad (the anchor of the table's route node, SharedTableGrad.route).  Autograd runs this
    backward after the route node's, which runs after every node that reads the routed table -- the boundary and the colour query -- so
    here both have added their ray rows into the step's accumulators, and `run` maps them onto the caller's rays
    (nsb_gather_rays_backward)."""

    @staticmethod
    def forward(ctx, run, anchor):
        ctx.run = run
        return anchor.view_as(anchor)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, _g):
        ctx.run()
        return None, None


class _State:
    """what the kernels of one static step share"""
    __slots__ = ("meta", "grid16", "dec", "net", "held", "rays_o", "rays_d", "ml", "collect", "cnt", "ws", "table_grad", "ray_grads")


def _fp16_images(model, radiance=True):
    """fp16 images of the masters, re-cast INSIDE the step (a captured graph must not rely on a host-side version check).  radiance=False:
    the table and the decoder only, and a net struct without a radiance net (rad_width = 0) for the geometry-only colour query"""
    s = model.implicit_surface
    d = s.decoder.layers
    ps = [s.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias]
    b = model.radiance_net.blocks.layers if radiance else None
    if radiance:
        ps += [b[0].weight, b[0].bias, b[1].weight, b[1].bias, b[2].weight, b[2].bias]
    # one multi-tensor cast for the small tensors (a launch each otherwise: at 4096 rays per step the step is launch-bound), one for the table
    t = [torch.empty(p.shape, dtype=torch.half, device=p.device) for p in ps]
    with torch.no_grad():
        t[0].copy_(ps[0].detach())
        torch._foreach_copy_(t[1:], [p.detach() for p in ps[1:]])
    return t, sdf_decoder_c(t[1:5], d), color_net_c(t[1:], d, b, model._nablas_fac()), ps


def render_static(model, rays_o, rays_d, rays_h_appear=None, *, near=None, far=None, march_cap, kept_cap, coherent=False, with_rgb=True, with_normal=True,
                  perturb=False, training=None, depth_use_normalized_vw=True, cnt=None, d_h_appear=None, d_rays=None, max_level_dev=None,
                  ray_grad_hook=None, rng_dev=None):
    """One chunk of rays, ray test -> query -> integration, without a host read.  -> (rendered dict of whole-chunk images, cnt int64[32]).
    `coherent`: image-ordered rays (the boundary / fine queries then walk the samples ray-tiled) -- a host decision here (the host-sized
    path measures it in the ray-test kernel).  `d_h_appear` [R, n_appear] (optional): zero-filled here, and the backward pass writes the
    gradient of the codes rays_h_appear into it, in the caller's ray order (the codes themselves are read detached).  `d_rays` =
    (d_rays_o, d_rays_d) [R, 3] (optional): the same for the rays -- zero-filled here, and the backward pass writes the gradient of the
    loss to rays_o and rays_d (the caller's frame and order; 0 for rays that miss the box or keep no sample), the depths held constant
    as on the host-sized path.  `max_level_dev` (optional): a device int32 scalar every LoTD kernel of the step reads its level bound from
    (nsb_bind_device_max_level), so that a captured step follows a level schedule; None: the model's level at this call, fixed in a capture.
    `ray_grad_hook` (optional, with d_rays): called in the backward pass right after d_rays is written (the pose adjoint of StaticFrame).
    `perturb`: stratified coarse depths and up-sampling quantiles, the values torch's CUDA generator gives the host-sized path
    (graphics/neus.py:_query_fused) from the same state: the kernels of graphics/perturb.py draw them against the step's device counts.
    `rng_dev` = int64 [2] (seed, offset) on the device, the state the step draws from (StaticFrame refills it before every replay); None:
    the default CUDA generator's state at this call, which is then advanced by the step's reservation (perturb.reservation) -- eager calls
    only, as a capture would fix the state."""
    P, lib = L.ptr, L.lib()
    if with_rgb and getattr(model, "radiance_net", None) is None:
        raise RuntimeError("render_static(with_rgb=True): the model has no radiance net (radiance_cfg=False); render it with with_rgb=False")
    training = model.training if training is None else training
    R, dev = rays_o.shape[0], rays_o.device
    cfg = query_config(**(model.ray_query_cfg.get("query_param", {}) or {}), upsample_s_divisor=model.upsample_s_divisor)
    if cfg.num_coarse <= 0:
        raise RuntimeError("render_static: num_coarse=0 is not built (the boundary samples are the coarse and the fine ones)")
    nc1, max_steps = cfg.num_coarse + 1, cfg.max_steps
    march_cap, kept_cap = int(march_cap), int(kept_cap)
    if perturb:
        if ((model.ray_query_cfg.get("query_param", {}) or {}).get("march_cfg", {}) or {}).get("perturb_before_march", False):
            raise RuntimeError("render_static(perturb=True): march_cfg.perturb_before_march=True is not built; use the host-sized path")
        reserve = PT.reservation(R, cfg, TR.grid_cap(dev))
        if rng_dev is None:
            rng_dev = TR.take(TR.cuda_generator(None, dev), reserve)
        draws_coarse, draws_stage = PT.step_draws(CNT_SLOTS, nc1, cfg.num_fine)
    if cnt is None:
        cnt = torch.zeros(32, dtype=torch.int64, device=dev)
    else:
        cnt.zero_()
    st = _State()
    st.cnt = cnt
    wsb = (NF._scan_ws_bytes() + 255) // 256 * 256
    st.ws = torch.zeros(4, wsb, dtype=torch.uint8, device=dev)          # the zeroed workspaces of the step's four scans, one fill
    st.table_grad = SharedTableGrad()          # the boundary and colour backward nodes scatter into one table gradient
    with torch.no_grad():
        t16, st.dec, st.net, masters = _fp16_images(model, radiance=with_rgb)
        st.held, st.grid16 = t16, t16[0]
        st.meta = model.implicit_surface.encoding.meta
        st.ml = max_level_dev if max_level_dev is not None else model.implicit_surface._ml(model.max_level)
        st.collect = model.accel.occ.collect_struct() if training else None
        # ---------------- ray test (fields/space.py:_ray_test_fused without the host read)
        c3, r3 = model.space._center_radius_c()
        tested = NF.ray_test_aabb(rays_o, rays_d, c3, r3, near, far, _slot(cnt, CNT_SLOTS["pairs"]), _slot(cnt, CNT_SLOTS["row_len"]))
        rays_inds = torch.empty(R, dtype=torch.int64, device=dev)
        _scan(tested[4], cnt, CNT_SLOTS["n_rays"], index=rays_inds, ws=st.ws[0])
        # the boundary query walks its packs (the rays that passed) in 8 x 4 pixel blocks (csrc/neus_glue.cu: k_ray_block_order)
        order_b = _block_order(rays_inds, None, R, cnt, CNT_SLOTS["n_rays"]) if coherent else None
        # only the radiance head reads appearance codes: rays that render no rgb gather none
        ha = rays_h_appear.detach().contiguous().float() if (with_rgb and rays_h_appear is not None and model.use_h_appear) else None
        if ha is None and with_rgb and model.use_h_appear:
            ha = torch.zeros(R, model.radiance_net.blocks.layers[0].in_features - 22 - model.implicit_surface.encoding.out_features, device=dev)
        n_ha = ha.shape[1] if ha is not None else 0
        rbuf = torch.zeros(R * (8 + n_ha), device=dev)     # the compacted rays in ONE zero-filled allocation (rows beyond the live count stay 0)
        o_c, d_c = rbuf[:3 * R].view(R, 3), rbuf[3 * R:6 * R].view(R, 3)
        n_c, f_c = rbuf[6 * R:7 * R], rbuf[7 * R:8 * R]
        ha_c = rbuf[8 * R:].view(R, n_ha) if ha is not None else None
        if d_h_appear is not None:
            if ha is None:
                raise RuntimeError("render_static(d_h_appear=...): the colour query reads no appearance codes (with_rgb=False or a model without them)")
            d_h_appear.zero_()                              # the backward adds each kept ray's sum once into its row
        NF.gather_rays(rays_inds, R, tested[:4], (o_c, d_c, n_c, f_c), ha, ha_c, count=(cnt, CNT_SLOTS["n_rays"]))
        st.rays_o, st.rays_d = o_c, d_c
        vnorm = d_c.norm(dim=-1).clamp_min(1.0e-10) if with_rgb else None         # held constant, as the host-sized path holds it
        view_dirs = (d_c / vnorm.unsqueeze(-1)).contiguous() if with_rgb else None
        st.ray_grads, ray_g = None, None
        if d_rays is not None:
            # the backward passes add each compacted ray's gradient to its o_c, d_c (and view direction) at the ray's row in the caller's
            # order -- the ray map of the codes, which the colour entry point shares -- and the adjoint of the ray test then divides by r
            for t in d_rays:
                t.zero_()
            ray_g = torch.zeros(3 if with_rgb else 2, R, 3, device=dev)
            ray_g = (ray_g[0], ray_g[1], ray_g[2] if with_rgb else None)           # g_o, g_d, g_vd (no view term without rgb)
            st.ray_grads = (ray_g[0], ray_g[1], rays_inds)
        # ---------------- coarse samples + march
        if perturb:           # rows past the ray count are not read (nsb_assemble_boundary)
            coarse = PT.coarse_depths(n_c, f_c, nc1, rng_dev, cnt, draws_coarse, torch.empty(R, nc1, device=dev))
        else:
            coarse = batch_sample_step_linear(n_c, f_c, nc1, prefix_shape=[R]).contiguous()
        occ_grid = model.accel.occ.occ_grid
        res = occ_grid.shape[-3:]
        g8 = occ_grid.contiguous().view(torch.uint8)
        bits = NF.pack_occ_bits(occ_grid)
        roi = torch.tensor([-1, -1, -1, 1, 1, 1], dtype=torch.float32, device=dev) if getattr(model, "_static_roi", None) is None else model._static_roi
        model._static_roi = roi
        margs = NF.march_args(o_c, d_c, n_c, f_c, roi, occ_grid, cfg.step_size, cfg.max_step_size, cfg.dt_gamma, max_steps)
        num_steps = torch.empty(R, dtype=torch.int32, device=dev)
        # small batches: a march costs the latency of its longest ray -> march ONCE, recording the samples per ray, and copy (csrc/march.cu)
        rec_t = torch.empty(R * max_steps, dtype=torch.float32, device=dev) if march_onepass(R, max_steps) else None
        with L.KERNEL_TIMER.time("march", R):
            if rec_t is not None:
                _call(lib.nsb_ray_marching_record, "ray_marching_record", cnt, CNT_SLOTS["n_rays"], None, L.c_i64(R), P(o_c, "f32"), P(d_c, "f32"), P(n_c, "f32"),
                      P(f_c, "f32"), P(roi, "f32"), L.c_i32(res[0]), L.c_i32(res[1]), L.c_i32(res[2]), P(g8, "u8"), L.c_f32(cfg.step_size), L.c_f32(cfg.max_step_size),
                      L.c_f32(cfg.dt_gamma), ctypes.c_uint32(max_steps), P(num_steps), P(rec_t), P(bits), L.stream_ptr())
            else:
                NF.march_listed(margs, bits, num_steps=num_steps, count=(cnt, CNT_SLOTS["n_rays"]))
        info2 = torch.empty(R, 2, dtype=torch.int32, device=dev)
        ridx_hit = torch.empty(R, dtype=torch.int64, device=dev)
        pack_infos = torch.empty(R, 2, dtype=torch.int64, device=dev)
        _scan(num_steps, cnt, CNT_SLOTS["marched_raw"], info2=info2, index=ridx_hit, pack=pack_infos, ws=st.ws[1])
        _query_counts(cnt, 0, nc1, cfg.num_fine, march_cap, kept_cap)
        depth = torch.empty(march_cap, dtype=torch.float32, device=dev)
        ridx32 = torch.empty(march_cap, dtype=torch.int32, device=dev)
        with L.KERNEL_TIMER.time("march", R):
            if rec_t is not None:
                _call(lib.nsb_march_compact, "march_compact", cnt, CNT_SLOTS["hit"], None, P(rec_t, "f32"), ctypes.c_uint32(max_steps), P(info2, "i32"),
                      P(ridx_hit, "i64"), L.c_i64(R), P(depth), P(ridx32), L.stream_ptr())
            else:
                NF.march_listed(margs, bits, info2=info2, t_starts=depth, ridx=ridx32, ray_list=ridx_hit, n_list=R, count=(cnt, CNT_SLOTS["hit"]))
        ridx = ridx32.long()
        # ---------------- up-sampling (no grad)
        def sdf_on_rays(ridx_, t, packs, count):
            """the fused SDF query of the capacity-sized samples t (the counted ones are queried)"""
            sdf = torch.empty(t.numel(), dtype=torch.float32, device=dev)
            with L.KERNEL_TIMER.time("lotd_gather", t.numel()):
                if packs is None and t.dim() == 2:
                    ridx_ = ridx_.unsqueeze(-1).expand(t.shape).reshape(-1)
                sdf_fwd(st.meta, st.grid16, st.dec, sdf, st.ml, rays_o=o_c, rays_d=d_c, t=t.view(-1), ridx=ridx_, packs=packs, collect=st.collect, count=count)
            return sdf
        # the ray of every boundary sample: only the incoherent boundary query (one sample per row) reads it; everything else derives it
        d1, _mid, ridx_all, pinfo = upsample_boundary((ridx_hit, pack_infos, depth, ridx), o_c, d_c, coarse, cfg, sdf_on_rays,
                                                      (lambda via: _block_order(rays_inds, via, R, cnt, CNT_SLOTS["hit"])) if coherent else None,
                                                      table=(st.meta, st.grid16, st.dec, st.ml, st.collect), counts=(cnt, CNT_SLOTS), n_out=march_cap,
                                                      want_mid=False, want_ridx=not coherent, perturb=perturb,
                                                      sampler=(lambda i, dep, cdf, pi, nf: PT.invert_cdf(dep, cdf, pi, nf, rng_dev, cnt, draws_stage[i],
                                                                                                         torch.empty(R, nf, device=dev))) if perturb else None)
    # ---------------- boundary SDF (grad) -> alpha -> compression
    s = model.implicit_surface
    dl = s.decoder.layers
    inv_s = model.forward_inv_s()
    anchor = None
    if d_rays is not None:
        # after both backward nodes: the adjoint of the ray test, from the accumulators to the caller's rays (the anchor also makes the
        # nodes run when no parameter requires grad: a pose refined against a fixed model)
        def ray_adjoint():
            NF.gather_rays_backward(rays_inds, R, r3, ray_g, vnorm, d_rays, count=(cnt, CNT_SLOTS["n_rays"]))
            if ray_grad_hook is not None:
                ray_grad_hook()
        anchor = _RayGradAdjoint.apply(ray_adjoint, torch.zeros((), device=dev, requires_grad=True))
    table = st.table_grad.route(s.encoding.flattened_params, anchor)    # the table as both backward nodes' input
    if not isinstance(inv_s, torch.Tensor):
        inv_s = torch.tensor(float(inv_s), device=dev)
    alpha_k, t_k, ridx_k, pinfo_kept, rays_inds_hit = _StaticBoundary.apply(
        st, d1, pinfo, ridx_all, order_b, rays_inds, kept_cap,
        (nc1, cfg.num_fine, march_cap, kept_cap), inv_s, table, dl[0].weight, dl[0].bias, dl[1].weight, dl[1].bias)
    # ---------------- colour / normal query on the kept samples (none when neither is rendered: depth and mask need alpha alone)
    rgb = nab = x = None
    if with_rgb or with_normal:
        params = (table, dl[0].weight, dl[0].bias, dl[1].weight, dl[1].bias)
        if with_rgb:
            b = model.radiance_net.blocks.layers
            params += (b[0].weight, b[0].bias, b[1].weight, b[1].bias, b[2].weight, b[2].bias)
        keep_acts = torch.is_grad_enabled() and (any(p.requires_grad for p in params) or d_h_appear is not None or d_rays is not None)
        # the code (and ray) gradient of the compacted ray r goes to row rays_inds[r] of d_h_appear (and of the ray accumulators; the
        # kernels stop at the device counts)
        q = ColorQuery(st.meta, st.grid16, st.net, st.held, st.rays_o, st.rays_d, st.ml, st.collect, (cnt, CNT_SLOTS["kept"]), st.table_grad,
                       (d_h_appear, rays_inds) if d_h_appear is not None else None,
                       ray_g + (rays_inds,) if d_rays is not None else None)
        out = _FusedColor.apply(q, ridx_k, t_k, view_dirs, ha_c, None, None, keep_acts, *params)
        nab, x = out[1], out[-1]
        rgb = out[2] if with_rgb else None
        if not cfg.nablas_has_grad:
            nab = nab.detach()
    nab_i = nab if with_normal else None
    if nab_i is not None and not training:
        nab_i = F.normalize(nab_i.clamp(-1, 1), dim=-1)
    vw, m, d, c, nn_ = NF.composite(alpha_k, t_k, pinfo_kept, rgb=rgb, nablas=nab_i, normalize_depth=bool(depth_use_normalized_vw), ray_index=rays_inds_hit,
                                    n_rays=R, count=(cnt, CNT_SLOTS["kept_rays"]))
    rendered = dict(mask_volume=m, depth_volume=d)
    if with_rgb:
        rendered["rgb_volume"] = c
    if with_normal:
        rendered["normals_volume"] = nn_
    buffers = dict(opacity_alpha=alpha_k, t=t_k, rgb=rgb, nablas=nab, net_x=x, vw=vw, pack_infos_hit=pinfo_kept, rays_inds_hit=rays_inds_hit, ridx=ridx_k,
                   pack_infos_boundary=pinfo, march_pack_infos=pack_infos)
    return rendered, cnt, buffers


def sliced_volume_buffer(buffers, cnt):
    """The reference's packed `volume_buffer` (renderer_mixin.py:263-303) out of a static step's capacity-sized buffers: ONE host read of the
    counts, then views.  (Losses that read the buffer -- eikonal on `nablas` -- can use it; gradients flow through the views.)"""
    c = cnt.tolist()
    K, Pu = c[CNT_SLOTS["kept"]], c[CNT_SLOTS["kept_rays"]]
    if c[CNT_SLOTS["overflow"]]:
        raise RuntimeError(f"static step: arena overflow (flags {c[CNT_SLOTS['overflow']]}: 1 = marched samples, 2 = kept samples)")
    if K == 0:
        return dict(type="empty", rays_inds_hit=[])
    vb = dict(type="packed", rays_inds_hit=buffers["rays_inds_hit"][:Pu], pack_infos_hit=buffers["pack_infos_hit"][:Pu])
    for k in ("opacity_alpha", "t", "rgb", "nablas", "net_x", "vw"):
        if buffers[k] is not None:                           # rgb / nablas / net_x: None when the step did not query them
            vb[k] = buffers[k][:K]
    return vb


def static_volume_buffer(buffers, cnt):
    """The volume buffer a loss inside the captured step reads (StaticFrame(loss_on_ret=True)): the step's capacity-sized kept-sample
    buffers t, vw [kept_cap], rays_inds_hit, pack_infos_hit [R], ridx, with their sizes in the device count block `cnt` (CNT_SLOTS:
    "kept" samples, "kept_rays" rays).  No host read.  Its type "packed_static" is one the reference's losses refuse, so nothing reads
    the capacity-sized tensors as if they were exact-size."""
    return dict(type="packed_static", t=buffers["t"], vw=buffers["vw"], rays_inds_hit=buffers["rays_inds_hit"], pack_infos_hit=buffers["pack_infos_hit"],
                ridx=buffers["ridx"], cnt=cnt, CNT_SLOTS=CNT_SLOTS)


# ---------------------------------------------------------------------------------------------------------------- one-launch step
class StaticFrame:
    """fwd (+ loss + bwd) of one fixed-size ray batch as ONE CUDA graph launch.

        frame = StaticFrame(model, n_rays, loss_fn=lambda rendered: ..., near=0.01)
        loss = frame.step(rays_o, rays_d, rays_h_appear)        # device tensors (or pinned host tensors): copied into the graph's inputs
        frame.rendered["rgb_volume"], p.grad                    # static outputs / accumulated gradients
        frame.check()                                           # optional: one D2H of the counts; re-captures with larger arenas on overflow

    `h_appear_grad=True` (off by default: the graph is fixed at capture, and the step does a little more work): every step also writes
    `frame.d_h_appear` [n_rays, n_appear], the gradient of the loss with respect to the rays' appearance codes in the order they were
    passed (rows of rays that keep no sample are 0; each step overwrites it).  The codes are inputs the caller copies in, so the caller
    applies it to its own codes, e.g. `codes.backward(frame.d_h_appear)`.

    `ray_grad=True` (off by default, for the same reasons): every step also writes `frame.d_rays_o` and `frame.d_rays_d` [n_rays, 3], the
    gradient of the loss with respect to the rays passed, in their order and frame (world; the depths are held constant, as on the
    host-sized path; rows of rays that miss the box or keep no sample are 0; each step overwrites them).  The rays are copied in, so a
    trainer that refines its pose applies the gradient to the pose itself, outside the graph:

        o, d = pose_transform(pose, rays_o_cam, rays_d_cam)       # learnable rays
        loss = frame.step(o.detach(), d.detach(), codes)
        torch.autograd.backward([o, d], [frame.d_rays_o, frame.d_rays_d])      # -> pose.grad

    `pose=CameraPoses(...)` (graphics/pose.py; off by default) moves that pose into the graph: the frame owns static buffers
    `frame.dirs` [n_rays, 3] (camera-space directions) and `frame.pidx` [n_rays] (int64 pose indices), filled by `set_rays(dirs, pidx)` or
    by `step(dirs=..., pidx=...)`; the graph first builds `frame.rays_o` / `frame.rays_d` from them (nsb_pose_rays) and, when dq or dt
    requires grad, ends its backward with the pose adjoint (nsb_pose_rays_backward), which ADDS the gradient into `dq.grad` / `dt.grad`:

        frame = StaticFrame(model, n_rays, loss_fn, near=0.01, pose=poses)
        loss = frame.step(rays_h_appear=codes, dirs=dirs_cam, pidx=pidx)      # -> poses.dq.grad, poses.dt.grad; one graph launch

    The gradient buffers stay the ones the graph writes: `step()` re-attaches them before each replay (a `.grad` set to None counts as
    zeros, another tensor is copied in), and `zero_grads=True` zeroes them inside the graph with the model's.  `ray_grad=True` still fills
    `d_rays_o` / `d_rays_d`.  Switching `requires_grad` of dq / dt (the reference's `enable_after`) re-captures once: the graph without
    grad runs the forward kernel only.

    `loss_on_ret=True` (off by default: then `loss_fn(rendered)`): `loss_fn` receives the reference-shaped `ret = {"rendered": ...,
    "volume_buffer": vb}`, vb = static_volume_buffer(...) (the capacity-sized kept-sample buffers and their device counts), so a loss on
    the per-sample buffers -- neuralsim_b200.loss.LidarLoss -- runs inside the captured step.  Per-step inputs of such a loss are static
    buffers the caller refreshes before `step()` (LidarLoss.set_step).

    The LoTD level bound follows the model (`model.max_level`, else the encoding's annealed level) from replay to replay: `step()` refills a
    device scalar the kernels read (`max_level_dev`), as it refills the variance schedule's weight, so one capture serves a whole level
    schedule (LoTDEncoding's `anneal_cfg`; the trainer calls `model.training_before_per_step(it)` before `step()`).  A new level moves the
    surface, so a step may need more samples than the arenas were sized for; `check()` then re-sizes them from the current level.

    `perturb=True` (off by default) trains with stratified samples, as the shipped StreetSurf configs do (`renderer.train.perturb`): the
    graph draws the coarse depths and the up-sampling quantiles in its kernels from torch's CUDA generator (`generator`, else the default
    one of the model's device; graphics/perturb.py).  `step()` writes the generator's state into the device block `frame.rng` and advances
    it by `frame.rng_reservation` (torch_rng.take: no synchronisation), so a replay draws exactly what the host-sized perturbed step draws
    from the same state, and its images, loss and gradients are that step's; runs of the two drift apart (torch_rng.py).  `check()`'s
    retry replays the same draw.

    `sampler=` (off by default; needs a loss_fn) draws every batch inside the graph: a CameraSampler (neuralsim_b200/importance.py;
    `step(cam=k)`) or a LidarSampler (neuralsim_b200/lidar_sampler.py; `step(frame_ind=f)`).  `step()` fills the sampler's index and
    generator block (its draws first, the perturbed ones after them); the replay draws the batch into the frame's inputs and
    `frame.ground_truth`, renders, calls `loss_fn(rendered_or_ret, frame.ground_truth)` and runs the backward (the samplers' `attach`,
    `select`, `draw`, `loss` and `check` say what else each one needs, writes and updates).

    The first call probes the sizes with the host-sized path (SingleVolumeRenderer.ray_query, no grad), sizes the arenas with `slack`,
    warms up and captures.  Gradients are accumulated into `p.grad` (kept in place; `zero_grads=True` or a `pre_hook` zeroes them inside the graph).
    Capture precondition (PyTorch): no autograd graph of an EARLIER backward on the default stream may still be referenced (a kept loss / rendered
    tensor): it pins the parameters' AccumulateGrad nodes to the default stream, which cannot take part in a capture."""

    def __init__(self, model, n_rays, loss_fn=None, *, near=None, far=None, with_rgb=True, with_normal=True, slack=1.5, march_cap=None, kept_cap=None,
                 coherent=None, use_graph=True, zero_grads=False, h_appear_dim=None, pre_hook=None, h_appear_grad=False, ray_grad=False,
                 loss_on_ret=False, pose=None, perturb=False, generator=None, sampler=None):
        self.model, self.n_rays, self.loss_fn, self.loss_on_ret = model, int(n_rays), loss_fn, bool(loss_on_ret)
        self.near, self.far, self.with_rgb, self.with_normal, self.slack = near, far, with_rgb, with_normal, float(slack)
        self.march_cap, self.kept_cap, self.coherent = march_cap, kept_cap, coherent
        self.use_graph, self.zero_grads, self.pre_hook = use_graph, zero_grads, pre_hook
        dev = model.device
        self.device = dev
        self.rays_o = torch.zeros(self.n_rays, 3, device=dev)
        self.rays_d = torch.zeros(self.n_rays, 3, device=dev)
        # the radiance input is [x(3), SH4(v) (16), n(3), h(2L), h_appear]
        na = h_appear_dim if h_appear_dim is not None else (
            model.radiance_net.blocks.layers[0].in_features - 22 - model.implicit_surface.encoding.out_features if model.use_h_appear else 0)
        self.h_appear = torch.zeros(self.n_rays, na, device=dev) if na > 0 else None
        if h_appear_grad and (self.h_appear is None or not with_rgb or not model.use_h_appear):
            raise RuntimeError("StaticFrame(h_appear_grad=True): the step renders no rgb from appearance codes")
        self.d_h_appear = torch.zeros(self.n_rays, na, device=dev) if h_appear_grad else None
        self.d_rays_o = self.d_rays_d = None
        if ray_grad:
            self.d_rays_o, self.d_rays_d = torch.zeros(2, self.n_rays, 3, device=dev).unbind(0)
        self.cnt = torch.zeros(32, dtype=torch.int64, device=dev)
        self.perturb, self.rng, self.rng_reservation, self._gen = bool(perturb), None, 0, None
        if generator is not None and not self.perturb and sampler is None:
            raise RuntimeError("StaticFrame(generator=...): the generator is read only with perturb=True or a sampler")
        if self.perturb or sampler is not None:
            self._gen = TR.cuda_generator(generator, dev)
        if self.perturb:
            cfg = query_config(**(model.ray_query_cfg.get("query_param", {}) or {}), upsample_s_divisor=model.upsample_s_divisor)
            self.rng_reservation = PT.reservation(self.n_rays, cfg, TR.grid_cap(dev))
            self.rng = torch.zeros(2, dtype=torch.int64, device=dev)
        self.max_level_dev = torch.zeros((), dtype=torch.int32, device=dev)
        self.pose, self._pose = pose, (FramePose(pose, self.n_rays, dev) if pose is not None else None)
        if pose is not None:
            self.dirs, self.pidx = self._pose.dirs, self._pose.pidx
        self.sampler = sampler
        if sampler is not None:
            if loss_fn is None or sampler.device != dev:
                raise RuntimeError(f"StaticFrame(sampler=...): needs a loss_fn, and the sampler on the model's device {dev} (it is on {sampler.device})")
            self._rng_sampler = torch.zeros(2, dtype=torch.int64, device=dev)      # the sampler's (seed, offset); it chains its end into self.rng
            self.sampler_reservation = sampler.attach(self)
        self.graph, self.loss, self.rendered, self.buffers, self._occ_captured, self._grad_captured = None, None, None, None, None, None
        self.captures, self._warming = 0, False

    # -- sizes
    @torch.no_grad()
    def _probe(self):
        """sizes of this batch from the host-sized path (two host reads): M (merged marched samples), K (kept), coherence"""
        from ..renderer import SingleVolumeRenderer
        r = SingleVolumeRenderer(dict(near=self.near, far=self.far, with_rgb=self.with_rgb, with_normal=self.with_normal))
        r.train(self.model.training)
        out = r.ray_query(self.model, self.rays_o, self.rays_d, self.h_appear, return_buffer=True, return_details=True)
        det, vb = out.get("details", {}), out["volume_buffer"]
        nf = query_config(**(self.model.ray_query_cfg.get("query_param", {}) or {}), upsample_s_divisor=self.model.upsample_s_divisor).num_fine
        M = int(det["march.num_per_ray"].sum()) if "march.num_per_ray" in det else 0
        n_hit = int(det["march.num_per_ray"].shape[0]) if "march.num_per_ray" in det else 0
        K = int(vb["t"].shape[0]) if vb.get("type") == "packed" else 0
        return M + n_hit * sum(nf[:-1]), K, bool(out["ray_tested"].get("rays_coherent", False))

    def _size(self, grow=1.0):
        need_m, need_k, coh = self._probe()
        if self.coherent is None:
            self.coherent = coh
        floor = 4096 + 8 * min(self.n_rays, 65536)
        m = int(max(need_m * self.slack, floor) * grow)
        k = int(max(need_k * self.slack, floor) * grow)
        self.march_cap = max(self.march_cap or 0, m)
        self.kept_cap = max(self.kept_cap or 0, k)

    def set_rays(self, dirs, pidx):
        """copy camera-space directions [n_rays, 3] and pose indices [n_rays] (int64 in [0, P), checked: one host read) into `dirs`, `pidx`"""
        if self._pose is None:
            raise RuntimeError("StaticFrame.set_rays: the frame was built without pose=; pass rays_o / rays_d to step()")
        self._pose.set_rays(dirs, pidx)

    def _variance_control(self):
        """the model's variance schedule (ctrl_var with a host-side mix_weight), its device weight `_w_dev` made on first use; or None"""
        cv = getattr(self.model, "ctrl_var", None)
        if hasattr(cv, "mix_weight") and getattr(cv, "_w_dev", None) is None:
            cv._w_dev = torch.zeros((), device=self.device)
        return cv if hasattr(cv, "mix_weight") else None

    # -- the step
    def _run(self):
        if self.pre_hook is not None:
            self.pre_hook()
        if self.zero_grads:
            for p in self.model.parameters():
                if p.grad is not None:
                    p.grad.zero_()
        if self.sampler is not None:
            self.sampler.draw(self, self._rng_sampler)
        d_rays, hook = ((self.d_rays_o, self.d_rays_d) if self.d_rays_o is not None else None), None
        if self._pose is not None:
            d_rays, hook = self._pose.run(self.rays_o, self.rays_d, d_rays, self.zero_grads)
        cv = self._variance_control()
        if cv is not None:
            cv._use_w_dev = True                             # inv_s annealing weight from a device scalar (refreshed in step())
        try:
            rendered, _, buffers = render_static(self.model, self.rays_o, self.rays_d, self.h_appear, near=self.near, far=self.far, march_cap=self.march_cap,
                                                 kept_cap=self.kept_cap, coherent=bool(self.coherent), with_rgb=self.with_rgb, with_normal=self.with_normal, cnt=self.cnt,
                                                 d_h_appear=self.d_h_appear, d_rays=d_rays, max_level_dev=self.max_level_dev, ray_grad_hook=hook,
                                                 perturb=self.perturb, rng_dev=self.rng)
        finally:
            if cv is not None:
                cv._use_w_dev = False
        loss = None
        if self.loss_fn is not None:
            arg = dict(rendered=rendered, volume_buffer=static_volume_buffer(buffers, self.cnt)) if self.loss_on_ret else rendered
            loss, after_backward = self.sampler.loss(self, arg) if self.sampler is not None else (self.loss_fn(arg), None)
            if loss.requires_grad:
                loss.backward()
            loss = loss.detach()
            if after_backward is not None and not self._warming:         # the warm-up runs leave the sampler's state alone
                ov = CNT_SLOTS["overflow"]
                after_backward(self.cnt[ov:ov + 1])                       # (an overflowed step rendered nothing: skipped on the device)
        return rendered, buffers, loss

    def capture(self):
        if self.sampler is not None:
            self.sampler.draw(self, self._rng_sampler)      # this step's batch: the probe and the check below read its rays
        if self._pose is not None:
            if not bool(self.dirs.any()):                   # (zero directions: see below)
                raise RuntimeError("StaticFrame.capture: the pose inputs hold no rays yet; call set_rays(dirs, pidx) or step(dirs=..., pidx=...) first")
            self._pose.run(self.rays_o, self.rays_d)        # the probe and the check below read the rays
        if self.march_cap is None or self.kept_cap is None or self.coherent is None:
            self._size()
        if not self.use_graph:
            self.graph = None
            return self
        if not bool(self.rays_d.any()):
            # the warm-up and the capture RUN the step on the input buffers; a zero direction never leaves the marcher's voxel-skipping loop
            # (the reference's kernel has the same loop, occ_grid/helpers_march.h:58-69) -- refuse instead of hanging the device
            raise RuntimeError("StaticFrame.capture: the input buffers hold no rays yet; call step(rays_o, rays_d, ...) or fill frame.rays_o / frame.rays_d first")
        was = L.KERNEL_TIMER.enabled
        L.KERNEL_TIMER.enabled = False                      # events cannot be recorded into a capture
        import gc
        gc.collect()                                        # autograd graphs of earlier (default-stream) backward passes that only the cycle collector
        #                                                     frees keep the parameters' AccumulateGrad nodes on the default stream -> capture error
        try:
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._warming = True
                try:
                    for _ in range(2):                      # warm-up on a side stream (allocator, lazy module state)
                        self._run()
                finally:
                    self._warming = False
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            # capture on the warm-up's stream: the parameters' AccumulateGrad nodes were created there.  (A backward that ran on the default
            # stream BEFORE this and whose graph is still referenced -- a kept loss / rendered tensor -- pins those nodes to the default
            # stream and invalidates the capture: drop such references first.)
            self._occ_captured = self.model.accel.occ.occ_grid
            self._grad_captured = self._pose is not None and self._pose.wants_grad()
            with torch.cuda.graph(g, stream=side):
                self.rendered, self.buffers, self.loss = self._run()
            self.graph = g
            self.captures += 1
        finally:
            L.KERNEL_TIMER.enabled = was
        return self

    def step(self, rays_o=None, rays_d=None, rays_h_appear=None, *, dirs=None, pidx=None, cam=None, frame_ind=None):
        """copy the batch into the graph's inputs (H2D if the tensors are on the host) and launch.  -> loss (device scalar) or None.
        With pose=: no rays_o / rays_d; dirs and pidx (set_rays), or neither to replay the rays set last.  With sampler=: the camera cam
        (CameraSampler) or the LiDAR frame frame_ind (LidarSampler) whose batch the graph draws, alone."""
        after_step = None
        if self.sampler is not None:
            after_step = self.sampler.select(self, cam=cam, frame_ind=frame_ind, rays=(rays_o, rays_d, rays_h_appear, dirs, pidx))
        elif cam is not None or frame_ind is not None:
            raise RuntimeError("StaticFrame.step: cam= and frame_ind= are read only with sampler=")
        elif self._pose is None:
            if rays_o is None or rays_d is None or dirs is not None or pidx is not None:
                raise RuntimeError("StaticFrame.step: a frame without pose= takes rays_o and rays_d (and no dirs / pidx)")
            self.rays_o.copy_(rays_o, non_blocking=True)
            self.rays_d.copy_(rays_d, non_blocking=True)
        elif rays_o is not None or rays_d is not None or (dirs is None) != (pidx is None):
            raise RuntimeError("StaticFrame.step: a frame with pose= takes dirs and pidx (or neither), not rays_o / rays_d")
        elif dirs is not None:
            self.set_rays(dirs, pidx)
        if self._pose is not None:
            self._pose.bind_grads()
            if self.graph is not None and self._grad_captured != self._pose.wants_grad():
                self.graph = None                           # requires_grad of the pose switched: re-capture (with / without the adjoint)
        if self.h_appear is not None and rays_h_appear is not None:
            self.h_appear.copy_(rays_h_appear, non_blocking=True)
        cv = self._variance_control()
        if cv is not None:
            cv._w_dev.fill_(cv.mix_weight())                  # the variance schedule's host-side weight of THIS iteration
        self.max_level_dev.fill_(self.model.implicit_surface._ml(self.model.max_level))     # the LoTD level bound of THIS iteration
        if self.sampler is not None:        # the sampler's draws first; its kernel chains the offset after them into self.rng
            TR.take(self._gen, self.sampler_reservation + self.rng_reservation, self._rng_sampler)
        elif self.perturb:
            TR.take(self._gen, self.rng_reservation, self.rng)                                 # the random state of THIS iteration
        if self.graph is None and (self.use_graph or self.march_cap is None):
            self.capture()
        if self.graph is not None:
            occ = self.model.accel.occ.occ_grid
            if self._occ_captured is not None and occ.data_ptr() != self._occ_captured.data_ptr():
                # somebody RE-ASSIGNED the grid (the reference's EMA does, ema_single.py:190): the graph reads the tensor it captured -> refresh it
                self._occ_captured.copy_(occ)
            self.graph.replay()
        else:
            self.rendered, self.buffers, self.loss = self._run()
        if after_step is not None:
            after_step()
        return self.loss

    def counts(self):
        """host copy of the step's sizes (one D2H + sync)"""
        c = self.cnt.tolist()
        return {k: c[v] for k, v in CNT_SLOTS.items()}

    def check(self, retry=True):
        """True if the last step fitted its arenas.  Otherwise the arenas are re-sized from this batch, the graph is re-captured and --
        with `retry` -- the step is run again (gradients of the overflowed step were those of an empty render: nothing accumulated).
        With sampler=: raises if loss_fn gave the error map a negative error since the last check."""
        if self.sampler is not None:
            self.sampler.check(self)
        if int(self.cnt[CNT_SLOTS["overflow"]]) == 0:
            return True
        self.march_cap = self.kept_cap = None
        self._size(grow=1.25)
        self.graph = None
        if self.use_graph:
            self.capture()
        if retry:
            if self.graph is not None:
                self.graph.replay()
            else:
                self.rendered, self.buffers, self.loss = self._run()
        return False

    def volume_buffer(self):
        return sliced_volume_buffer(self.buffers, self.cnt)
