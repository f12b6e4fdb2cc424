"""The StreetSurf LiDAR loss (reference: app/loss/lidar.py, `LidarLoss` with `DepthLoss` and the `neus_unisim` `LineOfSightLoss`) as
fused, count-aware CUDA kernels (csrc/lidar_loss.cu) that read the renderer's buffers in place and never read a size back to the host.

    lidar_loss = LidarLoss(**config["training"]["losses"]["lidar"])
    # host-sized path: the reference's call
    ret = SingleVolumeRenderer(...).render(model, rays_o, rays_d, return_buffer=True)
    losses = lidar_loss(scene, ret, sample, {"ranges": ranges}, it=it)
    # one-launch graph step: the step's ranges and iteration go in first, the loss reads them from static buffers
    frame = StaticFrame(model, n, loss_fn=lambda ret: sum(lidar_loss(None, ret).values()), loss_on_ret=True, with_rgb=False)
    lidar_loss.set_step(ranges, it)
    frame.step(rays_o, rays_d)
    # the graph step that draws its own batch: the ranges come with the step's ground truth, the iteration's weights from set_step
    frame = StaticFrame(model, n, loss_fn=lambda ret, gt: sum(lidar_loss(None, ret, ground_truth=gt).values()), loss_on_ret=True,
                        with_rgb=False, sampler=LidarSampler(...))
    lidar_loss.set_step(None, it)
    frame.step(frame_ind=f)

`ret["volume_buffer"]` is either the reference's exact-size `"packed"` dict or the capacity-sized `"packed_static"` dict of
`StaticFrame(loss_on_ret=True)` (its sizes in the step's device count block).  The per-step values -- the ranges and the annealed weights
and epsilon -- live in device buffers that `set_step` refreshes, so a captured step follows them on replay without re-capture.

Differences from the reference, each by construction:
  - the median of the outlier discard is a device-side radix select (no sort, no host read); it equals `torch.sort(err).values[R // 2]`;
  - the line-of-sight term is summed over the whole-image rows (0 for rays that keep nothing) and divided by the device count of kept rays,
    so the host-sized path and the graph step give the same bits; with no kept ray the graph step's term is 0 where the host-sized path, as
    the reference, returns no `lidar_loss.los.empty` key for an `"empty"` buffer;
  - only what the shipped StreetSurf configurations use is built: depth `fn_type` l1 / l2_relative, line of sight `neus_unisim`, annealers
    of type `milestones`, `discard_outliers` = 0, packed buffers.  Everything else raises a RuntimeError that names it.
"""
from __future__ import annotations

from bisect import bisect_right

import torch
import torch.nn as nn

from .. import _lib as L

__all__ = ["DepthLoss", "LineOfSightLoss", "LidarLoss", "anneal_milestones"]

FN_TYPES = {"l1": 0, "l2_relative": 1}
KTH_ONE_CTA_MAX = 1 << 16            # csrc/lidar_loss.cu: up to this many rays the median needs no scratch


def anneal_milestones(it, milestones, vals):
    """nr3d_lib/models/annealers.py get_anneal_val_milestones: vals[bisect_right(milestones, it)]"""
    if len(milestones) + 1 != len(vals):
        raise RuntimeError(f"milestones annealer: `vals` ({len(vals)}) must have one more element than `milestones` ({len(milestones)})")
    return vals[bisect_right(milestones, it)]


def _annealer(anneal, what):
    if anneal is None:
        return None
    anneal = dict(anneal)
    kind = anneal.pop("type", None)
    if kind != "milestones":
        raise RuntimeError(f"{what}: annealer type={kind!r} is not built (only 'milestones', which the StreetSurf configurations use)")
    return lambda it: anneal_milestones(it, **anneal)


class DepthLoss(nn.Module):
    """the depth term w f(pred, gt) mask / R (app/loss/lidar.py:22-53); f = l1 or l2_relative"""

    def __init__(self, w: float = 1.0, anneal: dict = None, fn_type: str = "l1_log", fn_param: dict = None) -> None:
        super().__init__()
        if fn_type not in FN_TYPES:
            raise RuntimeError(f"DepthLoss: fn_type={fn_type!r} is not built (built: {', '.join(FN_TYPES)})")
        if fn_param:
            raise RuntimeError(f"DepthLoss: fn_param={fn_param!r} is not built (the l1 / l2_relative losses take none)")
        self.w, self.w_fn, self.fn_type = w, _annealer(anneal, "DepthLoss"), fn_type

    def weight(self, it):
        return self.w if self.w_fn is None else self.w_fn(it)


class LineOfSightLoss(nn.Module):
    """the `neus_unisim` line-of-sight term w mean over kept rays of mask sum_i [|t_i - gt| > eps] vw_i^2 (app/loss/lidar.py:174-210)"""

    def __init__(self, w: float = 1.0, anneal: dict = None, fn_type: str = "nerf", fn_param: dict = None) -> None:
        super().__init__()
        if fn_type != "neus_unisim":
            raise RuntimeError(f"LineOfSightLoss: fn_type={fn_type!r} is not built (only 'neus_unisim', which the StreetSurf configurations use)")
        fn_param = dict(fn_param or {})
        eps, eps_anneal = fn_param.pop("epsilon", 1.0), fn_param.pop("epsilon_anneal", None)
        if fn_param:
            raise RuntimeError(f"LineOfSightLoss: fn_param keys {sorted(fn_param)} are not built (neus_unisim takes epsilon, epsilon_anneal)")
        self.w, self.w_fn, self.fn_type = w, _annealer(anneal, "LineOfSightLoss"), fn_type
        self.eps, self.eps_fn = eps, _annealer(eps_anneal, "LineOfSightLoss epsilon_anneal")

    def weight(self, it):
        return self.w if self.w_fn is None else self.w_fn(it)

    def epsilon(self, it):
        return self.eps if self.eps_fn is None else self.eps_fn(it)


class _LidarLossFn(torch.autograd.Function):
    """-> out [2] = (depth term, line-of-sight term); differentiable in depth_pred and vw (their cotangents feed _Composite.backward)"""

    @staticmethod
    def forward(ctx, cfg, depth_pred, vw, mask_pred, t, pinfo, rih, gt, blk, count):
        fn, thresh, toofar, factor = cfg
        P, lib = L.ptr, L.lib()
        R, dev = gt.numel(), gt.device
        pred = depth_pred.detach().contiguous().view(-1)
        rows = torch.empty(4, R, dtype=torch.float32, device=dev)
        mask, err, drow, lrow = rows[0], rows[1], rows[2] if fn is not None else None, rows[3] if vw is not None else None
        out = torch.empty(2, dtype=torch.float32, device=dev)
        L.call(lib.nsb_lidar_mask_err, "lidar_mask_err", P(pred, "f32"), P(mask_pred.detach().contiguous().view(-1), "f32"), P(gt, "f32"), L.c_i64(R),
               L.c_f32(thresh), L.c_i32(toofar is not None), L.c_f32(toofar or 0.0), P(mask), P(err), L.stream_ptr())
        med = None
        if factor > 0:
            med = torch.empty(1, dtype=torch.float32, device=dev)
            scratch = torch.empty(int(lib.nsb_kth_smallest_scratch_bytes()), dtype=torch.uint8, device=dev) if R > KTH_ONE_CTA_MAX else None
            L.call(lib.nsb_kth_smallest, "kth_smallest", P(err), L.c_i64(R), L.c_i64(R // 2), P(med), P(scratch, allow_none=True), L.stream_ptr())
        L.call(lib.nsb_lidar_rows, "lidar_rows", P(pred), P(gt), P(err), P(med, allow_none=True), L.c_f32(factor), L.c_i32(fn or 0), L.c_i64(R),
               P(mask), P(drow, allow_none=True), P(lrow, allow_none=True), L.stream_ptr())
        n_kept = 0
        if vw is not None:
            n_kept = pinfo.shape[0]
            L.call(lib.nsb_lidar_los_rows, "lidar_los_rows", P(t, "f32"), P(vw, "f32"), P(pinfo, "i64"), P(rih, "i64"), L.c_i64(n_kept), P(gt),
                   P(mask), P(blk, "f32"), P(lrow), L.stream_ptr(), count=count)
        L.call(lib.nsb_lidar_loss_reduce, "lidar_loss_reduce", P(drow, allow_none=True), P(lrow, allow_none=True), L.c_i64(R), L.c_i64(n_kept),
               P(blk), P(out), L.stream_ptr(), count=count if vw is not None else None)
        ctx.save_for_backward(pred, gt, mask, blk, t, vw, pinfo, rih)
        ctx.cfg, ctx.count, ctx.pred_shape = cfg, count, depth_pred.shape
        ctx.mark_non_differentiable(mask)
        return out, mask

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out, _g_mask):
        pred, gt, mask, blk, t, vw, pinfo, rih = ctx.saved_tensors
        fn = ctx.cfg[0]
        P, lib = L.ptr, L.lib()
        g_out = g_out.contiguous()
        g_depth = g_vw = None
        if fn is not None and ctx.needs_input_grad[1]:
            g_depth = torch.empty_like(pred)
            L.call(lib.nsb_lidar_depth_backward, "lidar_depth_backward", P(pred), P(gt), P(mask), L.c_i64(pred.numel()), L.c_i32(fn), P(blk), P(g_out, "f32"),
                   P(g_depth), L.stream_ptr())
            g_depth = g_depth.view(ctx.pred_shape)
        if vw is not None and ctx.needs_input_grad[2]:
            g_vw = torch.zeros_like(vw)                     # capacity rows past the kept samples stay 0
            L.call(lib.nsb_lidar_los_backward, "lidar_los_backward", P(t), P(vw), P(pinfo), P(rih), L.c_i64(pinfo.shape[0]), P(gt), P(mask), P(blk),
                   P(g_out), P(g_vw), L.stream_ptr(), count=ctx.count)
        return None, g_depth, g_vw, None, None, None, None, None, None, None


class LidarLoss(nn.Module):
    """app/loss/lidar.py:212-294 on the fused kernels.  Constructor arguments and the returned keys are the reference's."""

    def __init__(self, depth: dict = None, line_of_sight: dict = None, discard_toofar: float = None, discard_outliers: float = 0,
                 discard_outliers_median: float = 100.0, mask_pred_thresh: float = 1.0e-7) -> None:
        super().__init__()
        if discard_outliers > 0:
            raise RuntimeError(f"LidarLoss: discard_outliers={discard_outliers} is not built (no StreetSurf configuration uses it; "
                               "discard_outliers_median is)")
        self.depth_loss = DepthLoss(**depth) if depth is not None else None
        self.line_of_sight_loss = LineOfSightLoss(**line_of_sight) if line_of_sight is not None else None
        self.discard_toofar, self.discard_outliers = discard_toofar, discard_outliers
        self.discard_outliers_median, self.mask_pred_thresh = discard_outliers_median, mask_pred_thresh
        self.ranges = None                 # [n_rays] device: the step's ground-truth ranges (set_step)
        self._blk = None                   # device fp32 {w_depth, w_los, epsilon} of the step's iteration (set_step)
        self.mask = None                   # [n_rays] the last step's validity mask (after the outlier discard)

    @torch.no_grad()
    def set_step(self, ranges, it, device=None):
        """the step's ranges [n_rays] and iteration -> the static buffers the loss reads (device copies and fills: no host read).  Call it
        before StaticFrame.step; the buffers keep their addresses, so a captured step follows them on replay.  ranges None: the weights
        of iteration `it` only (a step whose ranges come with its ground truth, StaticFrame(sampler=LidarSampler(...)); the weights are
        made on `device`, default the current CUDA device, when no step set them before)."""
        if ranges is not None:
            r = ranges.reshape(-1)
            if self.ranges is None or self.ranges.shape != r.shape or self.ranges.device != r.device:
                self.ranges = torch.empty(r.shape, dtype=torch.float32, device=r.device)
            if self._blk is None or self._blk.device != r.device:
                self._blk = torch.zeros(3, dtype=torch.float32, device=r.device)
            self.ranges.copy_(r, non_blocking=True)
        elif self._blk is None:
            self._blk = torch.zeros(3, dtype=torch.float32, device=device if device is not None else torch.device("cuda", torch.cuda.current_device()))
        d, s = self.depth_loss, self.line_of_sight_loss
        self._blk[0].fill_(d.weight(it) if d is not None else 0.0)
        self._blk[1].fill_(s.weight(it) if s is not None else 0.0)
        self._blk[2].fill_(s.epsilon(it) if s is not None else 0.0)

    def forward(self, scene, ret: dict, sample: dict = None, ground_truth: dict = None, *, it: int = None, far: float = None, logger=None):
        """the reference's call; with ground_truth None the ranges and iteration of the last set_step are used (the graph step).  With
        ground_truth and it None, once a set_step has run: ground_truth["ranges"] is read in place (a float32 device buffer the step
        fills, StaticFrame(sampler=LidarSampler(...)).ground_truth) with the weights of the last set_step(None, it)."""
        if ground_truth is not None and it is None and self._blk is not None:
            ranges = ground_truth["ranges"].reshape(-1)
            if ranges.dtype != torch.float32 or ranges.device != self._blk.device or not ranges.is_contiguous():
                raise RuntimeError(f"LidarLoss: ground_truth['ranges'] read in place must be a contiguous float32 tensor on {self._blk.device}")
        elif ground_truth is not None:
            self.set_step(ground_truth["ranges"], it)
            ranges = self.ranges
        elif self.ranges is None:
            raise RuntimeError("LidarLoss: no ranges: pass ground_truth={'ranges': ...} or call set_step(ranges, it) before the step")
        else:
            ranges = self.ranges
        depth_pred, mask_pred = ret["rendered"]["depth_volume"], ret["rendered"]["mask_volume"]
        if depth_pred.numel() != ranges.numel():
            raise RuntimeError(f"LidarLoss: {depth_pred.numel()} rendered rays, {ranges.numel()} ranges")
        vw = t = pinfo = rih = count = None
        if self.line_of_sight_loss is not None:
            vb = ret["volume_buffer"]
            kind = vb["type"]
            if kind in ("packed", "packed_static"):
                t, vw, pinfo, rih = vb["t"], vb["vw"], vb["pack_infos_hit"], vb["rays_inds_hit"]
                if kind == "packed_static":
                    count = (vb["cnt"], vb["CNT_SLOTS"]["kept_rays"])
            elif kind != "empty":
                raise RuntimeError(f"LidarLoss: volume buffer type={kind!r} is not built (packed / packed_static / empty)")
        if self.depth_loss is None and vw is None:
            return {}
        cfg = (FN_TYPES[self.depth_loss.fn_type] if self.depth_loss is not None else None, float(self.mask_pred_thresh),
               float(self.discard_toofar) if self.discard_toofar is not None and self.discard_toofar > 0 else None,
               float(self.discard_outliers_median))
        out, self.mask = _LidarLossFn.apply(cfg, depth_pred, vw, mask_pred, t, pinfo, rih, ranges, self._blk, count)
        losses = {}
        if self.depth_loss is not None:
            losses["lidar_loss.depth"] = out[0]
        if vw is not None:
            losses["lidar_loss.los.empty"] = out[1]
        return losses
