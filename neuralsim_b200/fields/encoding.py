"""LoTD encoding modules -- API of `nr3d_lib.models.grid_encodings.lotd` for the hash-only configuration
(reference: nr3d_lib/nr3d_lib/models/grid_encodings/lotd/lotd.py:40-458, lotd_encoding.py, lotd_cfg.py:48-57).

Three autograd functions carry first and second order gradients exactly like the reference's
LoTDFunction / LoTDFunctionFwdDydx / LoTDFunctionBwdDydx, batched tables included (a per-point batch index `bidx`,
per-batch `batch_offsets`, or `input_batched` equal-size batches); the kernels behind them are csrc/lotd.cu.
"""
from __future__ import annotations

from math import prod
from typing import Optional

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from ..bindings import _lotd as _backend


def gen_ngp_cfg(min_res=16, dim=3, n_feats=2, log2_hashmap_size=19, per_level_scale=1.382, num_levels=16):
    """Geometric resolution ladder; a level is Dense while res^dim fits the hash table (lotd_cfg.py:48-57)."""
    hashmap_size = 2 ** log2_hashmap_size
    res = (min_res * per_level_scale ** np.arange(num_levels)).astype(int)
    types = ["Dense" if int(r) ** dim <= hashmap_size else "Hash" for r in res]
    return dict(lod_res=res.tolist(), lod_n_feats=[n_feats] * num_levels, lod_types=types, hashmap_size=hashmap_size)


def auto_ngp_cfg(stretch, target_num_params, *, dim=3, n_feats=2, log2_hashmap_size=19, min_res=4, per_level_scale=1.382, max_num_levels=128):
    """The [Dense -> Hash] ladder the reference computes for cuboid spaces (`lotd_auto_compute_cfg: {type: ngp}`, lotd_cfg.py:59-133): the last
    dense level holds ~ hashmap/2.5 cells with the aspect ratio of `stretch`, the dense levels shrink from it by per_level_scale down to
    ~min_res on the shortest side, the hashed levels grow from it; their number follows from target_num_params."""
    stretch = np.array([stretch] * dim if np.isscalar(stretch) else list(stretch), dtype=np.float64)
    hashmap_size = 2 ** log2_hashmap_size
    dense_factor = (stretch / stretch.min()).prod()
    dense_last_min_res = int((hashmap_size / 2.5 / dense_factor) ** (1 / 3))
    num_dense = max(int(np.exp(np.log(dense_last_min_res / min_res) / per_level_scale) + 1), 1)
    num_hash = max(int(target_num_params / (hashmap_size * n_feats) - 1 + 0.5), 0)
    num_levels = num_dense + num_hash
    if max_num_levels is not None:
        num_levels = min(num_levels, max_num_levels)
        num_hash = num_levels - num_dense
    last = stretch / (stretch.min() / dense_last_min_res)
    res_dense = (last[..., None] / (per_level_scale ** np.arange(num_dense)))[:, ::-1].T.astype(int)
    res_hash = (last[..., None] * (per_level_scale ** (np.arange(num_hash) + 1))).T.astype(int)
    res = np.concatenate([res_dense, res_hash], axis=0)
    return dict(lod_res=res.tolist(), lod_n_feats=[n_feats] * num_levels, lod_types=["Dense"] * num_dense + ["Hash"] * num_hash, hashmap_size=hashmap_size)


def generate_meta(n_input_dim, lod_res, lod_n_feats, lod_types, hashmap_size=None, use_smooth_step=False):
    if isinstance(lod_n_feats, int):
        lod_n_feats = [lod_n_feats] * len(lod_res)
    if isinstance(lod_types, str):
        lod_types = [lod_types] * len(lod_res)
    return _backend.LoDMeta(n_input_dim, lod_res, lod_n_feats, lod_types, hashmap_size, use_smooth_step)


def _flat_bidx(bidx):
    return None if bidx is None else bidx.contiguous().long().flatten()


class LoTDFunction(torch.autograd.Function):
    """y = encode(clamp(x)); backward gives dL_dgrid (and dL_dx when x needs it).  First order only.
    bidx / batch_offsets / batch_data_size select each point's table when `grid` holds several (lotd.py:48-119)."""

    @staticmethod
    def forward(ctx, meta, x, grid, bidx=None, batch_offsets=None, batch_data_size=None, loss_scale=1.0, max_level=None):
        ctx.set_materialize_grads(False)
        prefix = x.shape[:-1]
        x = x.clamp(1.0e-6, 1 - 1.0e-6)
        bidx = _flat_bidx(bidx)
        need_x = ctx.needs_input_grad[1]
        y, dy_dx = _backend.lod_fwd(meta, x.flatten(0, -2).contiguous(), grid, bidx, batch_offsets, batch_data_size, max_level, need_x)
        if need_x or ctx.needs_input_grad[2]:
            ctx.save_for_backward(x, grid, dy_dx, bidx, batch_offsets)
            ctx.meta, ctx.prefix, ctx.loss_scale, ctx.max_level, ctx.batch_data_size = meta, prefix, loss_scale, max_level, batch_data_size
        return y.unflatten(0, prefix)

    @staticmethod
    @once_differentiable
    def backward(ctx, dL_dy):
        if dL_dy is None:
            return (None,) * 8
        x, grid, dy_dx, bidx, batch_offsets = ctx.saved_tensors
        s = ctx.loss_scale
        dL_dx, dL_dgrid = _backend.lod_bwd(ctx.meta, (dL_dy.flatten(0, -2) * s).contiguous(), x.flatten(0, -2), grid, dy_dx, bidx, batch_offsets,
                                           ctx.batch_data_size, ctx.max_level, ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        dL_dx = None if dL_dx is None else dL_dx.unflatten(0, ctx.prefix) / s
        dL_dgrid = None if dL_dgrid is None else dL_dgrid / s
        return None, dL_dx, dL_dgrid, None, None, None, None, None


class LoTDFunctionFwdDydx(torch.autograd.Function):
    """(y, dy_dx) = encode_with_jacobian(clamp(x)).  Use LoTDFunctionBwdDydx for nablas; this backward only
    routes dL_dy to the table (and to x when `need_dL_dinput`).  (lotd.py:121-191)"""

    @staticmethod
    def forward(ctx, meta, x, grid, bidx=None, batch_offsets=None, batch_data_size=None, loss_scale=1.0, max_level=None, need_dL_dinput=None):
        if need_dL_dinput is None:
            need_dL_dinput = torch.is_grad_enabled() and x.requires_grad
        ctx.set_materialize_grads(False)
        prefix = x.shape[:-1]
        x = x.clamp(1.0e-6, 1 - 1.0e-6)
        bidx = _flat_bidx(bidx)
        y, dy_dx = _backend.lod_fwd(meta, x.flatten(0, -2).contiguous(), grid, bidx, batch_offsets, batch_data_size, max_level, True)
        ctx.save_for_backward(x, grid, dy_dx, bidx, batch_offsets)
        ctx.meta, ctx.prefix, ctx.loss_scale, ctx.max_level, ctx.need_dL_dinput = meta, prefix, loss_scale, max_level, need_dL_dinput
        ctx.batch_data_size = batch_data_size
        ctx.mark_non_differentiable(dy_dx)
        return y.unflatten(0, prefix), dy_dx

    @staticmethod
    @once_differentiable
    def backward(ctx, dL_dy, _):
        if dL_dy is None:
            return (None,) * 9
        x, grid, dy_dx, bidx, batch_offsets = ctx.saved_tensors
        s = ctx.loss_scale
        dL_dx, dL_dgrid = _backend.lod_bwd(ctx.meta, (dL_dy.flatten(0, -2) * s).contiguous(), x.flatten(0, -2), grid, dy_dx, bidx, batch_offsets,
                                           ctx.batch_data_size, ctx.max_level, ctx.need_dL_dinput, ctx.needs_input_grad[2])
        dL_dx = None if dL_dx is None else dL_dx.unflatten(0, ctx.prefix) / s
        dL_dgrid = None if dL_dgrid is None else dL_dgrid / s
        return None, dL_dx, dL_dgrid, None, None, None, None, None, None


class LoTDFunctionBwdDydx(torch.autograd.Function):
    """dL_dx = J(x)^T dL_dy as a differentiable op: its backward is the second-order pass towards dL_dy and the table.
    (lotd.py:193-268)"""

    @staticmethod
    def forward(ctx, meta, dL_dy, x, grid, dy_dx, bidx=None, batch_offsets=None, batch_data_size=None, loss_scale=1.0, max_level=None,
                grad_guard=None):
        ctx.set_materialize_grads(False)
        prefix = x.shape[:-1]
        x = x.clamp(1.0e-6, 1 - 1.0e-6)
        bidx = _flat_bidx(bidx)
        dL_dx, _ = _backend.lod_bwd(meta, (dL_dy.flatten(0, -2) * loss_scale).contiguous(), x.flatten(0, -2).contiguous(), grid, dy_dx,
                                    bidx, batch_offsets, batch_data_size, max_level, True, False)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[3]:
            ctx.save_for_backward(dL_dy, x, grid, dy_dx.contiguous(), bidx, batch_offsets)
            ctx.meta, ctx.loss_scale, ctx.max_level, ctx.grad_guard = meta, loss_scale, max_level, grad_guard
            ctx.batch_data_size = batch_data_size
        return dL_dx.unflatten(0, prefix) / loss_scale

    @staticmethod
    @once_differentiable
    def backward(ctx, dL_ddLdx):
        if dL_ddLdx is None:
            return (None,) * 11
        dL_dy, x, grid, dy_dx, bidx, batch_offsets = ctx.saved_tensors
        prefix, s = x.shape[:-1], ctx.loss_scale
        ddLdy, dgrid, _ = _backend.lod_bwd_bwd_input(
            ctx.meta, dL_ddLdx.flatten(0, -2).contiguous(), (dL_dy.flatten(0, -2) * s).contiguous(), x.flatten(0, -2), grid, dy_dx,
            bidx, batch_offsets, ctx.batch_data_size, ctx.max_level, ctx.needs_input_grad[1], ctx.needs_input_grad[3], False)
        ddLdy = None if ddLdy is None else ddLdy.unflatten(0, prefix)
        dgrid = None if dgrid is None else dgrid / s
        if ctx.grad_guard is not None and (dgrid is not None or ddLdy is not None):
            ctx.grad_guard.custom_grad_clip_step(dL_ddLdx, dy_dx, dgrid, ddLdy)
        return None, ddLdy, None, dgrid, None, None, None, None, None, None, None


def _batch_data_size(input, input_batched):
    """input_batched: `input` is [B, ..., D] and its points of batch b read table b (lotd.py:275-279)"""
    return prod(input.shape[1:-1]) if input_batched else 0


def lotd_encoding(input, params, bidx=None, batch_offsets=None, input_batched=False, max_level=None,
                  meta=None, n_input_dim=None, lod_res=None, lod_n_feats=None, lod_types=None):
    """lotd.py:270-282"""
    if meta is None:
        meta = generate_meta(n_input_dim, lod_res, lod_n_feats, lod_types)
    if input_batched:
        bidx = None
    loss_scale = 128.0 if params.dtype == torch.float16 else 1.0
    return LoTDFunction.apply(meta, input, params, bidx, batch_offsets, _batch_data_size(input, input_batched), loss_scale, max_level)


def lotd_encoding_fwd_dydx(input, params, bidx=None, batch_offsets=None, input_batched=False, max_level=None, need_dL_dinput: Optional[bool] = None,
                           meta=None, n_input_dim=None, lod_res=None, lod_n_feats=None, lod_types=None):
    """lotd.py:284-298 -> (y, dy_dx, meta)"""
    if need_dL_dinput is None:
        need_dL_dinput = torch.is_grad_enabled() and input.requires_grad
    if meta is None:
        meta = generate_meta(n_input_dim, lod_res, lod_n_feats, lod_types)
    if input_batched:
        bidx = None
    loss_scale = 128.0 if params.dtype == torch.float16 else 1.0
    y, dy_dx = LoTDFunctionFwdDydx.apply(meta, input, params, bidx, batch_offsets, _batch_data_size(input, input_batched), loss_scale, max_level,
                                         need_dL_dinput)
    return y, dy_dx, meta


def lotd_encoding_bwd_dydx(meta, dL_dy, dy_dx, input, params, bidx=None, batch_offsets=None, input_batched=False, max_level=None):
    """lotd.py:300-309"""
    if input_batched:
        bidx = None
    loss_scale = 128.0 if params.dtype == torch.float16 else 1.0
    return LoTDFunctionBwdDydx.apply(meta, dL_dy, input, params, dy_dx, bidx, batch_offsets, _batch_data_size(input, input_batched), loss_scale,
                                     max_level)


class LoTD(nn.Module):
    """Stateless encoder: holds the level layout, the table is passed to every call (lotd.py:321-458)."""

    def __init__(self, in_features, lod_res, lod_n_feats, lod_types, hashmap_size: int = None, log2_hashmap_size: int = None,
                 use_smooth_step=False, dtype=torch.half, device=None):
        super().__init__()
        assert dtype in (torch.float, torch.float16), "dtype must be one of torch.float or torch.float16"
        if log2_hashmap_size is not None:
            assert hashmap_size is None, "Do not specify `hashmap_size` when `log2_hashmap_size` is already specified."
            hashmap_size = 2 ** log2_hashmap_size
        self.dtype = dtype
        self.loss_scale = 128.0 if dtype == torch.float16 else 1.0
        self.meta = generate_meta(in_features, lod_res, lod_n_feats, lod_types, hashmap_size, use_smooth_step)

    in_features = property(lambda self: self.meta.n_dims_to_encode)
    out_features = property(lambda self: self.meta.n_encoded_dims)
    n_levels = property(lambda self: self.meta.n_levels)
    n_params = property(lambda self: self.meta.n_params)
    level_res_multidim = property(lambda self: self.meta.level_res_multidim)
    level_n_feats = property(lambda self: self.meta.level_n_feats)
    level_offsets = property(lambda self: self.meta.level_offsets)
    level_sizes = property(lambda self: self.meta.level_sizes)
    level_n_params = property(lambda self: self.meta.level_n_params)

    # bidx / batch_offsets / input_batched: `params` holds several tables (lotd.py:425-458); keyword-only here, after max_level
    def forward(self, input, params, max_level: int = None, *, bidx=None, batch_offsets=None, input_batched=False):
        bds = self._batch_data_size(input, bidx, input_batched)
        return LoTDFunction.apply(self.meta, input, params.to(self.dtype), bidx, batch_offsets, bds, self.loss_scale, max_level)

    def forward_dydx(self, input, params, max_level: int = None, need_dL_dinput: Optional[bool] = None, *, bidx=None, batch_offsets=None,
                     input_batched=False):
        bds = self._batch_data_size(input, bidx, input_batched)
        return LoTDFunctionFwdDydx.apply(self.meta, input, params.to(self.dtype), bidx, batch_offsets, bds, self.loss_scale, max_level,
                                         need_dL_dinput)

    def backward_dydx(self, dL_dy, dy_dx, input, params, max_level: int = None, grad_guard=None, *, bidx=None, batch_offsets=None,
                      input_batched=False):
        bds = self._batch_data_size(input, bidx, input_batched)
        return LoTDFunctionBwdDydx.apply(self.meta, dL_dy, input, params.to(self.dtype), dy_dx, bidx, batch_offsets, bds, self.loss_scale,
                                         max_level, grad_guard)

    @staticmethod
    def _batch_data_size(input, bidx, input_batched):
        if input_batched:
            assert bidx is None, 'bidx is only taken care of when input is not batched.'
        return _batch_data_size(input, input_batched)


class MultiresAnnealer(nn.Module):
    """The level schedule of a multi-resolution encoding (multires_annealer.py:19-64), hard-mask form: `forward(it)` -> (max_level, None);
    levels 0..max_level are used.  max_level starts at `start_level` (clamped to [-1, L-1]; -1 = no level) at `start_it` and gains one level
    per 1/(L-1-start_level) of the stages up to `stop_it`; a stage is `update_every` iterations.  Before the first `set_iter` / `forward(it)`
    the annealer is in its stop state (all levels).  It holds no tensors: the state dict of the encoding does not change."""

    def __init__(self, level_n_feats, type: str, stop_it: int, start_it: int = 0, update_every: int = 1, start_level: int = 0):
        super().__init__()
        if type == "cosine":
            raise RuntimeError("MultiresAnnealer: anneal type 'cosine' is not built (its per-feature window is not applied by the fused kernels); "
                               "use 'hardmask'")
        if type != "hardmask":
            raise RuntimeError(f"Invalid anneal_type={type}")
        self.num_levels = len(level_n_feats)
        self.start_it, self.stop_it, self.update_every = int(start_it), int(stop_it), int(update_every)
        self.total_stages = (self.stop_it - self.start_it) // self.update_every
        if self.total_stages == 0:
            raise RuntimeError(f"MultiresAnnealer: stop_it={self.stop_it}, start_it={self.start_it}, update_every={self.update_every} give no stage "
                               "to anneal over ((stop_it - start_it) // update_every == 0)")
        self.it = self.stop_it
        self.start_level = max(min(int(start_level), self.num_levels - 1), -1)

    def set_iter(self, it: int):
        self.it = it

    def forward(self, it: int = None):
        it = self.it if it is None else it
        alpha = min(1.0, max(0.0, ((it - self.start_it) // self.update_every) / self.total_stages))
        length = (self.num_levels - 1) - self.start_level
        return self.start_level + min(int(alpha * length), length), None


class LoTDEncoding(nn.Module):
    """LoTD + its parameter table `flattened_params` (fp32 master) for inputs in [-1,1]^D
    (lotd_encoding.py:37-213; state-dict key `...encoding.flattened_params`).  anneal_cfg (lotd_encoding.py:99-103): the keys of
    MultiresAnnealer; `set_anneal_iter(it)` then sets `max_level` (every query without an explicit level uses it)."""

    def __init__(self, input_ch=3, *, lotd_cfg: dict = None, lotd_auto_compute_cfg: dict = None, param_init_cfg=dict(type="uniform_to_type", bound=1.0e-4),
                 dtype=torch.half, device=None, generator=None, lotd_use_cuboid=False, aabb=None, anneal_cfg: dict = None):
        super().__init__()
        if lotd_cfg is None:
            auto = dict(lotd_auto_compute_cfg or dict(type="gen_ngp"))
            kind = auto.pop("type", "gen_ngp")
            if kind == "gen_ngp":
                lotd_cfg = gen_ngp_cfg(dim=input_ch, **auto)
            elif kind == "ngp":
                # lotd_encoding.py:60-75: cuboid spaces stretch the level resolutions with the aabb's aspect ratio
                stretch = 1.0
                if lotd_use_cuboid:
                    if aabb is None:
                        raise RuntimeError("lotd_use_cuboid needs the aabb of the space")
                    ab = torch.as_tensor(aabb, dtype=torch.float64)
                    stretch = (ab[1] - ab[0]).tolist()
                lotd_cfg = auto_ngp_cfg(stretch, dim=input_ch, **auto)
            else:
                raise RuntimeError(f"lotd_auto_compute_cfg type={kind!r} is not built (gen_ngp, ngp)")
        self.lotd_cfg = lotd_cfg
        self.lotd = LoTD(input_ch, **lotd_cfg, dtype=dtype, device=device)
        self.dtype = dtype
        self.in_features, self.out_features = input_ch, self.lotd.out_features
        self.max_level, self.window = None, None
        self.annealer = MultiresAnnealer(self.lotd.level_n_feats, **anneal_cfg) if anneal_cfg is not None else None
        bound = float(param_init_cfg.get("bound", 1.0e-4))
        p = torch.empty(self.lotd.n_params, dtype=torch.float, device=device)
        p.uniform_(-bound, bound, generator=generator)
        self.flattened_params = nn.Parameter(p, requires_grad=True)

    @property
    def meta(self):
        return self.lotd.meta

    def set_anneal_iter(self, cur_it: int):
        if self.annealer is not None:
            self.max_level, self.window = self.annealer(cur_it)

    @property
    def inference_param(self):
        return self.flattened_params.data.to(self.dtype)

    def forward(self, input, max_level: int = None):
        out = self.lotd.forward(input / 2. + 0.5, self.flattened_params, max_level=(max_level or self.max_level))
        return out * self.window if self.window is not None else out

    def forward_dydx(self, input, max_level: int = None, need_dL_dinput: Optional[bool] = None):
        out, dy_dx = self.lotd.forward_dydx(input / 2. + 0.5, self.flattened_params, max_level=(max_level or self.max_level),
                                            need_dL_dinput=need_dL_dinput)
        return (out * self.window if self.window is not None else out), dy_dx

    def backward_dydx(self, dL_dy, dy_dx, input, max_level: int = None, grad_guard=None):
        nablas = self.lotd.backward_dydx(dL_dy, dy_dx, input / 2. + 0.5, self.flattened_params, max_level=(max_level or self.max_level),
                                         grad_guard=grad_guard)
        return nablas / 2.   # the table sees x/2+0.5
