"""Drop-in for `nr3d_lib.bindings._lotd` (reference: nr3d_lib/csrc/lotd/src/lotd.cpp:22-107) over the C ABI.

Same names, argument order and error behaviour (RuntimeError) as the pybind11 module; the encoding kernels
are the sm_90a ones of neuralsim_b200/csrc/lotd.cu.  Supported: Dense / Hash levels, linear interpolation,
single (non-batched, non-forest) tables -- the `c_hash_only` configuration every NeuS config of the reference
uses.  Unsupported arguments raise instead of silently taking another path.
"""
from __future__ import annotations

import ctypes
from enum import IntEnum

import torch

from .. import _lib as L


class LoDType(IntEnum):          # lotd_types.h:16-26
    Dense = 0
    VectorMatrix = 1
    VecZMatXoY = 2
    CP = 3
    CPfast = 4
    NPlaneMul = 5
    NPlaneSum = 6
    Hash = 7


class InterpolationType(IntEnum):
    Linear = 0
    Smoothstep = 1


_TYPE_OF = {"dense": LoDType.Dense, "hash": LoDType.Hash}


class LoDMeta:
    """LoDMeta(n_input_dims, lod_res | lod_res_multidim, lod_n_feats, lod_types, hashmap_size=None,
    use_smooth_step=None) with the read-only attributes of the reference class (lotd.cpp:66-104)."""

    def __init__(self, n_input_dims, lod_res, lod_n_feats, lod_types, hashmap_size=None, use_smooth_step=None):
        if use_smooth_step:
            raise RuntimeError("neuralsim_b200 LoTD: smoothstep interpolation is not built (hot path uses Linear)")
        n_levels = len(lod_res)
        if not (len(lod_n_feats) == n_levels == len(lod_types)):
            raise RuntimeError("LoTDEncoding: Expect los_res, lod_n_feats, lod_str_types to have the same length")
        res = []
        for r in lod_res:
            res += ([int(r)] * n_input_dims) if isinstance(r, int) or not hasattr(r, "__len__") else [int(v) for v in r]
        types = []
        for t in lod_types:
            if str(t).lower() not in _TYPE_OF:
                raise RuntimeError(f"neuralsim_b200 LoTD: level type {t!r} is not built (Dense / Hash only)")
            types.append(int(_TYPE_OF[str(t).lower()]))
        self._c = L.LotdMetaC()
        arr = lambda xs: (ctypes.c_int32 * len(xs))(*xs)
        L.check(L.lib().nsb_lotd_meta_create(ctypes.c_int32(n_input_dims), ctypes.c_int32(n_levels), arr(res),
                                             arr([int(f) for f in lod_n_feats]), arr(types),
                                             ctypes.c_uint32(int(hashmap_size or 0)), ctypes.byref(self._c)), "LoDMeta")
        c, D = self._c, n_input_dims
        self.level_types_str = list(lod_types)
        self.n_levels, self.n_pseudo_levels = int(c.n_levels), int(c.n_pseudo_levels)
        self.n_feat_per_pseudo_lvl, self.n_dims_to_encode = int(c.n_feat_per_pseudo_lvl), int(c.n_dims_to_encode)
        self.n_encoded_dims, self.n_params = int(c.n_encoded_dims), int(c.n_params)
        self.level_res_multidim = [[int(c.level_res[l][d]) for d in range(D)] for l in range(self.n_levels)]
        self.level_res = [r[0] if all(v == r[0] for v in r) else 0 for r in self.level_res_multidim]
        self.level_n_feats = [int(c.level_n_feats[l]) for l in range(self.n_levels)]
        self.level_types = [int(c.level_types[l]) for l in range(self.n_levels)]
        self.level_sizes = [int(c.level_sizes[l]) for l in range(self.n_levels)]
        self.level_n_params = [s * f for s, f in zip(self.level_sizes, self.level_n_feats)]
        self.level_offsets = [int(c.level_offsets[l]) for l in range(self.n_levels + 1)]
        self.map_levels = [int(c.map_levels[p]) for p in range(self.n_pseudo_levels)]
        self.map_cnt = [int(c.map_cnt[p]) for p in range(self.n_pseudo_levels)]
        self.interpolation_type = InterpolationType.Linear
        # performance switches of the reference class; accepted and ignored (one code path here)
        self.c_hash_only, self.c_profile, self.c_bmm_backend, self.c_prefetch, self.c_permute_dydx = True, False, 1, True, True

    @property
    def c_ref(self):
        return ctypes.byref(self._c)


def _no_batch(batch_inds, batch_offsets, batch_data_size):
    if batch_inds is not None or batch_offsets is not None or batch_data_size:
        raise RuntimeError("neuralsim_b200 LoTD: batched tables (batch_inds / batch_offsets / batch_data_size) are not built yet")


def _check_params(meta, params):
    if params.dim() != 1 or params.shape[0] % meta.n_params != 0 or params.shape[0] == 0:
        raise RuntimeError(f"LoTDEncoding::fwd: Expect size of `params`={params.shape[0]} to be an integral multiple of "
                           f"`n_param`={meta.n_params}")
    if params.dtype not in (torch.float16, torch.float32):
        raise RuntimeError("LoTDEncoding: params must be half or float")


def lod_fwd(lod_meta, input, params, batch_inds=None, batch_offsets=None, batch_data_size=None, max_level=None,
            need_input_grad=None):
    """-> (y[N,F] params.dtype, dy_dx[N,F*D] input.dtype | None)   (lotd_torch_api.cu:232-365)"""
    _no_batch(batch_inds, batch_offsets, batch_data_size)
    _check_params(lod_meta, params)
    if input.dim() != 2 or input.shape[1] != lod_meta.n_dims_to_encode:
        raise RuntimeError(f"lod_fwd: expected input of shape [N,{lod_meta.n_dims_to_encode}]")
    if input.dtype != torch.float32:
        raise RuntimeError("neuralsim_b200 LoTD: input must be float32 (the <float, half|float> instantiations)")
    n = input.shape[0]
    need = bool(input.requires_grad) if need_input_grad is None else bool(need_input_grad)
    ml = lod_meta.n_levels if max_level is None else int(max_level)
    y = torch.empty((n, lod_meta.n_encoded_dims), dtype=params.dtype, device=input.device)
    dy_dx = torch.empty((n, lod_meta.n_encoded_dims * lod_meta.n_dims_to_encode), dtype=torch.float32,
                        device=input.device) if need else None
    with L.KERNEL_TIMER.time("lotd_gather", n):
        L.check(L.lib().nsb_lotd_fwd(lod_meta.c_ref, L.ptr(input, "f32", "input"), L.ptr(params, None, "params"),
                                     ctypes.c_int(params.dtype == torch.float16), L.c_i64(n), L.c_i32(ml), L.ptr(y),
                                     L.ptr(dy_dx, "f32", allow_none=True), L.stream_ptr()), "lod_fwd")
    return y, dy_dx


def lod_bwd(lod_meta, dL_dy, input, params, dy_dx=None, batch_inds=None, batch_offsets=None, batch_data_size=None,
            max_level=None, need_input_grad=None, need_param_grad=None):
    """-> (dL_dx[N,D] | None, dL_dparam[P] params.dtype | None)      (lotd_torch_api.cu:397-520)"""
    _no_batch(batch_inds, batch_offsets, batch_data_size)
    _check_params(lod_meta, params)
    n = input.shape[0]
    ml = lod_meta.n_levels if max_level is None else int(max_level)
    need_x = bool(input.requires_grad) if need_input_grad is None else bool(need_input_grad)
    need_p = bool(params.requires_grad) if need_param_grad is None else bool(need_param_grad)
    dL_dy = dL_dy.contiguous()
    if dL_dy.dtype != params.dtype:
        raise RuntimeError("lod_bwd: dL_dy must have the dtype of params")
    is_half = ctypes.c_int(dL_dy.dtype == torch.float16)
    dL_dx = dL_dp = None
    if need_x:
        if dy_dx is None:
            raise RuntimeError("LoTDEncoding::bwd: need `dy_dx` to comput `dL_dx`.")
        dL_dx = torch.empty((n, lod_meta.n_dims_to_encode), dtype=torch.float32, device=input.device)
        L.check(L.lib().nsb_lotd_bwd_input(L.ptr(dL_dy), is_half, L.ptr(dy_dx.contiguous(), "f32", "dy_dx"), L.c_i64(n),
                                           L.c_i32(lod_meta.n_encoded_dims), L.c_i32(lod_meta.n_dims_to_encode),
                                           L.c_f32(1.0), L.ptr(dL_dx), L.stream_ptr()), "lod_bwd")
    if need_p:
        acc = torch.zeros(params.shape[0], dtype=torch.float32, device=input.device)
        with L.KERNEL_TIMER.time("lotd_bwd_grid", n):
            L.check(L.lib().nsb_lotd_bwd_grid(lod_meta.c_ref, L.ptr(dL_dy), is_half, L.ptr(input, "f32", "input"), L.c_i64(n),
                                              L.c_i32(ml), L.c_f32(1.0), L.ptr(acc), L.stream_ptr()), "lod_bwd")
        dL_dp = acc.to(params.dtype)
    return dL_dx, dL_dp


def lod_bwd_bwd_input(lod_meta, dL_ddLdx, dL_dy, input, params, dy_dx=None, batch_inds=None, batch_offsets=None,
                      batch_data_size=None, max_level=None, need_dLdinput_ddLdoutput=None, need_dLdinput_dparams=None,
                      need_dLdinput_dinput=None):
    """-> (dL_ddLdy[N,F] | None, dL_dparams[P] | None, dL_dinput | None)  (lotd_torch_api.cu:536-730)"""
    _no_batch(batch_inds, batch_offsets, batch_data_size)
    _check_params(lod_meta, params)
    if need_dLdinput_dinput:
        raise RuntimeError("neuralsim_b200 LoTD: d(dL_dx)/dx is not built (the reference disables it, lotd.py:256)")
    n = input.shape[0]
    ml = lod_meta.n_levels if max_level is None else int(max_level)
    need_y = bool(dL_dy.requires_grad) if need_dLdinput_ddLdoutput is None else bool(need_dLdinput_ddLdoutput)
    need_p = bool(params.requires_grad) if need_dLdinput_dparams is None else bool(need_dLdinput_dparams)
    dL_dy = dL_dy.contiguous()
    out_y = torch.empty((n, lod_meta.n_encoded_dims), dtype=torch.float32, device=input.device) if need_y else None
    acc = torch.zeros(params.shape[0], dtype=torch.float32, device=input.device) if need_p else None
    if need_y and dy_dx is None:
        raise RuntimeError("LoTDEncoding::bwd_bwd_input: need `dy_dx` to compute `dL_d(dLdy)`.")
    with L.KERNEL_TIMER.time("lotd_bwd_bwd", n):
      L.check(L.lib().nsb_lotd_bwd_bwd_input(
        lod_meta.c_ref, L.ptr(dL_ddLdx.contiguous(), "f32", "dL_ddLdx"), L.ptr(dL_dy), ctypes.c_int(dL_dy.dtype == torch.float16),
        L.ptr(input, "f32", "input"), L.ptr(None if dy_dx is None else dy_dx.contiguous(), "f32", allow_none=True),
        L.c_i64(n), L.c_i32(ml), L.c_f32(1.0), L.ptr(out_y, allow_none=True), L.ptr(acc, allow_none=True),
        L.stream_ptr()), "lod_bwd_bwd_input")
    return (None if out_y is None else out_y.to(dL_dy.dtype)), (None if acc is None else acc.to(params.dtype)), None


def lod_get_grid_index(*a, **k):
    """lotd.cpp: debugging helper that returns the table indices of the corners; not on any training / rendering path"""
    raise RuntimeError("_lotd.lod_get_grid_index is not built in neuralsim_b200 (debug helper outside the hot path)")
