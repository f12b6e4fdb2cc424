"""Batched LoTD tables on the CPU, stated on top of the unbatched oracle (oracle/lotd.py).  TEST INFRASTRUCTURE.

`params` holds several tables of n_params elements (lotd_hash_only.h:44-55): point i reads batch b = batch_inds[i] (negative: the
point is skipped), else i // batch_data_size, else 0; its table starts at batch_offsets[b], else at b * n_params.  Every function here
slices the table each group of points reads, calls the unbatched oracle on those points, and scatters the result back: rows into
their places (skipped points keep zero rows), table gradients added into the table's slice (tables that share or overlap elements
add up).  Without a batch argument each function is the unbatched one.
"""
from __future__ import annotations

import numpy as np

from . import lotd as olotd


def tables(meta, n, batch_inds=None, batch_offsets=None, batch_data_size=None):
    """-> {start of a table in params: rows of the points that read it}; None when there is no batch argument"""
    if batch_inds is None and batch_offsets is None and not batch_data_size:
        return None
    if batch_inds is not None:
        b = np.asarray(batch_inds, dtype=np.int64)
    else:
        b = np.arange(n, dtype=np.int64) // int(batch_data_size) if batch_data_size else np.zeros(n, dtype=np.int64)
    keep = b >= 0
    start = np.full(n, -1, dtype=np.int64)
    start[keep] = np.asarray(batch_offsets, dtype=np.int64)[b[keep]] if batch_offsets is not None else b[keep] * meta.n_params
    return {int(s): np.nonzero(start == s)[0] for s in np.unique(start[keep])}


def lod_fwd(meta, x, params, max_level=None, need_input_grad=False, batch_inds=None, batch_offsets=None, batch_data_size=None):
    """olotd.lod_fwd per table: y [N,F_total], dy_dx [N,F_total,D] | None"""
    x = np.asarray(x, dtype=np.float32)
    groups = tables(meta, len(x), batch_inds, batch_offsets, batch_data_size)
    if groups is None:
        return olotd.lod_fwd(meta, x, params, max_level, need_input_grad)
    y = np.zeros((len(x), meta.n_encoded_dims), dtype=params.dtype)
    dy_dx = np.zeros((len(x), meta.n_encoded_dims, x.shape[1]), dtype=np.float32) if need_input_grad else None
    for s, rows in groups.items():
        y[rows], d = olotd.lod_fwd(meta, x[rows], params[s:s + meta.n_params], max_level, need_input_grad)
        if need_input_grad:
            dy_dx[rows] = d
    return y, dy_dx


def lod_bwd_grid(meta, dL_dy, x, n_params, max_level=None, batch_inds=None, batch_offsets=None, batch_data_size=None):
    """olotd.lod_bwd_grid per table: dL_dparam [n_params] float64"""
    x = np.asarray(x, dtype=np.float32)
    groups = tables(meta, len(x), batch_inds, batch_offsets, batch_data_size)
    if groups is None:
        return olotd.lod_bwd_grid(meta, dL_dy, x, n_params, max_level)
    grad = np.zeros(n_params, dtype=np.float64)
    for s, rows in groups.items():
        grad[s:s + meta.n_params] += olotd.lod_bwd_grid(meta, dL_dy[rows], x[rows], meta.n_params, max_level)
    return grad


def lod_bwd_bwd_input(meta, dL_ddLdx, dL_dy, x, params, dy_dx=None, max_level=None, need_dLdy=True, need_param=True, need_input=False,
                      batch_inds=None, batch_offsets=None, batch_data_size=None):
    """olotd.lod_bwd_bwd_input per table: (dL_ddLdy [N,F] fp32 | None, dL_dparam [P] fp64 | None, None)"""
    x = np.asarray(x, dtype=np.float32)
    groups = tables(meta, len(x), batch_inds, batch_offsets, batch_data_size)
    if groups is None:
        return olotd.lod_bwd_bwd_input(meta, dL_ddLdx, dL_dy, x, params, dy_dx, max_level, need_dLdy, need_param, need_input)
    gin = np.asarray(dL_ddLdx, dtype=np.float32)
    out_dLdy = np.zeros((len(x), meta.n_encoded_dims), dtype=np.float32) if need_dLdy else None
    out_param = np.zeros(params.shape[0], dtype=np.float64) if need_param else None
    for s, rows in groups.items():
        a, b, _ = olotd.lod_bwd_bwd_input(meta, gin[rows], dL_dy[rows], x[rows], params[s:s + meta.n_params],
                                          None if dy_dx is None else dy_dx[rows], max_level, need_dLdy, need_param, need_input)
        if need_dLdy:
            out_dLdy[rows] = a
        if need_param:
            out_param[s:s + meta.n_params] += b
    return out_dLdy, out_param, None


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


class backend(olotd.backend):
    """Drop-in for `nr3d_lib.bindings._lotd` on CPU tensors, batch arguments included"""

    @staticmethod
    def lod_fwd(meta, input, params, batch_inds=None, batch_offsets=None, batch_data_size=None, max_level=None, need_input_grad=None):
        import torch
        need = bool(input.requires_grad) if need_input_grad is None else need_input_grad
        y, dydx = lod_fwd(meta, _np(input), _np(params), max_level, need, _np(batch_inds), _np(batch_offsets), batch_data_size)
        return torch.from_numpy(y), None if dydx is None else torch.from_numpy(dydx.reshape(dydx.shape[0], -1))

    @staticmethod
    def lod_bwd(meta, dL_dy, input, params, dy_dx=None, batch_inds=None, batch_offsets=None, batch_data_size=None, max_level=None,
                need_input_grad=None, need_param_grad=None):
        import torch
        dL_dx = dL_dp = None
        if need_input_grad:     # skipped points have zero dy_dx rows, hence zero dL_dx rows
            dL_dx = torch.from_numpy(olotd.lod_bwd_input(_np(dL_dy), _np(dy_dx).reshape(input.shape[0], meta.n_encoded_dims, -1)))
        if need_param_grad:
            g = lod_bwd_grid(meta, _np(dL_dy), _np(input), params.shape[0], max_level, _np(batch_inds), _np(batch_offsets), batch_data_size)
            dL_dp = torch.from_numpy(g).to(params.dtype)
        return dL_dx, dL_dp

    @staticmethod
    def lod_bwd_bwd_input(meta, dL_ddLdx, dL_dy, input, params, dy_dx=None, batch_inds=None, batch_offsets=None, batch_data_size=None,
                          max_level=None, need_dLdinput_ddLdoutput=None, need_dLdinput_dparams=None, need_dLdinput_dinput=None):
        import torch
        a, b, _ = lod_bwd_bwd_input(
            meta, _np(dL_ddLdx), _np(dL_dy), _np(input), _np(params),
            None if dy_dx is None else _np(dy_dx).reshape(input.shape[0], meta.n_encoded_dims, -1), max_level,
            bool(need_dLdinput_ddLdoutput), bool(need_dLdinput_dparams), bool(need_dLdinput_dinput),
            _np(batch_inds), _np(batch_offsets), batch_data_size)
        return (None if a is None else torch.from_numpy(a).to(dL_dy.dtype)), (None if b is None else torch.from_numpy(b).to(params.dtype)), None
