"""Drop-in for `nr3d_lib.bindings._pack_ops` (reference: nr3d_lib/csrc/pack_ops/pack_ops.cpp:20-58) over the C ABI.

fp32 feature tensors, int64 pack_infos [P,2] -- the types the rendering path uses.  Unlike the reference wrappers
(`pack_infos.index({-1,0}).item()` in every call, e.g. pack_ops_cuda.cu:839) nothing here synchronises the host,
except where the output size itself is data dependent (interleave_*), exactly as many syncs as unavoidable.
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib as L

_OPS = dict(add=0, sub=1, mul=2, div=3, gt=4, geq=5, lt=6, leq=7, eq=8, neq=9)


def _f32(t, name):
    if t.dtype != torch.float32:
        raise RuntimeError(f"neuralsim_b200 pack_ops: {name} must be float32, got {t.dtype}")
    return t.contiguous()


def _pi(pack_infos):
    if pack_infos.dtype != torch.int64 or pack_infos.dim() != 2 or pack_infos.shape[1] != 2:
        raise RuntimeError("pack_infos must be an int64 tensor of shape [num_packs, 2]")
    return pack_infos.contiguous()


def _binary(name):
    op = _OPS[name]

    def fn(feats, other, pack_infos):
        feats, other, pack_infos = _f32(feats, "feats"), _f32(other, "other"), _pi(pack_infos)
        C = 1 if feats.dim() == 1 else feats.shape[1]
        if other.shape[0] != pack_infos.shape[0] or other.numel() != pack_infos.shape[0] * C:
            raise RuntimeError(f"packed_{name}: `other` must be [num_packs{', feat_dim' if C > 1 else ''}]")
        out = torch.empty_like(feats) if op <= 3 else torch.empty(feats.shape, dtype=torch.bool, device=feats.device)
        L.check(L.lib().nsb_packed_binary(ctypes.c_int(op), L.ptr(feats), L.ptr(other), L.ptr(pack_infos),
                                          L.c_i64(pack_infos.shape[0]), L.c_i32(C), L.ptr(out), L.stream_ptr()), f"packed_{name}")
        return out
    fn.__name__ = f"packed_{name}"
    return fn


packed_add, packed_sub, packed_mul, packed_div = (_binary(n) for n in ("add", "sub", "mul", "div"))
packed_gt, packed_geq, packed_lt, packed_leq, packed_eq, packed_neq = (_binary(n) for n in ("gt", "geq", "lt", "leq", "eq", "neq"))


def packed_matmul(feats, other, pack_infos):
    """out[i] = other[pack(i)] @ feats[i]  (kernel_packed_matmul); small per-ray rotations of code_multi."""
    o = torch.repeat_interleave(other, pack_infos[:, 1], dim=0)
    return (o * feats.unsqueeze(-2)).sum(-1)


def packed_sum(feats, pack_infos):
    feats, pack_infos = _f32(feats, "feats"), _pi(pack_infos)
    C = 1 if feats.dim() == 1 else feats.shape[1]
    P = pack_infos.shape[0]
    out = torch.empty((P,) if feats.dim() == 1 else (P, C), dtype=torch.float32, device=feats.device)
    L.check(L.lib().nsb_packed_sum(L.ptr(feats), L.ptr(pack_infos), L.c_i64(P), L.c_i32(C), L.ptr(out), L.stream_ptr()), "packed_sum")
    return out


def packed_cumsum(feats, pack_infos, exclusive=False, reverse=False):
    feats, pack_infos = _f32(feats, "feats"), _pi(pack_infos)
    C = 1 if feats.dim() == 1 else feats.shape[1]
    out = torch.empty_like(feats)
    L.check(L.lib().nsb_packed_cumsum(L.ptr(feats), L.ptr(pack_infos), L.c_i64(pack_infos.shape[0]), L.c_i32(C),
                                      ctypes.c_int(bool(exclusive)), ctypes.c_int(bool(reverse)), L.ptr(out), L.stream_ptr()),
            "packed_cumsum")
    return out


def packed_cumprod(feats, pack_infos, exclusive=False, reverse=False):
    """Not on the rendering path (packed_alpha_to_vw replaced it, nerf_utils.py:47-60).  Inclusive only: the
    reference's exclusive variant returns zeros by construction (pack_ops_cuda.cu:951 + :884-893)."""
    if exclusive:
        return torch.zeros_like(feats)
    lg = packed_cumsum(torch.log(feats.abs().clamp_min(1e-38)), pack_infos, False, reverse)
    neg = packed_cumsum((feats < 0).float(), pack_infos, False, reverse)
    return torch.exp(lg) * (1 - 2 * (neg.long() % 2)).to(feats.dtype)


def _diff(feats, pack_infos, edge_val, edge_fill, backward, who):
    feats, pack_infos = _f32(feats, "feats"), _pi(pack_infos)
    C = 1 if feats.dim() == 1 else feats.shape[1]
    out = torch.empty_like(feats)
    ev = None if edge_val is None else _f32(edge_val, "pack edge values")
    ef = None if edge_fill is None else _f32(edge_fill, "pack edge fill")
    L.check(L.lib().nsb_packed_diff(L.ptr(feats), L.ptr(pack_infos), L.c_i64(pack_infos.shape[0]), L.c_i32(C),
                                    L.ptr(ev, allow_none=True), L.ptr(ef, allow_none=True), ctypes.c_int(backward),
                                    L.ptr(out), L.stream_ptr()), who)
    return out


def packed_diff(feats, pack_infos, pack_appends=None, pack_last_fill=None):
    return _diff(feats, pack_infos, pack_appends, pack_last_fill, 0, "packed_diff")


def packed_backward_diff(feats, pack_infos, pack_prepends=None, pack_first_fill=None):
    return _diff(feats, pack_infos, pack_prepends, pack_first_fill, 1, "packed_backward_diff")


def packed_searchsorted(bins, vals, pack_infos):
    bins, vals, pack_infos = _f32(bins, "bins"), _f32(vals, "vals"), _pi(pack_infos)
    if vals.dim() != 2 or vals.shape[0] != pack_infos.shape[0]:
        raise RuntimeError("packed_searchsorted: vals must be [num_packs, n]")
    out = torch.empty(vals.shape, dtype=torch.int64, device=vals.device)
    L.check(L.lib().nsb_packed_searchsorted(L.ptr(bins), L.ptr(vals), L.ptr(pack_infos), L.c_i64(vals.shape[0]),
                                            L.c_i32(vals.shape[1]), L.ptr(out), L.stream_ptr()), "packed_searchsorted")
    return out


def packed_invert_cdf(bins, cdfs, u_vals, pack_infos):
    bins, cdfs, u_vals, pack_infos = _f32(bins, "bins"), _f32(cdfs, "cdfs"), _f32(u_vals, "u_vals"), _pi(pack_infos)
    if bins.shape != cdfs.shape or u_vals.dim() != 2 or u_vals.shape[0] != pack_infos.shape[0]:
        raise RuntimeError("packed_invert_cdf: expected bins/cdfs [S], u_vals [num_packs, n]")
    samples = torch.empty_like(u_vals)
    bidx = torch.empty(u_vals.shape, dtype=torch.int64, device=u_vals.device)
    L.check(L.lib().nsb_packed_invert_cdf(L.ptr(bins), L.ptr(cdfs), L.ptr(u_vals), L.ptr(pack_infos), L.c_i64(u_vals.shape[0]),
                                          L.c_i32(u_vals.shape[1]), L.ptr(samples), L.ptr(bidx), L.stream_ptr()), "packed_invert_cdf")
    return samples, bidx


def try_merge_two_packs_sorted_aligned(vals_a, pack_infos_a, vals_b, pack_infos_b, b_sorted=True):
    vals_a, vals_b = _f32(vals_a, "vals_a"), _f32(vals_b, "vals_b")
    pa, pb = _pi(pack_infos_a), _pi(pack_infos_b)
    if pa.shape != pb.shape:
        raise RuntimeError("try_merge_two_packs_sorted_aligned: the two pack_infos must be aligned (same num_packs)")
    n_per = pa[:, 1] + pb[:, 1]
    cs = n_per.cumsum(0)
    pack_infos = torch.stack([cs - n_per, n_per], 1).contiguous()
    pidx_a = torch.empty(vals_a.shape[0], dtype=torch.int64, device=vals_a.device)
    pidx_b = torch.empty(vals_b.shape[0], dtype=torch.int64, device=vals_b.device)
    L.check(L.lib().nsb_merge_two_packs_sorted_aligned(L.ptr(vals_a), L.ptr(pa), L.ptr(vals_b), L.ptr(pb), L.ptr(pack_infos),
                                                       L.c_i64(pa.shape[0]), ctypes.c_int(bool(b_sorted)), L.ptr(pidx_a),
                                                       L.ptr(pidx_b), L.stream_ptr()), "try_merge_two_packs_sorted_aligned")
    return pidx_a, pidx_b, pack_infos


def packed_alpha_to_vw_forward(alphas, pack_infos, early_stop_eps, alpha_thre, compression):
    alphas, pack_infos = _f32(alphas, "alphas"), _pi(pack_infos)
    if alphas.dim() != 1:
        raise RuntimeError("packed_alpha_to_vw_forward: alphas must be 1-D")
    P = pack_infos.shape[0]
    if compression:
        steps = torch.empty(P, dtype=torch.int64, device=alphas.device)
        sel = torch.empty(alphas.shape[0], dtype=torch.bool, device=alphas.device)
        L.check(L.lib().nsb_packed_alpha_to_vw_forward(L.ptr(alphas), L.ptr(pack_infos), L.c_i64(P), L.c_f32(early_stop_eps),
                                                       L.c_f32(alpha_thre), None, L.ptr(steps), L.ptr(sel), L.stream_ptr()),
                "packed_alpha_to_vw_forward")
        cs = steps.cumsum(0)
        return None, torch.stack([cs - steps, steps], 1), sel
    w = torch.empty_like(alphas)
    L.check(L.lib().nsb_packed_alpha_to_vw_forward(L.ptr(alphas), L.ptr(pack_infos), L.c_i64(P), L.c_f32(early_stop_eps),
                                                   L.c_f32(alpha_thre), L.ptr(w), None, None, L.stream_ptr()),
            "packed_alpha_to_vw_forward")
    return w, None, None


def packed_alpha_to_vw_backward(weights, grad_weights, alphas, pack_infos, early_stop_eps, alpha_thre):
    weights, grad_weights, alphas = _f32(weights, "weights"), _f32(grad_weights, "grad_weights"), _f32(alphas, "alphas")
    pack_infos = _pi(pack_infos)
    ga = torch.empty_like(alphas)
    L.check(L.lib().nsb_packed_alpha_to_vw_backward(L.ptr(weights), L.ptr(grad_weights), L.ptr(alphas), L.ptr(pack_infos),
                                                    L.c_i64(pack_infos.shape[0]), L.c_f32(early_stop_eps), L.c_f32(alpha_thre),
                                                    L.ptr(ga), L.stream_ptr()), "packed_alpha_to_vw_backward")
    return ga


def interleave_arange(stop, return_idx=True):
    stop = stop.contiguous()
    if stop.dtype != torch.int64:
        raise RuntimeError("interleave_arange: stop must be int64")
    cs = stop.cumsum(0)
    total = int(cs[-1].item()) if stop.numel() else 0     # output size is data dependent: one sync
    out = torch.empty(total, dtype=torch.int64, device=stop.device)
    nidx = torch.empty(total, dtype=torch.int64, device=stop.device) if return_idx else None
    L.check(L.lib().nsb_interleave_arange(L.ptr(stop), L.ptr(cs), L.c_i64(stop.shape[0]), L.ptr(out),
                                          L.ptr(nidx, allow_none=True), L.stream_ptr()), "interleave_arange")
    return out, nidx


def interleave_linstep(start, num_steps, step_size, return_idx=True):
    start = _f32(start, "start")
    num_steps = num_steps.contiguous()
    if num_steps.dtype != torch.int64:
        raise RuntimeError("interleave_linstep: num_steps must be int64")
    cs = num_steps.cumsum(0)
    total = int(cs[-1].item()) if num_steps.numel() else 0
    out = torch.empty(total, dtype=torch.float32, device=start.device)
    nidx = torch.empty(total, dtype=torch.int64, device=start.device) if return_idx else None
    st = _f32(step_size, "step_size") if isinstance(step_size, torch.Tensor) else None
    L.check(L.lib().nsb_interleave_linstep(L.ptr(start), L.ptr(num_steps), L.ptr(cs), L.ptr(st, allow_none=True),
                                           L.c_f32(0.0 if st is not None else step_size), L.c_i64(start.shape[0]), L.ptr(out),
                                           L.ptr(nidx, allow_none=True), L.stream_ptr()), "interleave_linstep")
    return out, nidx


def packed_sort_qsort(vals, pack_infos, return_idx=True):
    """In place on `vals` (ascending per pack, stable, NaN last); returns the global gather indices, the identity on elements
    between packs (the reference's arange)."""
    if not vals.is_contiguous() or vals.dtype != torch.float32 or vals.dim() != 1:
        raise RuntimeError("packed_sort_qsort: vals must be a 1-D contiguous float32 tensor (sorted in place)")
    pack_infos = _pi(pack_infos)
    idx = torch.arange(vals.shape[0], dtype=torch.int64, device=vals.device) if return_idx else None
    L.check(L.lib().nsb_packed_sort(L.ptr(vals), L.c_i64(vals.shape[0]), L.ptr(pack_infos), L.c_i64(pack_infos.shape[0]),
                                    L.ptr(idx, allow_none=True), L.stream_ptr()), "packed_sort_qsort")
    return idx


def mark_pack_boundaries_cuda(ids):
    ids = ids.contiguous().long()
    out = torch.empty(ids.shape[0], dtype=torch.int32, device=ids.device)
    L.check(L.lib().nsb_mark_pack_boundaries(L.ptr(ids), L.c_i64(ids.shape[0]), L.ptr(out), L.stream_ptr()), "mark_pack_boundaries")
    return out


def packed_sort_thrust(vals, pack_infos, return_idx=True):
    """pack_ops.cpp: the thrust variant of the per-pack sort (commented out at its only call site, pack_ops.py:75): same contract as the qsort entry"""
    return packed_sort_qsort(vals, pack_infos, return_idx)


def _not_built(name, where):
    def fn(*a, **k):
        raise RuntimeError(f"_pack_ops.{name} is not built in neuralsim_b200: {where}")
    fn.__name__ = name
    return fn


# producers / searches no shipped NeuS query mode reaches (their callers: AABBSpace.ray_step_coarse `wrt_depth` modes, aabb.py:128;
# ForestBlockSpace, forest.py:407; octree segments): named so that a call fails with a message instead of an AttributeError
interleave_sample_step_wrt_depth_clamped = _not_built("interleave_sample_step_wrt_depth_clamped", "depth-proportional coarse stepping (CFG uses step_mode 'linear')")
interleave_sample_step_wrt_depth_in_packed_segments = _not_built("interleave_sample_step_wrt_depth_in_packed_segments", "forest block segments")
packed_searchsorted_packed_vals = _not_built("packed_searchsorted_packed_vals", "ragged search values (no caller on the NeuS path)")
octree_mark_consecutive_segments = _not_built("octree_mark_consecutive_segments", "octree (forest) ray segments")
