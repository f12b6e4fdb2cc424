"""CPU restatement of the LoTD Dense+Hash ("hash-only") grid encoding.  TEST INFRASTRUCTURE.

Follows (paths relative to nr3d_lib):
  meta            csrc/lotd/src/lotd_torch_api.cu:29-230   (LoDMeta::create_meta)
  config          nr3d_lib/models/grid_encodings/lotd/lotd_cfg.py:48-57 (gen_ngp_cfg)
  index / hash    csrc/lotd/include/lotd/lotd_cuda.h:92-143
  pos_fract       csrc/lotd/include/lotd/lotd_cuda.h:959-1084 (Linear interpolation only)
  interpolation   csrc/lotd/include/lotd/linear_interpolate.cuh:9-150
  forward         csrc/lotd/include/lotd/lotd_hash_only.h:15-267
  backward grid   csrc/lotd/include/lotd/lotd_hash_only.h:380-470, lotd_encoding.h:431-467
  bwd-bwd grid    csrc/lotd/include/lotd/lotd_hash_only.h:472-574, lotd_encoding.h:714-757
  dL_dx / dL_ddLdy  lotd_hash_only.h:839-856, 982-1001 (at::sum_out(at::mul(..)))

Arithmetic model (the <float input, half param, float compute> instantiation,
lotd_hash_only.h:777): positions and weights are fp32; a table value is fp16; each
corner's contribution `w * float(v)` is rounded to fp16 and *accumulated in fp16*
in corner order 0..7 (linear_interpolate.cuh:118, `result_ptr[f] += (PARAM_T)(...)`).
`pos = x*scale + 0.5` is evaluated as one fused multiply-add (nvcc contracts it).
Gradients wrt. the table are accumulated here in float64 (the reference uses
non-deterministic fp16 atomics, lotd_cuda.h:494-561, so it has no bit-exact value).
"""
from __future__ import annotations

import os

import numpy as np

DENSE = 0  # lotd_types.h:16-26 (enum LoDType)
HASH = 7
_PRIMES = np.array([1, 2654435761, 805459861, 3674653429], dtype=np.uint64)  # lotd_cuda.h:122


def gen_ngp_cfg(min_res=16, dim=3, n_feats=2, log2_hashmap_size=19, per_level_scale=1.382, num_levels=16):
    """lotd_cfg.py:48-57."""
    hashmap_size = 2 ** log2_hashmap_size
    level_res = (min_res * per_level_scale ** np.arange(num_levels)).astype(int)
    types = ["Dense" if int(r) ** dim <= hashmap_size else "Hash" for r in level_res]
    return dict(lod_res=level_res.tolist(), lod_n_feats=[n_feats] * num_levels, lod_types=types,
                hashmap_size=hashmap_size)


class LoDMeta:
    """Restates LoDMeta::create_meta (lotd_torch_api.cu:29-230) for Dense/Hash levels."""

    def __init__(self, n_input_dims, lod_res, lod_n_feats, lod_types, hashmap_size=None, use_smooth_step=False):
        if use_smooth_step:
            raise NotImplementedError("oracle covers InterpolationType::Linear only (hot path)")
        if n_input_dims not in (2, 3, 4):
            raise RuntimeError("LoTDEncoding: `n_input_dim` must be 2/3/4.")
        n_levels = len(lod_res)
        if isinstance(lod_n_feats, int):
            lod_n_feats = [lod_n_feats] * n_levels
        if isinstance(lod_types, str):
            lod_types = [lod_types] * n_levels
        if not (len(lod_n_feats) == n_levels == len(lod_types)):
            raise RuntimeError("LoTDEncoding: Expect los_res, lod_n_feats, lod_str_types to have the same length")
        if n_levels > 32:
            raise RuntimeError("LoTDEncoding: num_level exceeds maximum level=32")
        self.n_dims_to_encode = n_input_dims
        self.n_levels = n_levels
        self.level_types_str = list(lod_types)
        for g in (8, 4, 2):
            if all(f % g == 0 for f in lod_n_feats):
                self.n_feat_per_pseudo_lvl = g
                break
        else:
            raise RuntimeError("LoTDEncoding: the greatest common divisor of `lod_n_feats` must be at least 2")
        self.level_res_multidim, self.level_res = [], []
        self.level_n_feats, self.level_types = [], []
        self.level_sizes, self.level_n_params, self.level_offsets = [], [], []
        self.map_levels, self.map_cnt = [], []
        self.n_encoded_dims = 0
        acc = 0
        for lvl in range(n_levels):
            res = lod_res[lvl]
            res = [int(res)] * n_input_dims if np.isscalar(res) else [int(r) for r in res]
            if any(r <= 2 for r in res):
                raise RuntimeError("LoTDEncoding: only support grid resolutions >= 3")
            t = lod_types[lvl].lower()
            if t == "dense":
                typ, size = DENSE, int(np.prod(res))
            elif t == "hash":
                if not hashmap_size:
                    raise RuntimeError("LoTDEncoding: Hash mode need `hashmap_size`")
                typ, size = HASH, int(hashmap_size)
            else:
                raise NotImplementedError(f"oracle covers Dense/Hash only, got {lod_types[lvl]}")
            nf = int(lod_n_feats[lvl])
            self.level_res_multidim.append(res)
            self.level_res.append(res[0] if all(r == res[0] for r in res) else 0)
            self.level_n_feats.append(nf)
            self.level_types.append(typ)
            self.level_sizes.append(size)
            self.level_n_params.append(size * nf)
            self.level_offsets.append(acc)
            acc += size * nf
            for j in range(nf // self.n_feat_per_pseudo_lvl):
                self.map_levels.append(lvl)
                self.map_cnt.append(j)
            self.n_encoded_dims += nf
        self.level_offsets.append(acc)
        self.n_params = acc
        self.n_pseudo_levels = len(self.map_levels)
        self.c_hash_only = True


def _f32(a):
    return np.asarray(a, dtype=np.float32)


def pos_fract(x, scale):
    """lotd_cuda.h:959-984 (Linear).  x [N,D] fp32 in [0,1]; scale [D] -> (cell uint32 [N,D], frac fp32 [N,D]).
    `x*scale+0.5` as one FMA: the product of two fp32 is exact in fp64, and for |x|<=1, scale<2^12 the
    fp64 sum with 0.5 is exact too, so a single rounding to fp32 equals fmaf()."""
    v = (x.astype(np.float64) * scale.astype(np.float64) + 0.5).astype(np.float32)
    fl = np.floor(v)
    return fl.astype(np.uint32), (v - fl).astype(np.float32)


def grid_index(meta: LoDMeta, level: int, cell):
    """lotd_cuda.h:92-143.  cell [N,D] uint32 -> element index (not yet times n_feat)."""
    D = meta.n_dims_to_encode
    res = meta.level_res_multidim[level]
    if meta.level_types[level] == DENSE:
        idx = np.zeros(cell.shape[0], dtype=np.uint64)
        stride = 1
        for d in range(D - 1, -1, -1):  # last dim (z) contiguous; uint32 wrap-around as on device
            idx = (idx + cell[:, d].astype(np.uint64) * stride) & 0xFFFFFFFF
            stride = (stride * res[d]) & 0xFFFFFFFF
        return idx.astype(np.int64)
    h = np.zeros(cell.shape[0], dtype=np.uint64)
    for d in range(D):
        h ^= (cell[:, d].astype(np.uint64) * _PRIMES[d]) & 0xFFFFFFFF
    return (h % np.uint64(meta.level_sizes[level])).astype(np.int64)


def _corner_weights(frac, D):
    """Yield (corner idx, offset [D], weight fp32 [N]) in the reference order (bit d of idx -> +1 on dim d)."""
    one = np.float32(1.0)
    for idx in range(1 << D):
        w = np.ones(frac.shape[0], dtype=np.float32)
        off = np.zeros(D, dtype=np.uint32)
        for d in range(D):
            if idx & (1 << d):
                w = w * frac[:, d]
                off[d] = 1
            else:
                w = w * (one - frac[:, d])
        yield idx, off, w


def _half_add(a16, b16):
    """Correctly-rounded fp16 addition (the exact sum of two fp16 fits fp64)."""
    return (a16.astype(np.float64) + b16.astype(np.float64)).astype(np.float16)


THREADS = [None]            # None: min(16, usable cores); set to [1] to force the serial walk


def _usable_cpus():
    n = os.cpu_count() or 1
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = max(1, min(n, int(int(quota) / int(period))))
    except Exception:
        pass
    return n


def _for_levels(fn, levels, n_points):
    """The levels of the table are independent (disjoint output columns / gradient ranges): walk them on a thread pool (numpy releases the
    GIL inside its vector loops) -- the CPU port should use the host cores it has, like the GPU path uses its SMs."""
    nt = THREADS[0] or min(16, _usable_cpus())
    if nt <= 1 or len(levels) <= 1 or n_points < 2048:
        for l in levels:
            fn(l)
        return
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(nt, len(levels))) as ex:
        list(ex.map(fn, levels))


def _level_iter(meta, max_level):
    F = meta.n_feat_per_pseudo_lvl
    for psl in range(meta.n_pseudo_levels):
        lvl = meta.map_levels[psl]
        if lvl > max_level:
            continue
        yield psl, lvl, meta.level_offsets[lvl], meta.map_cnt[psl] * F, psl * F


def lod_fwd(meta: LoDMeta, x, params, max_level=None, need_input_grad=False):
    """y [N,F_total] (dtype of params), dy_dx [N,F_total,D] fp32 | None.
    lotd_hash_only.h:15-267 + lotd_torch_api.cu:232-320.  `x` must already be clamped to [1e-6,1-1e-6]
    (lotd.py:60)."""
    x = _f32(x)
    N, D = x.shape
    assert D == meta.n_dims_to_encode
    ptype = params.dtype
    assert ptype in (np.float16, np.float32)
    max_level = meta.n_levels if max_level is None else max_level
    Ft = meta.n_encoded_dims
    y = np.zeros((N, Ft), dtype=ptype)
    dy_dx = np.zeros((N, Ft, D), dtype=np.float32) if need_input_grad else None
    if max_level <= -1:
        return y, dy_dx
    F = meta.n_feat_per_pseudo_lvl

    def one_level(args):
        psl, lvl, loff, foff, ooff = args
        res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        nf = meta.level_n_feats[lvl]
        cell, frac = pos_fract(x, scale)
        vals = []
        acc = np.zeros((N, F), dtype=ptype)
        for idx, off, w in _corner_weights(frac, D):
            gi = grid_index(meta, lvl, cell + off) * nf + foff + loff
            v = params[gi[:, None] + np.arange(F)[None, :]]          # [N,F] ptype
            vals.append(v)
            contrib = (w[:, None] * v.astype(np.float32)).astype(ptype)
            acc = _half_add(acc, contrib) if ptype == np.float16 else (acc + contrib).astype(np.float32)
        y[:, ooff:ooff + F] = acc
        if need_input_grad:
            one = np.float32(1.0)
            for gd in range(D):
                g = np.zeros((N, F), dtype=np.float32)
                others = [d for d in range(D) if d != gd]
                for idx in range(1 << (D - 1)):
                    w = np.full(N, scale[gd], dtype=np.float32)     # scale * pos_derivative(=1)
                    left = 0
                    for k, d in enumerate(others):
                        if idx & (1 << k):
                            w = w * frac[:, d]
                            left += 1 << d
                        else:
                            w = w * (one - frac[:, d])
                    right = left + (1 << gd)
                    diff = vals[right].astype(np.float32) - vals[left].astype(np.float32)
                    # grads += w*diff is an FFMA on device: product exact in fp64, one rounding
                    g = (g.astype(np.float64) + w[:, None].astype(np.float64) * diff.astype(np.float64)).astype(np.float32)
                dy_dx[:, ooff:ooff + F, gd] = g

    _for_levels(one_level, list(_level_iter(meta, max_level)), N)
    return y, dy_dx


def lod_bwd_input(dL_dy, dy_dx):
    """dL_dx[n,d] = sum_f float(dL_dy[n,f]) * dy_dx[n,f,d]   (lotd_hash_only.h:839-856)."""
    return np.einsum("nf,nfd->nd", dL_dy.astype(np.float32).astype(np.float64), dy_dx.astype(np.float64)).astype(np.float32)


def lod_bwd_grid(meta: LoDMeta, dL_dy, x, n_params, max_level=None):
    """dL_dparam[P] in float64 (exact reduction): sum over points/corners of float(dL_dy)*w.
    lotd_hash_only.h:380-470 + lotd_encoding.h:431-467."""
    x = _f32(x)
    N, D = x.shape
    max_level = meta.n_levels if max_level is None else max_level
    grad = np.zeros(n_params, dtype=np.float64)
    if max_level <= -1:
        return grad
    F = meta.n_feat_per_pseudo_lvl
    g32 = dL_dy.astype(np.float32)
    def one_level(args):                     # every (pseudo) level writes its own range of `grad`
        psl, lvl, loff, foff, ooff = args
        res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        nf = meta.level_n_feats[lvl]
        cell, frac = pos_fract(x, scale)
        for idx, off, w in _corner_weights(frac, D):
            gi = grid_index(meta, lvl, cell + off) * nf + foff + loff
            for f in range(F):
                np.add.at(grad, gi + f, g32[:, ooff + f].astype(np.float64) * w.astype(np.float64))

    levels = list(_level_iter(meta, max_level))
    # pseudo levels of one level share its range (map_cnt): keep those on one thread; the shipped configurations have one pseudo level per level
    _for_levels(one_level, levels, N) if len({l[1] for l in levels}) == len(levels) else [one_level(l) for l in levels]
    return grad


def lod_bwd_bwd_input(meta: LoDMeta, dL_ddLdx, dL_dy, x, params, dy_dx=None, max_level=None,
                      need_dLdy=True, need_param=True, need_input=False):
    """Second-order pass of dL_dx = J^T dL_dy  (lotd_hash_only.h:951-1056).
    Returns (dL_ddLdy [N,F] fp32 | None, dL_dparam [P] fp64 | None, dL_dinput [N,D] fp32 | None)."""
    x = _f32(x)
    N, D = x.shape
    max_level = meta.n_levels if max_level is None else max_level
    F = meta.n_feat_per_pseudo_lvl
    gin = _f32(dL_ddLdx)
    g32 = dL_dy.astype(np.float32)
    out_dLdy = None
    if need_dLdy:
        assert dy_dx is not None
        out_dLdy = np.einsum("nd,nfd->nf", gin.astype(np.float64), dy_dx.astype(np.float64)).astype(np.float32)
    out_param = np.zeros(params.shape[0], dtype=np.float64) if need_param else None
    if need_input:
        # d(dL_dx)/dx (off-diagonal Hessian, lotd_hash_only.h:576-695) is disabled on the hot path
        # (lotd.py:256 passes need_dLdinput_dinput=False) and is not restated here.
        raise NotImplementedError("bwd_bwd wrt input is outside the hot path")
    out_input = None
    if max_level <= -1 or not need_param:
        return out_dLdy, out_param, None
    one = np.float32(1.0)
    for psl, lvl, loff, foff, ooff in _level_iter(meta, max_level):
        res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        nf = meta.level_n_feats[lvl]
        cell, frac = pos_fract(x, scale)
        for gd in range(D):
            others = [d for d in range(D) if d != gd]
            grad_in = (scale[gd] * gin[:, gd]).astype(np.float32)       # * pos_derivative (=1)
            for idx in range(1 << (D - 1)):
                w = grad_in.copy()
                off = np.zeros(D, dtype=np.uint32)
                for k, d in enumerate(others):
                    if idx & (1 << k):
                        w = w * frac[:, d]
                        off[d] = 1
                    else:
                        w = w * (one - frac[:, d])
                for side, sgn in ((0, -1.0), (1, 1.0)):
                    off[gd] = side
                    gi = grid_index(meta, lvl, cell + off) * nf + foff + loff
                    if need_param:  # linear_interpolate.cuh:188-237
                        for f in range(F):
                            np.add.at(out_param, gi + f, sgn * w.astype(np.float64) * g32[:, ooff + f].astype(np.float64))
    return out_dLdy, out_param, None


# ----------------------------------------------------------------------------------------------
# torch-facing backend with the `nr3d_lib.bindings._lotd` call signatures (csrc/lotd/src/lotd.cpp:22-107)
# ----------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy()


class backend:
    """Drop-in for `nr3d_lib.bindings._lotd` on CPU tensors (single, non-batched tables)."""
    LoDMeta = LoDMeta

    @staticmethod
    def lod_fwd(meta, input, params, batch_inds=None, batch_offsets=None, batch_data_size=None,
                max_level=None, need_input_grad=None):
        import torch
        assert batch_inds is None and batch_offsets is None and not batch_data_size
        need = bool(input.requires_grad) if need_input_grad is None else need_input_grad
        y, dydx = lod_fwd(meta, _np(input).astype(np.float32), _np(params), max_level, need)
        y = torch.from_numpy(y)
        dydx = torch.from_numpy(dydx.reshape(dydx.shape[0], -1)) if dydx is not None else None
        return y, dydx

    @staticmethod
    def lod_bwd(meta, dL_dy, input, params, dy_dx=None, batch_inds=None, batch_offsets=None,
                batch_data_size=None, max_level=None, need_input_grad=None, need_param_grad=None):
        import torch
        dL_dx = dL_dp = None
        N = input.shape[0]
        if need_input_grad:
            dL_dx = torch.from_numpy(lod_bwd_input(_np(dL_dy), _np(dy_dx).reshape(N, meta.n_encoded_dims, -1)))
        if need_param_grad:
            g = lod_bwd_grid(meta, _np(dL_dy), _np(input), params.shape[0], max_level)
            dL_dp = torch.from_numpy(g).to(params.dtype)
        return dL_dx, dL_dp

    @staticmethod
    def lod_bwd_bwd_input(meta, dL_ddLdx, dL_dy, input, params, dy_dx=None, batch_inds=None,
                          batch_offsets=None, batch_data_size=None, max_level=None,
                          need_dLdinput_ddLdoutput=None, need_dLdinput_dparams=None, need_dLdinput_dinput=None):
        import torch
        N = input.shape[0]
        a, b, c = lod_bwd_bwd_input(
            meta, _np(dL_ddLdx), _np(dL_dy), _np(input), _np(params),
            None if dy_dx is None else _np(dy_dx).reshape(N, meta.n_encoded_dims, -1), max_level,
            bool(need_dLdinput_ddLdoutput), bool(need_dLdinput_dparams), bool(need_dLdinput_dinput))
        a = None if a is None else torch.from_numpy(a).to(dL_dy.dtype)
        b = None if b is None else torch.from_numpy(b).to(params.dtype)
        c = None if c is None else torch.from_numpy(c)
        return a, b, c
