"""CPU restatement of the reference `_pack_ops` native extension.  TEST INFRASTRUCTURE.

"Packed" tensors are ragged per-ray arrays described by pack_infos[P,2] = (first index, length).
Every function follows a kernel of nr3d_lib/csrc/pack_ops/pack_ops_cuda.cu (cited per
function) and keeps its serial, one-thread-per-pack evaluation order so that fp32 results are the
ones a sequential loop produces.  Call signatures are those exported by
csrc/pack_ops/pack_ops.cpp:20-58, on CPU torch tensors.
"""
from __future__ import annotations

import numpy as np
import torch


def _np(t):
    return t.detach().cpu().numpy()


def _packs(pack_infos):
    pi = _np(pack_infos).astype(np.int64)
    return [(int(b), int(n)) for b, n in pi]


def _total(pack_infos):
    if pack_infos.shape[0] == 0:
        return 0
    return int(pack_infos[-1, 0] + pack_infos[-1, 1])


# ---------------------------------------------------------------- producers
def interleave_arange(stop, return_idx=True):
    """kernel_interleave_arange, pack_ops_cuda.cu:48-81 / 83-112: per pack 0..stop-1 (+ pack index)."""
    n = _np(stop).astype(np.int64)
    out = np.concatenate([np.arange(k, dtype=np.int64) for k in n]) if n.size else np.zeros(0, np.int64)
    nidx = np.repeat(np.arange(n.size, dtype=np.int64), n)
    return torch.from_numpy(out), (torch.from_numpy(nidx) if return_idx else None)


def interleave_linstep(start, num_steps, step_size, return_idx=True):
    """interleave_linstep_impl, pack_ops_cuda.cu:114-140: out[j] = start + (scalar)j * step_size, in start's dtype."""
    s = _np(start)
    n = _np(num_steps).astype(np.int64)
    step = _np(step_size) if isinstance(step_size, torch.Tensor) else np.full(s.shape, step_size, dtype=s.dtype)
    step = step.astype(s.dtype)
    nidx = np.repeat(np.arange(n.size, dtype=np.int64), n)
    j = np.concatenate([np.arange(k, dtype=np.int64) for k in n]) if n.size else np.zeros(0, np.int64)
    if s.dtype == np.float32:   # start + (float)j*step is one fused multiply-add in the compiled reference kernel (fp64 product is exact)
        jf = j.astype(np.float32).astype(np.float64)               # (scalar_t)j: rounds once j is past 2^24
        out = (s[nidx].astype(np.float64) + jf * step[nidx].astype(np.float64)).astype(np.float32)
    else:
        out = (s[nidx] + (j.astype(s.dtype) * step[nidx]).astype(s.dtype)).astype(s.dtype)
    return torch.from_numpy(out), (torch.from_numpy(nidx) if return_idx else None)


def mark_pack_boundaries_cuda(ids):
    """pack_ops_cuda.cu (kaolin-derived): 1 where ids[i] != ids[i-1] (and at i=0)."""
    a = _np(ids)
    out = np.ones(a.shape[0], dtype=np.int32)
    if a.shape[0] > 1:
        out[1:] = (a[1:] != a[:-1]).astype(np.int32)
    return torch.from_numpy(out)


# ---------------------------------------------------------------- per-pack broadcast arithmetic
def _bcast(op):
    def fn(feats, other, pack_infos):
        """kernel_packed_{add,...}, pack_ops_cuda.cu:1961-2250: feats[i] (op) other[pack(i)]."""
        n = pack_infos[:, 1]
        o = torch.repeat_interleave(other, n, dim=0)
        total = _total(pack_infos)
        assert feats.shape[0] == total, "feats size disagrees with pack_infos"
        return op(feats, o)
    return fn


packed_add = _bcast(lambda a, b: a + b)
packed_sub = _bcast(lambda a, b: a - b)
packed_mul = _bcast(lambda a, b: a * b)
packed_div = _bcast(lambda a, b: a / b)
packed_gt = _bcast(lambda a, b: a > b)
packed_geq = _bcast(lambda a, b: a >= b)
packed_lt = _bcast(lambda a, b: a < b)
packed_leq = _bcast(lambda a, b: a <= b)
packed_eq = _bcast(lambda a, b: a == b)
packed_neq = _bcast(lambda a, b: a != b)


def packed_matmul(feats, other, pack_infos):
    """kernel_packed_matmul: out[i] = other[pack(i)] @ feats[i]."""
    o = torch.repeat_interleave(other, pack_infos[:, 1], dim=0)
    return (o * feats.unsqueeze(-2)).sum(-1)


# ---------------------------------------------------------------- reductions / scans
def packed_sum(feats, pack_infos):
    """kernel_packed_sum, pack_ops_cuda.cu:799-822 (serial left-to-right sum per pack and channel)."""
    a = _np(feats)
    out = np.zeros((pack_infos.shape[0],) + a.shape[1:], dtype=a.dtype)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        if n > 0:
            out[p] = np.cumsum(a[b:b + n], axis=0, dtype=a.dtype)[-1]
    return torch.from_numpy(out)


def _scan(feats, pack_infos, exclusive, reverse, mul):
    a = _np(feats)
    out = np.zeros_like(a)
    f = np.cumprod if mul else np.cumsum
    for b, n in _packs(pack_infos):
        if n == 0:
            continue
        seg = a[b:b + n]
        if reverse:
            seg = seg[::-1]
        if exclusive:
            # pack_ops_cuda.cu:884-893 / 1001-1011: out[begin] keeps its zero initialisation, then
            # out[i] = in[i-1] (op) out[i-1].  For cumprod this yields all zeros (reference quirk).
            r = np.zeros_like(seg)
            for i in range(1, n):
                r[i] = (seg[i - 1] * r[i - 1]) if mul else (seg[i - 1] + r[i - 1])
        else:
            r = f(seg, axis=0, dtype=a.dtype)
        out[b:b + n] = r[::-1] if reverse else r
    return torch.from_numpy(out)


def packed_cumsum(feats, pack_infos, exclusive=False, reverse=False):
    """kernel_packed_cumsum(_reverse), pack_ops_cuda.cu:983-1046."""
    return _scan(feats, pack_infos, exclusive, reverse, mul=False)


def packed_cumprod(feats, pack_infos, exclusive=False, reverse=False):
    """kernel_packed_cumprod(_reverse), pack_ops_cuda.cu:866-935."""
    return _scan(feats, pack_infos, exclusive, reverse, mul=True)


def packed_diff(feats, pack_infos, pack_appends=None, pack_last_fill=None):
    """kernel_packed_diff, pack_ops_cuda.cu:1099-1142: out[i]=in[i+1]-in[i]; last = append-in[last] | fill | 0."""
    a = _np(feats)
    out = np.zeros_like(a)
    ap = None if pack_appends is None else _np(pack_appends)
    lf = None if pack_last_fill is None else _np(pack_last_fill)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        if n == 0:
            continue
        out[b:b + n - 1] = a[b + 1:b + n] - a[b:b + n - 1]
        if ap is not None:
            out[b + n - 1] = ap[p] - a[b + n - 1]
        elif lf is not None:
            out[b + n - 1] = lf[p]
    return torch.from_numpy(out)


def packed_backward_diff(feats, pack_infos, pack_prepends=None, pack_first_fill=None):
    """kernel_packed_backward_diff, pack_ops_cuda.cu:1144-1187."""
    a = _np(feats)
    out = np.zeros_like(a)
    pp = None if pack_prepends is None else _np(pack_prepends)
    ff = None if pack_first_fill is None else _np(pack_first_fill)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        if n == 0:
            continue
        out[b + 1:b + n] = a[b + 1:b + n] - a[b:b + n - 1]
        if pp is not None:
            out[b] = a[b] - pp[p]
        elif ff is not None:
            out[b] = ff[p]
    return torch.from_numpy(out)


# ---------------------------------------------------------------- search / merge / sort
def _lower_bound(data, val):
    """binary_search_unsafe, pack_ops_cuda.cu:1336-1363: first i with !(data[i] < val)."""
    first, count = 0, len(data)
    while count > 0:
        step = count // 2
        it = first + step
        if data[it] < val:
            first = it + 1
            count -= step + 1
        else:
            count = step
    return first


def _binary_search(data, val):
    """binary_search, pack_ops_cuda.cu:1365-1372: clamped to length-1."""
    if len(data) == 0:
        return 0
    return min(_lower_bound(data, val), len(data) - 1)


def packed_searchsorted(bins, vals, pack_infos):
    """kernel_packed_searchsorted, pack_ops_cuda.cu:1375-1407 -> global indices int64 [P,n]."""
    b_, v_ = _np(bins), _np(vals)
    out = np.zeros(v_.shape, dtype=np.int64)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        for i in range(v_.shape[1]):
            out[p, i] = b + _binary_search(b_[b:b + n], v_[p, i])
    return torch.from_numpy(out)


def packed_invert_cdf(bins, cdfs, u_vals, pack_infos):
    """kernel_packed_invert_cdf, pack_ops_cuda.cu:1634-1682."""
    b_, c_, u_ = _np(bins), _np(cdfs), _np(u_vals)
    dt = b_.dtype.type
    eps = dt(1.0e-5)
    samples = np.zeros(u_.shape, dtype=b_.dtype)
    bidx = np.full(u_.shape, -1, dtype=np.int64)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        bb, cc = b_[b:b + n], c_[b:b + n]
        for i in range(u_.shape[1]):
            u = u_[p, i]
            pos = _binary_search(cc, u)
            bidx[p, i] = pos + b
            if pos == 0:
                samples[p, i] = b_[b]          # bins[begin]: an empty pack reads the element after it
            else:
                pmf = dt(cc[pos] - cc[pos - 1])
                if pmf < eps:
                    samples[p, i] = bb[pos - 1]
                else:
                    t = dt(dt(u - cc[pos - 1]) / pmf)
                    # b0 + t*(b1-b0) is one fused multiply-add in the compiled reference kernel (checked on the GPU against
                    # oracle/_ref): the fp32 x fp32 product is exact in fp64, so one fp64 add + one rounding reproduces it
                    samples[p, i] = dt(np.float64(t) * np.float64(dt(bb[pos] - bb[pos - 1])) + np.float64(bb[pos - 1]))
    return torch.from_numpy(samples), torch.from_numpy(bidx)


def try_merge_two_packs_sorted_aligned(vals_a, pack_infos_a, vals_b, pack_infos_b, b_sorted=True):
    """kernel_try_merge_two_packs_sorted_aligned + host, pack_ops_cuda.cu:1506-1632.
    Destination index of every element of a and b in the merged, per-pack sorted array; elements of b
    equal to an element of a go *before* it (lower-bound search), ties inside b keep b's order."""
    va, vb = _np(vals_a), _np(vals_b)
    pa, pb = _packs(pack_infos_a), _packs(pack_infos_b)
    assert len(pa) == len(pb)
    n_per = np.array([x[1] + y[1] for x, y in zip(pa, pb)], dtype=np.int64)
    first = np.cumsum(n_per) - n_per
    pidx_a = np.zeros(va.shape[0], dtype=np.int64)
    pidx_b = np.zeros(vb.shape[0], dtype=np.int64)
    for p, ((ab, an), (bb, bn)) in enumerate(zip(pa, pb)):
        a = va[ab:ab + an]
        b = vb[bb:bb + bn]
        cnt = np.zeros(an, dtype=np.int64)
        pos = np.zeros(bn, dtype=np.int64)
        last = 0
        for j in range(bn):
            if b_sorted:
                i = _lower_bound(a[last:], b[j]) + last
                last = i
            else:
                i = _lower_bound(a, b[j])
            pos[j] = i
            if i < an:
                cnt[i] += 1
        ia = np.zeros(an, dtype=np.int64)
        if an > 0:
            ia[0] = cnt[0] + first[p]
            for i in range(1, an):
                ia[i] = cnt[i] + ia[i - 1] + 1
        acc, last_i = 1, -1
        ib = np.zeros(bn, dtype=np.int64)
        for j in range(bn):
            i = pos[j]
            if i == last_i:
                acc += 1
            else:
                acc = 0
            ib[j] = acc + (first[p] if i == 0 else ia[i - 1] + 1)
            last_i = i
        pidx_a[ab:ab + an] = ia
        pidx_b[bb:bb + bn] = ib
    pack_infos = np.stack([first, n_per], 1)
    return torch.from_numpy(pidx_a), torch.from_numpy(pidx_b), torch.from_numpy(pack_infos)


def packed_sort_qsort(vals, pack_infos, return_idx=True):
    """kernel_packed_sort_qsort, pack_ops_cuda.cu:2671-2720: in-place per-pack ascending sort; returns the
    global gather indices.  (quicksort is not stable; ties are returned in a stable order here.)"""
    v = vals.detach().numpy()  # in-place on the caller's buffer, as the reference does
    idx = np.arange(v.shape[0], dtype=np.int64)
    for b, n in _packs(pack_infos):
        o = np.argsort(v[b:b + n], kind="stable")
        idx[b:b + n] = b + o
        v[b:b + n] = v[b:b + n][o]
    return torch.from_numpy(idx) if return_idx else None


# ---------------------------------------------------------------- volume rendering
def packed_alpha_to_vw_forward(alphas, pack_infos, early_stop_eps, alpha_thre, compression):
    """kernel_packed_alpha_to_vw_forward + host, pack_ops_cuda.cu:1736-1904 (nerfacc-derived).
    w_j = alpha_j * T, T *= (1 - alpha_j); stop when T < early_stop_eps; skip alpha <= alpha_thre."""
    a = _np(alphas)
    dt = a.dtype.type
    weights = None if compression else np.zeros_like(a)
    sel = np.zeros(a.shape[0], dtype=bool) if compression else None
    steps = np.zeros(pack_infos.shape[0], dtype=np.int64) if compression else None
    eps, thre, one = dt(early_stop_eps), dt(alpha_thre), dt(1.0)
    for p, (b, n) in enumerate(_packs(pack_infos)):
        T, cnt = one, 0
        for j in range(n):
            if T < eps:
                break
            al = a[b + j]
            if al <= thre:
                continue
            w = dt(al * T)
            T = dt(T * dt(one - al))
            if weights is not None:
                weights[b + j] = w
            if sel is not None:
                sel[b + j] = True
            cnt += 1
        if steps is not None:
            steps[p] = cnt
    if compression:
        cs = np.cumsum(steps)
        info = np.stack([cs - steps, steps], 1)
        return None, torch.from_numpy(info), torch.from_numpy(sel)
    return torch.from_numpy(weights), None, None


def packed_alpha_to_vw_backward(weights, grad_weights, alphas, pack_infos, early_stop_eps, alpha_thre):
    """kernel_packed_alpha_to_vw_backward, pack_ops_cuda.cu:1795-1848 (note: skips alpha < thre, not <=)."""
    w, gw, a = _np(weights), _np(grad_weights), _np(alphas)
    dt = a.dtype.type
    ga = np.zeros_like(a)
    eps, thre, one = dt(early_stop_eps), dt(alpha_thre), dt(1.0)
    for b, n in _packs(pack_infos):
        accum = dt(0)
        for j in range(n):
            accum = dt(accum + dt(gw[b + j] * w[b + j]))
        T = one
        for j in range(n):
            if T < eps:
                break
            al = a[b + j]
            if al < thre:
                continue
            # fmaxf(1 - alpha, 1e-10f): the number when the other operand is NaN (Python's max would return the NaN)
            ga[b + j] = dt(dt(dt(gw[b + j] * T) - accum) / np.fmax(dt(one - al), dt(1e-10)))
            accum = dt(accum - dt(gw[b + j] * w[b + j]))
            T = dt(T * dt(one - al))
    return torch.from_numpy(ga)


class backend:
    """Namespace with the `nr3d_lib.bindings._pack_ops` surface."""


for _name in ("interleave_arange interleave_linstep mark_pack_boundaries_cuda packed_add packed_sub packed_mul "
              "packed_div packed_gt packed_geq packed_lt packed_leq packed_eq packed_neq packed_matmul packed_sum "
              "packed_cumsum packed_cumprod packed_diff packed_backward_diff packed_searchsorted packed_invert_cdf "
              "try_merge_two_packs_sorted_aligned packed_sort_qsort packed_alpha_to_vw_forward "
              "packed_alpha_to_vw_backward").split():
    setattr(backend, _name, staticmethod(globals()[_name]))
