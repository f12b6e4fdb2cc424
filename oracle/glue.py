"""Serial statement of the index-bookkeeping kernels of the per-ray query (csrc/neus_glue.cu).  TEST INFRASTRUCTURE.

numpy only, int64 indices and float32 values, written from the contracts in the comments of csrc/neus_glue.cu and
include/neuralsim_b200.h: which sample lands in which slot, and the fixed fp32 operation sequence of the few values these kernels
compute (interval mid-points, the slab test).  Every result is an index or one such sequence, so callers compare bit for bit.
A count that the kernels would take from device memory is applied by the caller: pass the live part of the inputs, and expect the
outputs past it to keep the `fill` they were allocated with.  tests/test_glue_oracle.py pins this file.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
CANONICAL_NAN = np.uint32(0x7FC00000)


def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


# ---------------------------------------------------------------- scan + compaction of the non-zero entries
def scan_counts(counts, src=None):
    """counts[n] (int32, >= 0) -> dict(first[n] int32, info2[n,2] int32, nz_index[m] int64, nz_pack[m,2] int64, nz_src[m] | None,
    totals=(sum, m)).  Sums are carried in int64; `first` / `info2` are the int32 the kernel stores (valid while the sum < 2^31)."""
    c = np.asarray(counts, dtype=np.int32).astype(np.int64)
    incl = np.add.accumulate(c, dtype=np.int64) if c.size else np.zeros(0, np.int64)
    excl = incl - c
    nz = np.flatnonzero(c > 0).astype(np.int64)
    return dict(first=excl.astype(np.int32), info2=np.stack([excl, c], 1).astype(np.int32), nz_index=nz,
                nz_pack=np.stack([excl[nz], c[nz]], 1), nz_src=None if src is None else np.asarray(src, np.int64)[nz],
                totals=(int(incl[-1]) if c.size else 0, int(nz.size)))


# ---------------------------------------------------------------- merge of two sorted packs with payloads
def merge_vals(dep_a, sdf_a, pi_a, dep_b, sdf_b, n_out=None, fill=np.nan):
    """Pack p of a = (dep_a, sdf_a)[pi_a[p]], sorted; pack p of b = row p of (dep_b, sdf_b)[P, nb], sorted.  In the merged pack a_i sits at
    i + #{b <= a_i} and b_j at j + #{a < b_j} (a b equal to an a goes before it); pi_m[p] = (first_a + p nb, n_a + nb).
    -> dep_m, sdf_m | None, pi_m; slots no pack owns keep `fill`."""
    dep_a, dep_b = _f32(dep_a), _f32(dep_b)
    pi_a = np.asarray(pi_a, np.int64).reshape(-1, 2)
    P, nb = dep_b.shape
    pi_m = np.stack([pi_a[:, 0] + np.arange(P, dtype=np.int64) * nb, pi_a[:, 1] + nb], 1)
    n_out = int(dep_a.size + P * nb) if n_out is None else n_out
    dep_m = np.full(n_out, fill, np.float32)
    sdf_m = None if sdf_a is None else np.full(n_out, fill, np.float32)
    for p in range(P):
        a0, na = pi_a[p]
        m0 = pi_m[p, 0]
        a, b = dep_a[a0:a0 + na], dep_b[p]
        pos_a = m0 + np.arange(na) + np.searchsorted(b, a, side="right")      # #{b <= a_i}
        pos_b = m0 + np.arange(nb) + np.searchsorted(a, b, side="left")       # #{a < b_j}
        dep_m[pos_a], dep_m[pos_b] = a, b
        if sdf_m is not None:
            sdf_m[pos_a], sdf_m[pos_b] = _f32(sdf_a)[a0:a0 + na], _f32(sdf_b)[p]
    return dep_m, sdf_m, pi_m


# ---------------------------------------------------------------- boundary samples
def interval_mid(d, pack_len):
    """d[..., n] sorted rows of which the first pack_len are live: mid_k = fl(d_k + fl(fl(d_{k+1} - d_k) * 0.5)); the last sample + 0
    (so a last sample of -0.0 becomes +0.0).  Three separately rounded fp32 operations, no fused multiply-add."""
    d = _f32(d)
    nxt = np.concatenate([d[..., 1:], d[..., -1:]], -1)
    with np.errstate(invalid="ignore", over="ignore"):
        diff = (nxt - d).astype(np.float32)
        diff[..., pack_len - 1] = F32(0)
        return (d + (diff * F32(0.5)).astype(np.float32)).astype(np.float32)


def stable_rank(rows):
    """rank of every element of rows[H, n] in the stable sort of its row: #{smaller values} + #{equal values before it}.  +0.0 and
    -0.0 compare equal, so their order is the concatenation order.  Counted pair by pair: no use of the rows' run structure."""
    rows = _f32(rows)
    H, n = rows.shape
    rank = np.empty((H, n), np.int64)
    before = np.tril(np.ones((n, n), bool), -1)                               # [e, e']: e' < e
    step = max(1, (1 << 25) // max(n * n, 1))
    for h in range(0, H, step):
        v = rows[h:h + step]
        less = v[:, None, :] < v[:, :, None]                                  # [row, e, e']: v[e'] < v[e]
        tie = (v[:, None, :] == v[:, :, None]) & before
        rank[h:h + step] = (less | tie).sum(-1)
    return rank


def assemble_boundary(coarse, ridx_hit, fine, run_len=None, n_rays=None, n_hit=None, rays=None):
    """coarse[R, nc] sorted rows; ray ridx_hit[j] (ascending, unique) also carries fine[j, nf], a concatenation of sorted runs.
    Pack r = the stable merge of (coarse row, run 0, run 1, ...), i.e. the stable sort by value of that concatenation;
    first_r = nc r + nf #{listed rays < r}.  -> dict(d1, mid, ridx_all [S], pack_infos [R, 2]).  `run_len` only has to add up to nf:
    a stable sort does not need to know where the runs start.  n_rays / n_hit: the live counts.  rays: evaluate only these rays
    (d1 / mid elsewhere are NaN, ridx_all -1; pack_infos are always complete)."""
    coarse = _f32(coarse)
    R = coarse.shape[0] if n_rays is None else int(n_rays)
    nc = coarse.shape[1]
    coarse = coarse[:R]
    hit = np.zeros(0, np.int64) if ridx_hit is None else np.asarray(ridx_hit, np.int64)
    hit = hit[:hit.size if n_hit is None else int(n_hit)]
    nf = 0 if fine is None or hit.size == 0 else np.asarray(fine).shape[1]
    assert run_len is None or hit.size == 0 or int(np.sum(run_len)) == nf
    assert np.all(np.diff(hit) > 0) and (hit.size == 0 or (hit[0] >= 0))
    hit = hit[hit < R]                                                        # a listed ray past the live rays is never visited
    is_hit = np.zeros(R, bool)
    is_hit[hit] = True
    before = np.cumsum(is_hit) - is_hit                                       # listed rays < r
    n = nc + nf * is_hit
    first = nc * np.arange(R, dtype=np.int64) + nf * before
    S = int(n.sum())
    d1, mid, ridx_all = np.full(S, np.nan, np.float32), np.full(S, np.nan, np.float32), np.full(S, -1, np.int64)
    todo = np.ones(R, bool)
    if rays is not None:
        todo[:] = False
        todo[np.asarray(rays, np.int64)] = True
    miss = np.flatnonzero(~is_hit & todo)
    at = first[miss][:, None] + np.arange(nc)
    d1[at], mid[at], ridx_all[at] = coarse[miss], interval_mid(coarse[miss], nc), miss[:, None]
    sel = np.flatnonzero(todo[hit])
    if sel.size:
        rows = np.concatenate([coarse[hit[sel]], _f32(fine)[sel]], 1)
        srt = np.empty_like(rows)
        np.put_along_axis(srt, stable_rank(rows), rows, 1)
        at = first[hit[sel]][:, None] + np.arange(nc + nf)
        d1[at], mid[at], ridx_all[at] = srt, interval_mid(srt, nc + nf), hit[sel][:, None]
    return dict(d1=d1, mid=mid, ridx_all=ridx_all, pack_infos=np.stack([first, n], 1).astype(np.int64))


# ---------------------------------------------------------------- compaction of the kept samples
def compact_samples(selector, pi, first_out, kept, alpha, *, ridx_all=None, t=None, d1=None, n_out=None):
    """selector[S] (any non-zero byte keeps the sample), kept[p] = kept samples of pack p, first_out = their exclusive scan.
    Kept sample s of pack p -> slot first_out[p] + #{kept samples of p before s}.  ridx_all None: the ray is the pack.  t None: the
    depth is the interval mid-point of the pack in d1.  -> dict(pidx, ridx_c int64, t_c, alpha_c float32); unowned slots: -1 / NaN."""
    pi = np.asarray(pi, np.int64).reshape(-1, 2)
    P = pi.shape[0]
    selector, kept, first_out = np.asarray(selector), np.asarray(kept, np.int64), np.asarray(first_out, np.int64)
    n_out = int(kept.sum()) if n_out is None else n_out
    out = dict(pidx=np.full(n_out, -1, np.int64), ridx_c=np.full(n_out, -1, np.int64), t_c=np.full(n_out, np.nan, np.float32),
               alpha_c=np.full(n_out, np.nan, np.float32))
    for p in range(P):
        if kept[p] == 0:
            continue
        b, n = pi[p]
        k = np.flatnonzero(selector[b:b + n] != 0)
        assert k.size == kept[p], "kept[p] must be the number of selected samples of pack p"
        o = first_out[p] + np.arange(k.size)
        out["pidx"][o] = b + k
        out["ridx_c"][o] = p if ridx_all is None else np.asarray(ridx_all, np.int64)[b + k]
        out["t_c"][o] = _f32(t)[b + k] if t is not None else interval_mid(_f32(d1)[b:b + n], n)[k]
        out["alpha_c"][o] = _f32(alpha)[b + k]
    return out


def scatter_f32(src, idx, n_dst):
    dst = np.zeros(n_dst, np.float32)
    dst[np.asarray(idx, np.int64)] = _f32(src)
    return dst


def gather_rays(idx, *arrays):
    return tuple(np.asarray(a)[np.asarray(idx, np.int64)] for a in arrays)


def flag_nonzero(v, n_live=None):
    v = _f32(v)
    live = np.arange(v.size) < (v.size if n_live is None else n_live)
    return (live & (v != 0)).astype(np.int32)                                  # -0.0 -> 0; NaN, inf and denormals -> 1


# ---------------------------------------------------------------- AABB ray test
def _nan_or(a, b, r):
    return np.where(np.isnan(a) | np.isnan(b), CANONICAL_NAN, r.view(np.uint32)).astype(np.uint32).view(np.float32)


def max_nan(a, b):
    """NaN if either is NaN, else the larger; +0.0 is larger than -0.0 (the hardware's max)."""
    a, b = _f32(a), _f32(b)
    tie = (a.view(np.uint32) & b.view(np.uint32)).view(np.float32)            # equal values: the same bits, or +0 unless both are -0
    return _nan_or(a, b, np.where(a == b, tie, np.where(a > b, a, b)).astype(np.float32))


def min_nan(a, b):
    a, b = _f32(a), _f32(b)
    tie = (a.view(np.uint32) | b.view(np.uint32)).view(np.float32)
    return _nan_or(a, b, np.where(a == b, tie, np.where(a < b, a, b)).astype(np.float32))


def _fma(x, y, z):
    """one fused multiply-add in fp32: the product of two fp32 is exact in float64"""
    return (x.astype(np.float64) * y.astype(np.float64) + z.astype(np.float64)).astype(np.float32)


def ray_test_aabb(o, d, center, radius, near=None, far=None):
    """The kernel's fp32 sequence per ray and axis: o' = (o - c) / r, d' = d / r, ta = (-1 - o') / d', tb = (1 - o') / d',
    tn = max over axes of min(ta, tb), tf = min over axes of max(ta, tb), min / max propagating NaN; near / far clamp tn / tf
    unless they are NaN; flag = tf > tn and tf > (near or 0) and (no far or tn < far).
    -> dict(o_n, d_n [n,3], near, far [n], flag int32 [n], coherent_pairs, row_len)."""
    o, d = _f32(o).reshape(-1, 3), _f32(d).reshape(-1, 3)
    c, r = _f32(center), _f32(radius)
    n = o.shape[0]
    with np.errstate(all="ignore"):
        o_n = ((o - c).astype(np.float32) / r).astype(np.float32)
        d_n = (d / r).astype(np.float32)
        ta = ((F32(-1) - o_n).astype(np.float32) / d_n).astype(np.float32)
        tb = ((F32(1) - o_n).astype(np.float32) / d_n).astype(np.float32)
        lo, hi = min_nan(ta, tb), max_nan(ta, tb)
        tn, tf = lo[:, 0], hi[:, 0]
        for k in (1, 2):
            tn, tf = max_nan(tn, lo[:, k]), min_nan(tf, hi[:, k])
        if near is not None:
            tn = np.where(np.isnan(tn), tn, np.maximum(tn, F32(near))).astype(np.float32)
        if far is not None:
            tf = np.where(np.isnan(tf), tf, np.minimum(tf, F32(far))).astype(np.float32)
        m = (tf > tn) & (tf > F32(0.0 if near is None else near))
        if far is not None:
            m &= tn < F32(far)
        # ray i next to ray i - 1: direction within 3 % of its largest component, origin within 3 % of the box radius
        pairs = 0
        if n > 1:
            dd = np.fmax(F32(0), np.fmax.reduce(np.abs((d[1:] - d[:-1]).astype(np.float32)), -1))      # fmax skips NaN
            od = np.fmax(F32(0), np.fmax.reduce((np.abs((o[1:] - o[:-1]).astype(np.float32)) / r).astype(np.float32), -1))
            ln = np.fmax.reduce(np.abs(d[1:]), -1)
            pairs = int(((dd <= (F32(0.03) * ln).astype(np.float32)) & (od <= F32(0.03))).sum())
        # image row length: the first i >= 2 whose direction step points against the first step (a chain of three fused multiply-adds)
        row_len = -1
        if n > 2:
            step, ref = (d[2:] - d[1:-1]).astype(np.float32), (d[1] - d[0]).astype(np.float32)
            rev = np.zeros(n - 2, np.float32)
            for k in range(3):
                rev = _fma(step[:, k], np.broadcast_to(ref[k], step[:, k].shape), rev)
            back = np.flatnonzero(rev < 0)
            row_len = int(back[0]) + 2 if back.size else -1
    return dict(o_n=o_n, d_n=d_n, near=tn, far=tf, flag=m.astype(np.int32), coherent_pairs=pairs, row_len=row_len)


# ---------------------------------------------------------------- derived sizes of one query
def query_counts(c, phase, nc, n_fine, march_cap, kept_cap):
    """The 32-slot block of include/neuralsim_b200.h after nsb_query_counts; every slot the phase does not own is returned unchanged."""
    c = np.array(c, dtype=np.int64)
    if phase == 0:
        M, nh = int(c[3]), int(c[4])
        worst = M + sum(nh * f for f in n_fine[:-1])                           # the last stage's samples are never merged
        if worst > march_cap:
            c[20] |= 1
            M = nh = 0
        c[12], c[13] = M, nh
        merged = M
        for q in range(4):
            c[14 + q] = nh * n_fine[q] if q < len(n_fine) else 0
            if q + 1 < len(n_fine):
                merged += nh * n_fine[q]
            c[22 + q] = merged
        c[18] = c[0] * nc + nh * sum(n_fine)
    else:
        fits = c[6] <= kept_cap
        if not fits:
            c[20] |= 2
        c[19], c[21], c[26] = (c[6], c[7], c[0]) if fits else (0, 0, 0)
    return c
