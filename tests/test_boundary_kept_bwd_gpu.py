"""The kept-interval alpha backward of the graph step (csrc/neus_fused.cu: k_neus_alpha_bwd_kept / _list) against the boundary-wide chain
it replaces: scatter of the kept cotangents into zeros -> k_neus_alpha_bwd -> k_flag_nonzero -> scan.  The index list must be equal
element for element, d_sdf bit-equal at every listed index, the ray of every listed index its pack, d_inv_s equal up to summation order.
Plus k_compact_samples deriving the kept samples' depth and ray from d1 and the pack: bit-equal to the gather of k_assemble_boundary's
mid / ridx_all."""
import ctypes

import numpy as np
import pytest
import torch

from neuralsim_b200 import _lib as L
from neuralsim_b200.graphics import neus_fused as NF
from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _call, _scan

pytestmark = pytest.mark.gpu

INV_S_REL = 1.5e-5      # tests/test_neus_stages64_gpu.py: d_inv_s over the sum of |terms|
INV_S = 64.0


def _ws():
    return torch.zeros(NF._scan_ws_bytes(), dtype=torch.uint8, device="cuda")


def _run(lens, kept, sdf, g, cap_extra=0):
    """lens[p]: pack lengths; kept[p]: ascending kept sample indices of pack p; sdf [S]; g: cotangent of every kept sample (kept order).
    -> (old list, old d_sdf, old d_inv, new list, new d_sdf, new ray, new d_inv, pack of every sample)"""
    lib, P = L.lib(), L.ptr
    Pn = len(lens)
    first = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64) if Pn else np.zeros(0, np.int64)
    S = int(sum(lens))
    pinfo = torch.tensor(np.stack([first, np.asarray(lens, np.int64)], 1).reshape(-1, 2), device="cuda")
    rows = [p for p in range(Pn) if len(kept[p])]
    pidx = torch.tensor([first[p] + k for p in rows for k in kept[p]], dtype=torch.int64, device="cuda")
    K = pidx.numel()
    kcnt = np.asarray([len(kept[p]) for p in rows], np.int64)
    kfirst = np.concatenate([[0], np.cumsum(kcnt)[:-1]]).astype(np.int64) if rows else np.zeros(0, np.int64)
    cap = len(rows) + cap_extra
    nidx = torch.full((cap,), -1, dtype=torch.int64, device="cuda")
    pk = torch.full((cap, 2), -1, dtype=torch.int64, device="cuda")
    if rows:
        nidx[:len(rows)] = torch.tensor(rows, device="cuda")
        pk[:len(rows)] = torch.tensor(np.stack([kfirst, kcnt], 1), device="cuda")
    sdf = torch.as_tensor(sdf, dtype=torch.float32, device="cuda")
    g = torch.as_tensor(g, dtype=torch.float32, device="cuda")
    inv = torch.tensor([INV_S], device="cuda")
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[CNT_SLOTS["n_rays"]] = Pn
    cnt[CNT_SLOTS["boundary"]] = S
    cnt[CNT_SLOTS["kept_rays"]] = len(rows)
    Sa = max(S, 1)
    # the boundary-wide chain
    d_full = torch.zeros(Sa, device="cuda")
    d_full[pidx] = g
    d_old = torch.empty(Sa, device="cuda")
    inv_old = torch.zeros(1, device="cuda")
    if Pn:
        _call(lib.nsb_neus_alpha_backward, "alpha_bwd", cnt, CNT_SLOTS["n_rays"], None, P(sdf), P(pinfo), L.c_i64(Pn), P(inv), P(d_full), P(d_old),
              P(inv_old), L.stream_ptr())
    flag = torch.empty(Sa, dtype=torch.int32, device="cuda")
    _call(lib.nsb_flag_nonzero, "flag", cnt, CNT_SLOTS["boundary"], None, P(d_old), L.c_i64(Sa), P(flag), L.stream_ptr())
    keep_old = torch.empty(Sa, dtype=torch.int64, device="cuda")
    _scan(flag, cnt, CNT_SLOTS["nonzero"], index=keep_old, ws=_ws())
    n_old = int(cnt[CNT_SLOTS["nonzero"]])
    # the kept-interval chain (sentinels where nothing may be read)
    d_new = torch.full((Sa,), float("nan"), device="cuda")
    ray = torch.full((Sa,), -7, dtype=torch.int64, device="cuda")
    counts = torch.full((max(cap, 1),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    inv_new = torch.zeros(1, device="cuda")
    gk = g if K else torch.zeros(1, device="cuda")
    pidx_a = pidx if K else torch.zeros(1, dtype=torch.int64, device="cuda")
    a = (P(pinfo if Pn else torch.zeros(1, 2, dtype=torch.int64, device="cuda")), P(nidx if cap else ray), P(pk if cap else ray), P(pidx_a))
    if cap:
        _call(lib.nsb_neus_alpha_backward_kept, "kept_bwd", cnt, CNT_SLOTS["kept_rays"], None, P(sdf if S else d_new), *a, L.c_i64(cap), P(inv), P(gk),
              P(d_new), P(counts), P(inv_new), L.stream_ptr())
        assert bool((counts[len(rows):cap] == 0).all())
    offs = torch.empty(max(cap, 1), dtype=torch.int32, device="cuda")
    cnt[CNT_SLOTS["nonzero"]] = -1
    _scan(counts[:cap], cnt, CNT_SLOTS["nonzero"], first=offs, ws=_ws())
    n_new = int(cnt[CNT_SLOTS["nonzero"]])
    lst = torch.full((max(min(S, 2 * K), 1),), -9, dtype=torch.int64, device="cuda")
    if cap:
        _call(lib.nsb_neus_alpha_backward_kept_list, "kept_list", cnt, CNT_SLOTS["kept_rays"], None, *a, P(gk), P(d_new), P(offs), L.c_i64(cap), P(lst),
              P(ray), L.stream_ptr())
    torch.cuda.synchronize()
    pack_of = torch.repeat_interleave(torch.arange(Pn, device="cuda"), torch.as_tensor(lens, device="cuda")) if S else ray[:0]
    return dict(old=keep_old[:n_old], d_old=d_old, inv_old=inv_old, new=lst[:n_new], d_new=d_new, ray=ray, inv_new=inv_new, pack_of=pack_of,
                sdf=sdf)


def _check(r):
    assert torch.equal(r["new"], r["old"]), (r["new"][:20], r["old"][:20])
    i = r["new"]
    assert torch.equal(r["d_new"][i].view(torch.int32), r["d_old"][i].view(torch.int32))
    assert torch.equal(r["ray"][i], r["pack_of"][i])
    terms = (r["d_old"][r["old"]].double() * r["sdf"][r["old"]].double() / INV_S).abs().sum()
    assert abs(float(r["inv_new"]) - float(r["inv_old"])) <= INV_S_REL * float(terms) + 1e-30


def _ramp(lens, rng, rising=()):
    """sdf falling through 0 along every pack (alpha > 0); packs in `rising` rise (the clamp of the backward is active)"""
    out = []
    for p, n in enumerate(lens):
        t = np.sort(rng.random(n)).astype(np.float32)
        s = (0.6 - t) * (1.0 + rng.random()) + 0.01 * rng.standard_normal(n)
        out.append(-s if p in rising else s)
    return np.concatenate(out).astype(np.float32) if out else np.zeros(0, np.float32)


def test_edges():
    rng = np.random.default_rng(0)
    cases = {
        "length 1 and 2": ([1, 2, 2, 1], [[0], [0], [0, 1], []]),
        "nothing kept": ([5, 7], [[], []]),
        "everything kept": ([5, 40, 33], [list(range(5)), list(range(40)), list(range(33))]),
        "early stop at the first sample": ([9, 70], [[0], [0]]),
        "last interval kept": ([9, 70], [[7, 8], [68, 69]]),
        "kept intervals separated by alpha = 0": ([64, 100], [[0, 1, 2, 5, 6, 31, 32, 63], [0, 1, 30, 31, 33, 34, 64, 65, 96, 99]]),
        "only the last sample kept": ([9], [[8]]),
    }
    for lens, kept in cases.values():
        sdf = _ramp(lens, rng)
        g = rng.standard_normal(sum(len(k) for k in kept)).astype(np.float32)
        _check(_run(lens, kept, sdf, g))


def test_clamp_zero_cotangent_and_capacity():
    rng = np.random.default_rng(1)
    lens = [40, 40, 50]
    kept = [list(range(0, 20)), list(range(5, 35)), [0, 1, 2, 3, 10, 11, 12]]
    sdf = _ramp(lens, rng, rising=(1,))                          # pack 1: rising sdf, raw alpha < 0 -> the clamp zeroes its terms
    g = rng.standard_normal(sum(map(len, kept))).astype(np.float32)
    g[3] = 0.0                                                   # a kept interval with an exactly-zero cotangent
    g[4] = -0.0
    g[-7:-4] = 0.0
    r = _run(lens, kept, sdf, g, cap_extra=5)                    # capacity above the live count
    _check(r)


def test_frame_scale():
    """about the bench's boundary packs: 65 or 116 samples per ray, a kept prefix up to the early stop, many rays per warp"""
    rng = np.random.default_rng(2)
    n_rays = 20000
    lens = list(np.where(rng.random(n_rays) < 0.5, 116, 65))
    kept = []
    for n in lens:
        r = rng.random()
        if r < 0.3:
            kept.append([])
        elif r < 0.9:
            kept.append(list(range(int(rng.integers(1, n + 1)))))
        else:
            kept.append(sorted(rng.choice(n, int(rng.integers(1, n)), replace=False).tolist()))
    sdf = _ramp(lens, rng, rising=set(range(0, n_rays, 17)))
    g = rng.standard_normal(sum(map(len, kept))).astype(np.float32)
    g[rng.random(g.size) < 0.05] = 0.0
    _check(_run(lens, kept, sdf, g, cap_extra=1000))


def test_compact_from_d1_equals_gather_of_mid():
    g = torch.Generator().manual_seed(3)
    R, nc = 701, 65
    near = torch.rand(R, generator=g) + 0.5
    coarse = (near[:, None] + torch.linspace(0, 1, nc)[None, :] * (1 + torch.rand(R, 1, generator=g))).cuda().contiguous()
    ridx_hit = torch.randperm(R, generator=g)[:260].sort().values.cuda()
    fine = (coarse[ridx_hit, :1] + torch.rand(260, 51, generator=g).sort(-1).values.cuda() * 1.5).contiguous()
    d1, mid, ridx_all, pi = NF.assemble_boundary(coarse, ridx_hit, fine)
    S = d1.numel()
    sel = (torch.rand(S, generator=g) < 0.3).cuda()
    sel[pi[5, 0]:pi[5, 0] + pi[5, 1]] = True                    # a pack kept whole, its last sample included
    steps = torch.zeros(R, dtype=torch.int32, device="cuda")
    for p, (b, n) in enumerate(pi.tolist()):
        steps[p] = int(sel[b:b + n].sum())
    first = (torch.cumsum(steps, 0) - steps).int()
    K = int(steps.sum())
    alpha = torch.rand(S, device="cuda")
    out = []
    for with_mid in (True, False):
        pidx, rk = torch.empty(K, dtype=torch.int64, device="cuda"), torch.empty(K, dtype=torch.int64, device="cuda")
        tk, ak = torch.empty(K, device="cuda"), torch.empty(K, device="cuda")
        P = L.ptr
        L.check(L.lib().nsb_compact_samples(P(sel.view(torch.uint8), "u8"), P(pi), P(first), P(steps), L.c_i64(R),
                                            P(ridx_all) if with_mid else None, P(mid) if with_mid else None, P(d1), P(alpha), P(pidx), P(rk), P(tk),
                                            P(ak), L.stream_ptr()), "compact")
        out.append((pidx, rk, tk, ak))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][3], out[1][3])
    assert torch.equal(out[0][2].view(torch.int32), out[1][2].view(torch.int32))
    # and k_assemble_boundary without mid / ridx_all writes the same d1
    d1b = torch.empty_like(d1)
    pib = torch.empty_like(pi)
    L.check(L.lib().nsb_assemble_boundary(L.ptr(coarse), L.c_i64(R), L.c_i32(nc), L.ptr(ridx_hit), L.c_i64(260), L.ptr(fine), L.c_i32(51),
                                          (ctypes.c_int32 * 1)(51), L.c_i32(1), L.ptr(d1b), None, None, L.ptr(pib), L.stream_ptr()), "assemble")
    assert torch.equal(d1b, d1) and torch.equal(pib, pi)
