"""The `_pack_ops` kernels (csrc/pack_ops.cu) at their edges: NaN, +-inf, -0.0 against +0.0, ties, values equal to cdf entries,
pmf at the 1e-5 threshold, empty packs in the middle and at the end, pack lengths around the 32-element chunk and the lane loops,
the early stop of the transmittance replay on every lane position, gapped sort layouts, and one 800x600-frame case whose grid-stride
loops run at least 3 trips (sized from the SM count).  Checked against the serial CPU oracle (oracle/pack_ops.py) and against the
reference's own kernels, whose outputs are kept in tests/golden/ref__pack_ops_edges.npz (recorded with NSB_RECORD_REF, refgold.py).
Inputs the reference kernels would read or write out of bounds with (an empty qsort pack, an empty last search pack, an empty `a`
pack of the merge, empty packs of sum/cumsum/diff) are compared against the oracle only."""
import numpy as np
import pytest
import torch

from oracle import pack_ops as opk
from refgold import Golden
from test_pack_ops_edges import _layout, merge_edge_packs

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
LENS = [0, 1, 2, 31, 32, 33, 64, 65, 1024, 4097]
FRAME = 800 * 600


@pytest.fixture(autouse=True)
def _device(cuda):
    return cuda


@pytest.fixture(scope="module")
def G():
    g = Golden("_pack_ops_edges", module="_pack_ops")
    yield g
    g.save()


def B():
    from neuralsim_b200.bindings import _pack_ops
    return _pack_ops


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def wave_grid(work_items, block, ctas_per_sm=8):
    """csrc/nsb_common.cuh: whole waves of resident CTAs, at most 8 of them; grid-stride loops cover the rest"""
    need, wave = -(-work_items // block), sms() * ctas_per_sm
    return max(need, 1) if need <= wave else min(-(-need // wave), 8) * wave


def warp_trips(n_packs):
    """grid-stride trips of a warp-per-pack kernel (warp_grid: 256 threads per CTA)"""
    return -(-n_packs // (wave_grid(n_packs * 32, 256) * 8))


def thread_trips(n):
    return -(-n // (wave_grid(n, 256) * 256))


def bits(t):
    a = np.ascontiguousarray(t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def same(got, ref, what="", any_nan=False):
    """bit-equality; any_nan: NaN matches NaN whatever its payload (arithmetic on a NaN or inf - inf, whose payload is the
    processor's choice)"""
    g = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    r = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else np.asarray(ref)
    assert g.shape == r.shape and g.dtype == r.dtype, (what, g.shape, r.shape, g.dtype, r.dtype)
    if any_nan and g.dtype == np.float32:
        assert np.array_equal(np.isnan(g), np.isnan(r)), (what, np.flatnonzero(np.isnan(g) != np.isnan(r))[:8])
        k = ~np.isnan(g)
        g, r = g[k], r[k]
    bad = np.flatnonzero(bits(g).reshape(-1) != bits(r).reshape(-1))
    assert bad.size == 0, (what, bad[:8], g.reshape(-1)[bad[:4]], r.reshape(-1)[bad[:4]])


def nan_tailed(t, extra=64):
    """t on the device at the start of an allocation whose next `extra` elements are NaN: a read one past t is defined"""
    buf = torch.full((t.numel() + extra,), NAN, dtype=t.dtype, device="cuda")
    buf[:t.numel()].copy_(t.reshape(-1))
    return buf[:t.numel()]


def pack_ids(pi):
    return torch.repeat_interleave(torch.arange(pi.shape[0]), pi[:, 1])


# ------------------------------------------------------------------------------------------------ search / inverse cdf
E = np.float32(1e-5)
E_LO = np.nextafter(E, np.float32(0))


def search_inputs(lens, seed, n_vals=24):
    """per pack: an exclusive-cdf-like ascending pack with flat runs, one of several edge kinds; search values that hit cdf entries
    exactly, u = 0 / 1 / below / above, -0.0, +-inf, NaN"""
    rng = np.random.default_rng(seed)
    cdfs, bins, us = [], [], []
    for p, n in enumerate(lens):
        kind = p % 5
        c = np.sort(rng.integers(0, 8, n) / 8.0).astype(np.float32)          # runs of equal entries (flat cdf)
        if n:
            c[0] = 0.0
        if kind == 1 and n >= 2:
            c[:n // 2] = np.where(c[:n // 2] == 0, np.float32(-0.0), c[:n // 2])    # -0.0 entries against +0.0 searches
        elif kind == 2 and n >= 3:
            c[0], c[-1] = -INF, INF
        elif kind == 3 and n >= 3:
            c[-min(3, n - 1):] = NAN                                             # NaN at the tail of the cdf
        elif kind == 4 and n >= 4:
            c[:3] = [0, E if (p // 5) % 2 == 0 else E_LO, 2 * E]                 # pmf c[1] - c[0]: exactly 1e-5f, or one ulp below it
            c[3:] = np.maximum(c[3:], 2 * E)
        cdfs.append(c)
        bins.append(np.cumsum(rng.random(n) + 0.01).astype(np.float32))
        u = np.array([0, 1, -1, 2, -0.0, 0.0, INF, -INF, NAN, E, E / 2, 3 * E] + [0.5] * (n_vals - 12), np.float32)
        if n:
            u[12:] = c[rng.integers(0, n, n_vals - 12)]                          # exact ties with cdf entries
            u[12:15] = (c[rng.integers(0, n, 3)] + np.float32(1 / 16)).astype(np.float32)
        us.append(u)
    return (torch.from_numpy(np.concatenate(bins)), torch.from_numpy(np.concatenate(cdfs)), torch.from_numpy(np.stack(us)),
            _layout(lens))


def _check_search(bins_d, cdfs_d, u, pi, bins_np, cdfs_np, what):
    bins_c, cdfs_c = torch.from_numpy(bins_np), torch.from_numpy(cdfs_np)
    s, i = B().packed_invert_cdf(bins_d, cdfs_d, u.cuda(), pi.cuda())
    s_r, i_r = opk.packed_invert_cdf(bins_c, cdfs_c, u, pi)
    same(i, i_r, f"{what} bin_idx")
    same(s, s_r, f"{what} samples", any_nan=True)
    ss = B().packed_searchsorted(cdfs_d, u.cuda(), pi.cuda())
    same(ss, opk.packed_searchsorted(cdfs_c, u, pi), f"{what} searchsorted")
    return s, i, ss


def test_search_invert_cdf_edges(G):
    lens = [1, 2, 0, 31, 32, 33, 0, 64, 65, 1024, 4097, 6, 7, 8, 9, 10]     # empty packs in the middle, kinds on every length
    bins, cdfs, u, pi = search_inputs(lens, 11)
    bd, cd = bins.cuda(), cdfs.cuda()
    s, i, ss = _check_search(bd, cd, u, pi, bins.numpy(), cdfs.numpy(), "middle-empty")
    uc, pic = u.cuda(), pi.cuda()
    G.equal("search.samples", s, lambda ref: ref.packed_invert_cdf(bd, cd, uc, pic)[0])
    G.equal("search.bin_idx", i, lambda ref: ref.packed_invert_cdf(bd, cd, uc, pic)[1])
    G.equal("search.searchsorted", ss, lambda ref: ref.packed_searchsorted(cd, uc, pic))
    # an empty last pack reads bins[begin], one past the data: a NaN-tailed allocation pins it (oracle only)
    lens2 = lens + [0]
    bins2, cdfs2, u2, pi2 = search_inputs(lens2, 12)
    bd2, cd2 = nan_tailed(bins2), nan_tailed(cdfs2)
    tail = np.full(1, NAN, np.float32)
    s2, i2, _ = _check_search(bd2, cd2, u2, pi2, np.concatenate([bins2.numpy(), tail]), np.concatenate([cdfs2.numpy(), tail]), "last-empty")
    assert torch.isnan(s2[-1]).all() and (i2[-1] == int(pi2[-1, 0])).all()


# ------------------------------------------------------------------------------------------------ merge
def _merge_property(ga, gb, gp, va, vb):
    tot = va.shape[0] + vb.shape[0]
    both = torch.cat([ga.cpu(), gb.cpu()])
    assert torch.equal(both.sort().values, torch.arange(tot))              # a permutation of the merged packs
    merged = torch.empty(tot)
    merged[ga.cpu()], merged[gb.cpu()] = va, vb
    for b, n in gp.cpu().tolist():
        seg = merged[b:b + n]
        num = seg[~torch.isnan(seg)]
        assert torch.all(num[1:] >= num[:-1])                              # the numbers of every pack ascend
    return merged


@pytest.mark.parametrize("b_nan", [False, True])
def test_merge_sorted_aligned_edges(G, b_nan):
    va, pia, vb, pib = merge_edge_packs(7 + b_nan, b_nan)
    ra, rb, rp = opk.try_merge_two_packs_sorted_aligned(va, pia, vb, pib, True)
    vac, piac, vbc, pibc = va.cuda(), pia.cuda(), vb.cuda(), pib.cuda()
    ga, gb, gp = B().try_merge_two_packs_sorted_aligned(vac, piac, vbc, pibc, True)
    same(ga, ra, "pidx_a"), same(gb, rb, "pidx_b"), same(gp, rp, "pack_infos")
    merged = _merge_property(ga, gb, gp, va, vb)
    if not b_nan:                                                           # NaN only in a (last): every pack sorts, NaN last
        for b, n in gp.cpu().tolist():
            seg = merged[b:b + n]
            k = int((~torch.isnan(seg)).sum())
            assert torch.isnan(seg[k:]).all()
    # the reference's kernel writes pidx_a[begin] of an empty a pack (another pack's slot): its goldens use packs with a non-empty a
    keep = pia[:, 1] > 0
    pa2, pb2 = _layout(pia[keep, 1]), _layout(pib[keep, 1])
    va2 = torch.cat([va[b:b + n] for b, n in pia[keep].tolist()])
    vb2 = torch.cat([vb[b:b + n] for b, n in pib[keep].tolist()])
    va2c, pa2c, vb2c, pb2c = va2.cuda(), pa2.cuda(), vb2.cuda(), pb2.cuda()
    out = B().try_merge_two_packs_sorted_aligned(va2c, pa2c, vb2c, pb2c, True)
    for k, y in enumerate(out):
        G.equal(f"merge_sorted{int(b_nan)}.{k}", y, lambda ref: ref.try_merge_two_packs_sorted_aligned(va2c, pa2c, vb2c, pb2c, True)[k])


# ------------------------------------------------------------------------------------------------ alpha_to_vw
def alpha_inputs(seed):
    """hand-built packs: alpha == thre, -0.0, 1, > 1, NaN, +-inf, denormals; 0.5-halvings that bring T to exactly 2^-10 and below it
    with the crossing on lanes 0, 30, 31 of a chunk and on the last sample of a partial chunk; plus random packs of LENS"""
    rng = np.random.default_rng(seed)
    packs = []
    for c in (10, 31, 32, 33, 40, 63, 64, 65):                              # T drops below 2^-10 after sample c (the 11th half)
        a = np.zeros(96, np.float32)
        a[c - 10:c + 1] = 0.5
        packs.append(a)
    a = np.zeros(45, np.float32); a[34:] = 0.5; packs.append(a)             # crossing on the last sample of a partial chunk
    a = np.zeros(45, np.float32); a[20:30] = 0.5; a[30] = 0.01; a[31] = 0.25; packs.append(a)   # T == 2^-10 exactly, then alpha == thre
    specials = np.array([0.0, -0.0, 0.01, 0.01, 1.0, 1.5, NAN, INF, -INF, 1e-40, 1e-45, 0.3, 0.999], np.float32)
    for k, s in enumerate(specials):
        a = (rng.random(40) ** 4).astype(np.float32) * 0.2
        a[rng.random(40) < 0.3] = 0.0
        a[3 + k] = s
        packs.append(a)
    for n in LENS:
        a = (rng.random(n) ** 3).astype(np.float32)
        a[rng.random(n) < 0.4] = 0.0
        a[rng.random(n) < 0.05] = 0.01
        a[rng.random(n) < 0.002] = 0.999
        packs.append(a)
    alpha = torch.from_numpy(np.concatenate(packs))
    return alpha, _layout([len(a) for a in packs])


def _bwd_visits(a, pi, eps, thre):
    """the samples the backward visits: not skipped (alpha < thre) and before its early stop (T < eps), T in fp32 as it walks them"""
    a = a.numpy()
    vis = np.zeros(a.shape[0], bool)
    eps, thre = np.float32(eps), np.float32(thre)
    for b, n in pi.tolist():
        T = np.float32(1)
        for j in range(b, b + n):
            if T < eps:
                break
            if a[j] < thre:
                continue
            vis[j] = True
            T = np.float32(T * np.float32(np.float32(1) - a[j]))
    return vis


def _ga_close(ga, ga_r, pi, a, w, gw, eps, thre, what):
    """the backward's warp-summed accum differs from the serial sum by rounding: same NaN / inf positions, exact zeros at the samples
    it does not visit (skipped and stopped), the rest within rtol 1e-3, plus 1e-4 of the pack's largest finite value, plus the
    reordered sum's error bound n * 2^-23 * sum|gw w| of the pack divided by max(1 - alpha, 1e-10) (a cancellation at alpha near 1)"""
    g, r = ga.detach().cpu().numpy(), ga_r.detach().cpu().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(r)), (what, np.flatnonzero(np.isnan(g) != np.isnan(r))[:8])
    assert np.array_equal(np.isinf(g), np.isinf(r)) and np.array_equal(g[np.isinf(g)], r[np.isinf(r)]), what
    vis = _bwd_visits(a, pi, eps, thre)
    assert np.all(g[~vis] == 0) and np.all(r[~vis] == 0), (what, np.flatnonzero(~vis & ((g != 0) | (r != 0)))[:8])
    fin = np.isfinite(r)
    pid = pack_ids(pi).numpy()
    scale, terms = np.zeros(pi.shape[0]), np.zeros(pi.shape[0])
    np.maximum.at(scale, pid[fin], np.abs(r[fin]).astype(np.float64))
    gww = np.abs(gw.detach().cpu().numpy().astype(np.float64) * w.detach().cpu().numpy().astype(np.float64))
    np.add.at(terms, pid, np.where(np.isfinite(gww), gww, 0))
    n = pi[:, 1].numpy().astype(np.float64)
    den = np.maximum(np.float32(1) - a.numpy(), np.float32(1e-10)).astype(np.float64)
    den = np.where(np.isnan(den), 1e-10, den)
    tol = 1e-3 * np.abs(r.astype(np.float64)) + 1e-4 * scale[pid] + n[pid] * 2.0 ** -23 * terms[pid] / den
    err = np.abs(g.astype(np.float64) - r)
    assert np.all(err[fin] <= tol[fin]), (what, np.flatnonzero(fin)[np.argmax((err - tol)[fin])])


@pytest.mark.parametrize("eps,thre", [(2.0 ** -10, 0.01), (2.0 ** -10, 0.0), (1e-4, 0.01), (0.0, 0.0)])
def test_alpha_to_vw_edges(G, eps, thre):
    a, pi = alpha_inputs(5)
    ac, pic = a.cuda(), pi.cuda()
    w = B().packed_alpha_to_vw_forward(ac, pic, eps, thre, False)[0]
    w_r = opk.packed_alpha_to_vw_forward(a, pi, eps, thre, False)[0]
    same(w, w_r, "weights", any_nan=True)
    _, info, sel = B().packed_alpha_to_vw_forward(ac, pic, eps, thre, True)
    _, info_r, sel_r = opk.packed_alpha_to_vw_forward(a, pi, eps, thre, True)
    same(info, info_r, "num_steps"), same(sel, sel_r, "selector")
    tag = f"vw_{eps:g}_{thre:g}"
    G.equal(tag + ".w", w, lambda ref: ref.packed_alpha_to_vw_forward(ac, pic, eps, thre, False)[0])
    G.equal(tag + ".info", info, lambda ref: ref.packed_alpha_to_vw_forward(ac, pic, eps, thre, True)[1].long())
    G.equal(tag + ".sel", sel, lambda ref: ref.packed_alpha_to_vw_forward(ac, pic, eps, thre, True)[2])
    gw = torch.from_numpy(np.random.default_rng(6).normal(size=a.shape[0]).astype(np.float32))
    gwc = gw.cuda()
    ga = B().packed_alpha_to_vw_backward(w, gwc, ac, pic, eps, thre)
    _ga_close(ga, opk.packed_alpha_to_vw_backward(w.cpu(), gw, a, pi, eps, thre), pi, a, w, gw, eps, thre, tag + " vs oracle")
    _ga_close(ga, G.value(tag + ".ga", lambda ref: ref.packed_alpha_to_vw_backward(w, gwc, ac, pic, eps, thre)), pi, a, w, gw, eps, thre,
              tag + " vs reference")
    # the sample whose alpha equals thre: skipped by the forward (<=), visited by the backward (<)
    if thre > 0:
        at = (a == np.float32(thre)) & torch.from_numpy(~sel_r.numpy()) & (ga.cpu() != 0)
        assert bool(at.any())


# ------------------------------------------------------------------------------------------------ sort
def sort_values(lens, seed, gaps=None):
    rng = np.random.default_rng(seed)
    pool = np.array([NAN, -INF, INF, -0.0, 0.0, 1.0, 1.0, 0.5, -3.0], np.float32)
    pi = _layout(lens, gaps)
    S = int(pi[-1, 0] + pi[-1, 1])
    v = rng.normal(size=S).astype(np.float32)
    m = rng.random(S) < 0.5
    v[m] = rng.choice(pool, int(m.sum()))
    return torch.from_numpy(v), pi


def _sort_check(v, pi, return_idx, what):
    vg = v.cuda()
    idx = B().packed_sort_qsort(vg, pi.cuda(), return_idx)
    vr = v.clone()
    idx_r = opk.packed_sort_qsort(vr, pi, return_idx)
    same(vg, vr, what + " values")
    if return_idx:
        same(idx, idx_r, what + " idx")
    else:
        assert idx is None
    return vg, idx


@pytest.mark.parametrize("return_idx", [True, False])
def test_sort_edges(G, return_idx):
    lens = [1, 2, 31, 32, 33, 1024, 3000]
    v, pi = sort_values(lens, 21)
    vg, idx = _sort_check(v, pi, return_idx, "packs")
    _sort_check(*sort_values([3, 0, 31, 0, 0, 33, 1, 0], 22), return_idx, "empty packs")      # oracle only: qsort's h = num - 1 wraps
    vgap, pgap = sort_values([5, 31, 2, 64, 1], 23, gaps=[3, 0, 7, 1, 0])
    vg2, idx2 = _sort_check(vgap, pgap, return_idx, "gapped")
    # the reference's quicksort is not stable and meets NaN with `<=`: its idx is a permutation, vals == old[idx], and the numbers agree
    vc, pic = v.cuda(), pi.cuda()
    for name, vv, pp, mine in (("sort", v, pi, vg), ("sort_gapped", vgap, pgap, vg2)):
        vvc, ppc = vv.cuda(), pp.cuda()

        def run(ref, k):
            x = vvc.clone()
            i = ref.packed_sort_qsort(x, ppc, True)
            return (x, i)[k]
        rv = G.value(f"{name}.vals", lambda ref: run(ref, 0))
        if not return_idx:
            continue
        ri = G.value(f"{name}.idx", lambda ref: run(ref, 1))
        assert np.array_equal(bits(rv), bits(vv[ri]))
        for b, n in pp.tolist():
            assert torch.equal(ri[b:b + n].sort().values, torch.arange(b, b + n))
            r, o = rv[b:b + n], mine.cpu()[b:b + n]
            assert torch.equal(r[~torch.isnan(r)].sort().values, o[~torch.isnan(o)])     # the numbers, ascending (-0.0 == +0.0)
        inside = torch.zeros(vv.shape[0], dtype=torch.bool)
        for b, n in pp.tolist():
            inside[b:b + n] = True
        assert torch.equal(ri[~inside], torch.arange(vv.shape[0])[~inside])
    with pytest.raises(RuntimeError, match="last pack ends"):
        B().packed_sort_qsort(torch.zeros(int(pi[-1].sum()) + 1, device="cuda"), pi.cuda(), return_idx)


def test_sort_nan_is_a_permutation():
    """NaN ranks after every number (was: rank 0, two elements in one slot and the last slots of the pack unwritten)"""
    v = torch.tensor([2.0, NAN, 1.0, NAN, -0.0, 0.0, 1.0] * 5)
    pi = torch.tensor([[0, 35]])
    vg = v.cuda()
    idx = B().packed_sort_qsort(vg, pi.cuda(), True).cpu()
    assert torch.equal(idx.sort().values, torch.arange(35))
    vr = v.clone()
    same(idx, opk.packed_sort_qsort(vr, pi, True), "idx")
    same(vg, vr, "values")


# ------------------------------------------------------------------------------------------------ sum / cumsum / diff
def _special_feats(S, C, seed):
    rng = np.random.default_rng(seed)
    f = rng.normal(size=(S, C)).astype(np.float32)
    r = rng.random((S, C))
    f[r < 0.004] = NAN
    f[(r >= 0.004) & (r < 0.008)] = INF
    f[(r >= 0.008) & (r < 0.012)] = -INF
    f[(r >= 0.012) & (r < 0.014)] = 3e38                                    # partial sums that overflow
    return torch.from_numpy(f if C > 1 else f[:, 0].copy())


def _pattern_close(got, ref, skip, what):
    g, r = got.cpu().numpy(), ref.numpy()
    k = ~skip
    assert np.array_equal(np.isnan(g[k]), np.isnan(r[k])), what
    assert np.array_equal(np.isinf(g[k]), np.isinf(r[k])) and np.array_equal(g[k][np.isinf(g[k])], r[k][np.isinf(r[k])]), what
    fin = k & np.isfinite(r)
    assert np.allclose(g[fin], r[fin], rtol=1e-5, atol=1e-3), what


@pytest.mark.parametrize("C", [1, 3, 16])
def test_sum_cumsum_diff_edges(C):
    lens = [0, 1, 2, 31, 0, 32, 33, 64, 65, 1024, 4097, 0]
    pi = _layout(lens)
    S = int(pi[:, 1].sum())
    f = _special_feats(S, C, 30 + C)
    fc, pic = f.cuda(), pi.cuda()
    f2 = f.numpy().reshape(S, -1).astype(np.float64)
    big = np.abs(np.where(np.isfinite(f2), f2, 0)).reshape(S, -1)
    pid = pack_ids(pi).numpy()
    overflow = np.zeros((pi.shape[0], big.shape[1]), bool)
    np.logical_or.at(overflow, pid, big >= 1e38)                           # a pack whose partial sums may overflow: order decides
    sk_pack = overflow if C > 1 else overflow[:, 0]
    sk_elem = overflow[pid] if C > 1 else overflow[pid, 0]
    _pattern_close(B().packed_sum(fc, pic), opk.packed_sum(f, pi), sk_pack, "sum")
    for ex in (False, True):
        for rev in (False, True):
            _pattern_close(B().packed_cumsum(fc, pic, ex, rev), opk.packed_cumsum(f, pi, ex, rev), sk_elem, f"cumsum ex={ex} rev={rev}")
    P = pi.shape[0]
    app = torch.from_numpy(np.random.default_rng(C).normal(size=(P, C) if C > 1 else P).astype(np.float32))
    app[1] = INF
    for kw in (dict(), dict(a=app), dict(b=app)):
        ea, eb = kw.get("a"), kw.get("b")
        same(B().packed_diff(fc, pic, None if ea is None else ea.cuda(), None if eb is None else eb.cuda()),
             opk.packed_diff(f, pi, ea, eb), f"diff {list(kw)}", any_nan=True)
        same(B().packed_backward_diff(fc, pic, None if ea is None else ea.cuda(), None if eb is None else eb.cuda()),
             opk.packed_backward_diff(f, pi, ea, eb), f"backward_diff {list(kw)}", any_nan=True)


def test_exclusive_cumsum_ignores_its_own_element():
    """the exclusive sum at an inf or NaN element is the sum of the elements before it (it was inc - v: NaN)"""
    f = torch.tensor([1.0, INF, 2.0, NAN, 3.0] + [0.5] * 40)
    pi = torch.tensor([[0, 45]])
    got = B().packed_cumsum(f.cuda(), pi.cuda(), True, False).cpu()
    assert got[0] == 0 and got[1] == 1 and got[2] == INF and torch.isnan(got[4:]).all() and got[3] == INF


# ------------------------------------------------------------------------------------------------ binary ops
def test_binary_ops_edges():
    lens = [0, 3, 1, 33, 0, 64, 2]
    pi = _layout(lens)
    S = int(pi[:, 1].sum())
    vals = np.array([0.0, -0.0, 1.0, -1.0, INF, -INF, NAN, 1e-40, 3e38, 2.5], np.float32)
    rng = np.random.default_rng(40)
    for C in (1, 3):
        f = torch.from_numpy(rng.choice(vals, (S, C) if C > 1 else S))
        o = torch.from_numpy(rng.choice(vals, (len(lens), C) if C > 1 else len(lens)))
        for name in ("add", "sub", "mul", "div", "gt", "geq", "lt", "leq", "eq", "neq"):
            got = getattr(B(), f"packed_{name}")(f.cuda(), o.cuda(), pi.cuda())
            same(got, getattr(opk, f"packed_{name}")(f, o, pi), f"{name} C={C}", any_nan=True)


# ------------------------------------------------------------------------------------------------ producers
def test_interleave_edges():
    n = torch.tensor([0, 3, 0, 33, 65, (1 << 24) + 70, 1, 0])              # empty packs at both ends; j past 2^24
    P = n.shape[0]
    start = torch.tensor([0.5, -1.0, 2.0, 1e6, -3.25, 0.125, 7.0, 1.0])
    step = torch.tensor([0.1, -0.7, 0.0, 1.5, -1e-3, 0.3, 2.0, 1.0])         # negative and zero steps
    out, nidx = B().interleave_arange(n.cuda(), True)
    ro, rn = opk.interleave_arange(n, True)
    same(out, ro, "arange"), same(nidx, rn, "arange nidx")
    out, nidx = B().interleave_linstep(start.cuda(), n.cuda(), step.cuda(), True)
    ro, rn = opk.interleave_linstep(start, n, step, True)
    same(out, ro, "linstep tensor step"), same(nidx, rn, "linstep nidx")
    big = int(n[:5].sum()) + (1 << 24) + 1
    assert out[big] == out[big - 1] or step[5] == 0                         # (float)j: 2^24 + 1 rounds to 2^24
    for s in (-0.375, 0.0):
        out, none = B().interleave_linstep(start.cuda(), n.cuda(), s, False)
        assert none is None
        same(out, opk.interleave_linstep(start, n, s, False)[0], f"linstep scalar {s}")
    assert P == 8


# ------------------------------------------------------------------------------------------------ composite (replay_chunk's other caller)
def test_composite_nan_and_thre_alpha():
    """k_composite_fwd visits a NaN alpha and skips alpha == thre, k_composite_bwd visits both: against packed_alpha_to_vw + sums"""
    from neuralsim_b200.graphics import neus_fused as NF
    thre, eps = 0.01, 1e-4
    rng = np.random.default_rng(50)
    lens = [40, 40, 70, 5]
    pi = _layout(lens)
    S = int(pi[:, 1].sum())
    a = (rng.random(S) * 0.1).astype(np.float32)                           # no early stop: T >= 0.9^70
    a[3], a[45], a[46], a[90] = NAN, thre, thre, NAN                        # NaN in packs 0 and 2; alpha == thre in pack 1
    t = np.sort(rng.random(S)).astype(np.float32)
    ac = torch.from_numpy(a).cuda().requires_grad_(True)
    vw, m, d, _, _ = NF.composite(ac, torch.from_numpy(t).cuda(), pi.cuda(), normalize_depth=False, early_stop_eps=eps, alpha_thre=thre)
    w_r = opk.packed_alpha_to_vw_forward(torch.from_numpy(a), pi, eps, thre, False)[0]
    same(vw, w_r, "composite weights", any_nan=True)
    m_r = opk.packed_sum(w_r, pi)
    d_r = opk.packed_sum(w_r * torch.from_numpy(t), pi)
    assert np.array_equal(np.isnan(m.detach().cpu().numpy()), np.isnan(m_r.numpy()))
    fin = torch.isfinite(m_r)
    assert torch.allclose(m.detach().cpu()[fin], m_r[fin], rtol=1e-5) and torch.allclose(d.detach().cpu()[fin], d_r[fin], rtol=1e-5)
    gm = torch.from_numpy(rng.normal(size=len(lens)).astype(np.float32))
    (m * gm.cuda()).sum().backward()
    ga_r = opk.packed_alpha_to_vw_backward(w_r, gm[pack_ids(pi)], torch.from_numpy(a), pi, eps, thre)
    _ga_close(ac.grad, ga_r, pi, torch.from_numpy(a), w_r, gm[pack_ids(pi)], eps, thre, "composite d_alpha")
    # the forward visits and the backward's visits: the NaN sample in both, alpha == thre only in the backward
    g = ac.grad.cpu()
    w = vw.detach().cpu()
    assert torch.isnan(w[3]) and torch.isnan(w[90]) and torch.isnan(g[3]) and torch.isnan(g[90])
    b1, n1 = pi[1].tolist()
    at_thre = torch.from_numpy(a[b1:b1 + n1] == np.float32(thre))
    assert int(at_thre.sum()) == 2
    assert torch.equal(g[b1:b1 + n1] != 0, (w[b1:b1 + n1] != 0) | at_thre)


# ------------------------------------------------------------------------------------------------ frame scale
def _sub(pi, packs):
    """the packs `packs` of layout pi, re-laid end to end: (their layout, the element indices they came from)"""
    sel = pi[packs]
    src = torch.cat([torch.arange(b, b + n) for b, n in sel.tolist()]) if len(packs) else torch.zeros(0, dtype=torch.int64)
    return _layout(sel[:, 1]), src


def test_frame_scale(G):
    P = FRAME
    assert warp_trips(P) >= 3
    rng = np.random.default_rng(60)
    lens = rng.integers(1, 7, P)
    lens[rng.random(P) < 0.1] = 0
    lens[0] = lens[-1] = 3
    pi = _layout(lens)
    S = int(lens.sum())
    pic = pi.cuda()
    check = np.unique(np.concatenate([np.arange(0, P, 997), np.arange(P - 300, P)]))      # oracle on a spread of packs, the last trip's included
    spi, src = _sub(pi, check)

    # alpha_to_vw, sums, diff, sort
    a = (rng.random(S) ** 2).astype(np.float32)
    a[rng.random(S) < 0.3] = 0.0
    a[rng.random(S) < 0.01] = NAN
    ac = torch.from_numpy(a).cuda()
    w = B().packed_alpha_to_vw_forward(ac, pic, 1e-4, 0.0, False)[0]
    same(w.cpu()[src], opk.packed_alpha_to_vw_forward(torch.from_numpy(a)[src], spi, 1e-4, 0.0, False)[0], "frame weights", any_nan=True)
    G.equal("frame.vw", w, lambda ref: ref.packed_alpha_to_vw_forward(ac, pic, 1e-4, 0.0, False)[0])
    s = B().packed_sum(ac, pic).cpu()
    assert np.array_equal(np.isnan(s[check].numpy()), np.isnan(opk.packed_sum(torch.from_numpy(a)[src], spi).numpy()))
    cs = B().packed_cumsum(ac, pic, True, True).cpu()
    _pattern_close(cs[src], opk.packed_cumsum(torch.from_numpy(a)[src], spi, True, True), np.zeros(len(src), bool), "frame cumsum")
    same(B().packed_diff(ac, pic).cpu()[src], opk.packed_diff(torch.from_numpy(a)[src], spi), "frame diff", any_nan=True)
    v = ac.clone()
    idx = B().packed_sort_qsort(v, pic, True).cpu()
    vr = torch.from_numpy(a)[src].clone()
    idx_r = opk.packed_sort_qsort(vr, spi, True)
    same(v.cpu()[src], vr, "frame sort values")
    same(idx[src] - torch.repeat_interleave(pi[check, 0] - spi[:, 0], spi[:, 1]), idx_r, "frame sort idx")
    assert torch.equal(idx.sort().values, torch.arange(S))

    # search / inverse cdf: 16 values per pack
    NV = 16
    assert thread_trips(P * NV) >= 3
    cdf = np.zeros(S, np.float32)
    for k in range(1, 7):
        at = pi[:, 0].numpy()[lens > k] + k
        cdf[at] = cdf[at - 1] + np.float32(rng.integers(0, 3, at.size) / 4)          # flat runs
    bins = np.cumsum(rng.random(S) + 0.1).astype(np.float32)
    u = (rng.integers(0, 9, (P, NV)) / 4).astype(np.float32)                            # hits cdf entries exactly, and past them
    u[:, 0], u[:, 1] = NAN, -0.0
    bd, cd, uc = torch.from_numpy(bins).cuda(), torch.from_numpy(cdf).cuda(), torch.from_numpy(u).cuda()
    sm, bi = B().packed_invert_cdf(bd, cd, uc, pic)
    sm_r, bi_r = opk.packed_invert_cdf(torch.from_numpy(np.concatenate([bins[src.numpy()], [NAN]]).astype(np.float32)),
                                       torch.from_numpy(np.concatenate([cdf[src.numpy()], [NAN]]).astype(np.float32)),
                                       torch.from_numpy(u[check]), spi)
    off = (pi[check, 0] - spi[:, 0])[:, None]
    same(bi.cpu()[check] - off, bi_r, "frame bin_idx")
    nz = torch.from_numpy(lens[check] > 0)                                                # an empty pack's sample reads the next pack
    same(sm.cpu()[check][nz], sm_r[nz], "frame samples", any_nan=True)
    G.equal("frame.invert_cdf", sm, lambda ref: ref.packed_invert_cdf(bd, cd, uc, pic)[0])
    G.equal("frame.bin_idx", bi, lambda ref: ref.packed_invert_cdf(bd, cd, uc, pic)[1])

    # merge: unsorted b with ties and NaN (one thread per pack), and sorted b; a has no empty pack (the reference writes pidx_a[begin])
    la = np.maximum(lens, 1)
    pia = _layout(la)
    lb = rng.integers(0, 5, P)
    pib = _layout(lb)
    va_c = torch.from_numpy(rng.integers(0, 6, int(la.sum())).astype(np.float32) / 4).cuda()
    B().packed_sort_qsort(va_c, pia.cuda(), False)
    vb = (rng.integers(0, 6, int(lb.sum())) / 4).astype(np.float32)
    vb[rng.random(vb.size) < 0.05] = NAN
    vb_c = torch.from_numpy(vb).cuda()
    piac, pibc = pia.cuda(), pib.cuda()
    spa, srca = _sub(pia, check)
    spb, srcb = _sub(pib, check)
    va_h = va_c.cpu()
    for b_sorted in (False, True):
        if b_sorted:
            B().packed_sort_qsort(vb_c, pibc, False)
        ga, gb, gp = B().try_merge_two_packs_sorted_aligned(va_c, piac, vb_c, pibc, b_sorted)
        ra, rb, rp = opk.try_merge_two_packs_sorted_aligned(va_h[srca], spa, vb_c.cpu()[srcb], spb, b_sorted)
        o = torch.from_numpy(gp.cpu().numpy()[check, 0]) - rp[:, 0]
        same(ga.cpu()[srca] - torch.repeat_interleave(o, spa[:, 1]), ra, f"frame merge{b_sorted} a")
        same(gb.cpu()[srcb] - torch.repeat_interleave(o, spb[:, 1]), rb, f"frame merge{b_sorted} b")
        if b_sorted:                          # (unsorted b: the reference's run bookkeeping assumes equal bins are adjacent in b)
            assert torch.equal(torch.cat([ga, gb]).sort().values.cpu(), torch.arange(int(la.sum() + lb.sum())))
        vbs = vb_c.clone()
        for k, y in enumerate((ga, gb, gp)):
            G.equal(f"frame.merge{int(b_sorted)}.{k}", y, lambda ref: ref.try_merge_two_packs_sorted_aligned(va_c, piac, vbs, pibc, b_sorted)[k])
