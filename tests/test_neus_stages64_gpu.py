"""The per-ray NeuS stage kernels (csrc/neus_fused.cu: k_upsample_cdf, k_invert_cdf_shared_u, k_neus_alpha_fwd / _bwd, k_composite_fwd /
_bwd, and through them the device functions of csrc/neus_device.cuh) against the float64 statement of their contract, oracle/neus64.py.

One warp owns one pack and replays the serial transmittance recurrence 32 samples at a time (replay_chunk); early stop is tested after
each visited sample and once at the start of each chunk.  The inputs here put T's crossing of eps on purpose at lane 0, at lane 31 with
live samples in the next chunk, at lane 32, at the pack's last sample and within an ulp of eps, with a live sample after the stop in the
same chunk, exact-zero alphas at thre 0 and alphas equal to 0.01f at thre 0.01 (the backward visits those, the forward does not),
opaque samples (1 - alpha <= 1e-5), rising sdf (the clamp of the alpha backward) and saturated sigmoids.  Every test asserts from the
oracle's replay that its input reaches the edge it names.  Pack lengths run 0, 1, 2, 31, 32, 33, 63, 64, 65, 97, 500 and 4096 in one
launch; the grid-stride test sizes the pack count from the SM count so that every warp of every stage kernel runs >= 3 packs (state
kept across a warp's packs: acc_invs of k_neus_alpha_bwd) and the inverse-cdf launch loops too.  The count-bound launches run with a
device count below the capacity, NaN cotangents and sentinel outputs past it.

Decisions (selector, num_steps, vw, compression, the inverse cdf's bin) are compared bit for bit; values per element against float64
with bounds c 2^-24 sum|terms| (oracle/neus64.py returns the sum of |terms| of each value).  The constants c are about 3x the largest
ratio measured on an H100 80GB HBM3; DESIGN.md §4 lists them."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import neus64 as o64

pytestmark = pytest.mark.gpu

F32 = np.float32
U = o64.U32
EPS = 1e-4
LADDER = [0, 1, 2, 31, 32, 33, 63, 64, 65, 97, 500, 4096, 0]
# bounds: |kernel - float64| <= C * 2^-24 * (sum of |terms|) per element
C_ALPHA = 7.0          # alpha of k_neus_alpha_fwd (expf); measured <= 2.3
C_SUM = 10.0           # mask, depth, rgb, nablas, d_rgb, d_nablas; measured <= 3.6
C_CDF = 1.2            # cdf of k_upsample_cdf; measured <= 0.36
C_INV = 3.0            # inverse-cdf samples; measured <= 0.85
C_DALPHA = 12.0        # d_alpha of k_composite_bwd; measured <= 4.2
C_DSDF = 20.0          # d_sdf of k_neus_alpha_bwd (the sigmoid's derivative); measured <= 6.9
INV_S_REL = 1.5e-5     # d_inv_s of k_neus_alpha_bwd over the sum of |terms|; measured <= 4.9e-6 of |d_inv_s|
EST_CDF = 2e-6         # cdf with the up-sampling estimate alpha (not exposed: float64 alphas), absolute; measured 7.0e-7
CHAIN_REL = 1e-5       # the compress -> composite -> backward chain against float64 of the chain, rel-L2; measured <= 2.9e-6


def report(name, value):
    print(f"METRIC {name} {value:.4g}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _warps():
    """warps of a pack_grid launch at the grid-stride limit (wave_grid: 8 waves of 8 CTAs of 256 threads per SM)"""
    return 8 * 8 * _sms() * 256 // 32


def _pi(lengths):
    n = np.asarray(lengths, dtype=np.int64)
    return np.stack([np.cumsum(n) - n, n], 1)


def _cuda(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t if dtype is None else t.to(dtype)


def _ratio(err, scale, floor=1e-30):
    return float((np.abs(err) / (U * np.maximum(scale, floor))).max()) if np.size(err) else 0.0


# ============================================================================================================== inputs
def _sdf_pack(kind, n, rng):
    """sdf and depth of one pack: 'cross' (a surface with noise), 'flat' (constant: every alpha exactly 0), 'rise' (sdf rising: raw < 0),
    'sat' (sdf far outside: c == 1.0f), ('drop', K) (+1 up to K, then falling: alpha ~ 1 at interval K, tiny live alphas after)"""
    t = np.sort(rng.uniform(0.5, 2.5, n)).astype(F32)
    if kind == "cross":
        s = (1.4 - t) * rng.uniform(0.3, 2.0) + 0.02 * rng.standard_normal(n)
    elif kind == "flat":
        s = np.full(n, rng.uniform(-0.2, 0.5))
    elif kind == "rise":
        s = (t - 1.4) * rng.uniform(0.3, 2.0)
    elif kind == "sat":
        s = 1.0 + 0.5 * rng.random(n)
    else:
        K = kind[1]
        s = np.where(np.arange(n) <= K, 1.0, -1.0 - 0.01 * (np.arange(n) - K))
    return s.astype(F32), t


def _sdf_packs(kinds, lengths, seed):
    rng = np.random.default_rng(seed)
    pi = _pi(lengths)
    S = int(pi[:, 1].sum())
    sdf, dep = np.zeros(S, F32), np.zeros(S, F32)
    for (b, n), k in zip(pi, kinds):
        sdf[b:b + n], dep[b:b + n] = _sdf_pack(k, n, rng)
    return pi, sdf, dep


def _ladder_sdf(seed):
    kinds = ["cross", "cross", "rise", "cross", "cross", ("drop", 0), ("drop", 31), "flat", ("drop", 32), "sat", "cross", "cross", "cross"]
    return _sdf_packs(kinds, LADDER, seed)


def _near_eps_pair():
    """fp32 pairs (a1, a2) with T = fl32(fl32(1 - a1) fl32(1 - a2)) == eps exactly ('at': not a stop) and one fp32 step below ('below')"""
    eps = F32(EPS)
    a1 = (F32(0.999) + np.arange(-200, 200).astype(F32) * np.spacing(F32(0.999))).astype(F32)
    a2 = (F32(0.9) + np.arange(-8000, 8000).astype(F32) * np.spacing(F32(0.9))).astype(F32)
    T = ((F32(1) - a1)[:, None] * (F32(1) - a2)[None, :]).astype(F32)
    out = {}
    for name, target in (("at", eps), ("below", np.nextafter(eps, F32(0)))):
        i, j = np.argwhere(T == target)[0]
        out[name] = (a1[i], a2[j])
    return out


def _alpha_edges(thre):
    """hand-built alpha packs, one per replay edge -> (alpha [S] f32, pack_infos, names)"""
    opq = F32(1 - 5e-5)                  # T -> 5e-5 < eps at this sample
    near = _near_eps_pair()
    rng = np.random.default_rng(11)
    packs = []

    def live(n):
        return rng.uniform(0.05, 0.3, n).astype(F32)
    z = lambda n: np.zeros(n, F32)
    packs.append(("empty", z(0)))
    packs.append(("cross_lane0", np.concatenate([[opq], live(39)])))
    packs.append(("cross_lane31_live_next", np.concatenate([z(31), [opq], live(20)])))
    packs.append(("cross_lane32", np.concatenate([z(32), [opq], live(10)])))
    packs.append(("cross_last", np.concatenate([live(44) * F32(0.1), [opq]])))
    packs.append(("T_at_eps", np.concatenate([[near["at"][0], near["at"][1]], live(5)])))
    packs.append(("T_below_eps", np.concatenate([[near["below"][0], near["below"][1]], live(5)])))
    packs.append(("live_after_stop_same_chunk", np.concatenate([live(5), [opq], live(15)])))
    zt = live(70)
    zt[rng.random(70) < 0.4] = F32(thre)
    packs.append(("ties_with_thre", zt))
    packs.append(("opaque", np.concatenate([live(3), [F32(1 - 2e-6)], live(3), [F32(1.0)], live(3)])))
    packs.append(("long", np.concatenate([live(600) * F32(0.01), live(10)])))
    packs.append(("empty_last", z(0)))
    pi = _pi([len(a) for _, a in packs])
    return np.concatenate([a for _, a in packs]).astype(F32), pi, [n for n, _ in packs]


def _assert_alpha_edges(r, pi, names, alpha, thre):
    """the replay reaches the edge each hand-built pack names"""
    e = {n: p for p, n in enumerate(names)}
    cr, st, n = r["cross"], r["stop"], pi[:, 1]
    assert cr[e["cross_lane0"]] == 0 and cr[e["cross_lane32"]] == 32 and cr[e["cross_last"]] == n[e["cross_last"]] - 1
    p = e["cross_lane31_live_next"]
    assert cr[p] == 31 and (alpha[pi[p, 0] + 32:pi[p, 0] + n[p]] > thre).any()
    p, q = e["T_at_eps"], e["T_below_eps"]
    assert r["T"][pi[p, 0] + 2] == F32(EPS) and st[p] > 2 and r["vis"][pi[p, 0] + 2]          # T == eps: not a stop
    assert r["T"][pi[q, 0] + 2] == np.nextafter(F32(EPS), F32(0)) and st[q] == 2
    p = e["live_after_stop_same_chunk"]
    assert cr[p] == 5 and (alpha[pi[p, 0] + 6:pi[p, 0] + n[p]] > thre).all() and n[p] <= 32
    p = e["ties_with_thre"]
    b = pi[p, 0]
    assert (alpha[b:b + n[p]] == F32(thre)).sum() > 10
    assert alpha[pi[e["opaque"], 0]:].max() >= F32(1 - 1e-5)


# ============================================================================================================== kernel calls
def _alpha_fwd(sdf, pi, inv_s, thre):
    from neuralsim_b200.graphics import neus_fused as NF
    s = _cuda(sdf).requires_grad_(True)
    inv = torch.tensor(float(inv_s), device="cuda", requires_grad=True)
    a, sel, steps = NF._NeusAlpha.apply(s, inv, _cuda(pi), EPS, thre)
    return s, inv, a, sel, steps


def _check_alpha_fwd(sdf, pi, inv_s, thre, a, sel, steps):
    a_np = a.detach().cpu().numpy()
    r = o64.replay(a_np, pi, EPS, thre)
    assert np.array_equal(sel.cpu().numpy(), r["vis"]) and np.array_equal(steps.cpu().numpy(), r["steps"])
    a64, scale = o64.neus_alpha(sdf, pi, inv_s)
    cov = o64.pack_of(pi, sdf.shape[0]) >= 0
    ratio = _ratio((a_np - a64)[cov], scale[cov], 1.0)
    assert ratio <= C_ALPHA, ratio
    return r, ratio


def _inv_s_ratio(got, want):
    """|d_inv_s - float64| beyond what ambiguous clamp decisions may add, over the sum of |terms| (the kernel sums per lane, per warp
    and then with one atomic per warp: the order differs from any serial sum)"""
    return max(abs(got - want["d_inv_s"]) - want["d_inv_s_ambiguous"], 0.0) / want["d_inv_s_abs"]


# ============================================================================================================== tests
@pytest.mark.parametrize("thre", [0.0, 0.01])
@pytest.mark.parametrize("inv_s", [64.0, 1024.0])
def test_alpha_forward_backward_and_compression_ladder(thre, inv_s):
    """k_neus_alpha_fwd on the pack-length ladder: alpha against float64, selector / num_steps / compression bit for bit against the
    replay of the kernel's alphas, then k_neus_alpha_bwd: d_sdf per element and d_inv_s against float64"""
    from neuralsim_b200.graphics import neus_fused as NF
    pi, sdf, _ = _ladder_sdf(1)
    s, inv, a, sel, steps = _alpha_fwd(sdf, pi, inv_s, thre)
    r, ratio = _check_alpha_fwd(sdf, pi, inv_s, thre, a, sel, steps)
    report(f"alpha_ulps[{thre},{inv_s}]", ratio)
    a_np = a.detach().cpu().numpy()
    n = pi[:, 1]
    assert r["cross"][5] == 0 and r["cross"][6] == 31 and r["cross"][8] == 32        # the ('drop', K) packs reach their edges
    if inv_s == 64.0:                         # live (tiny) alphas in the chunk after lane 31; at 1024 the sigmoids underflow to 0
        assert (a_np[pi[6, 0] + 32:pi[6, 0] + n[6] - 1] > 0).all()                  # (the last sample's alpha is 0)
    assert (a_np[pi[7, 0]:pi[7, 0] + n[7]] == 0).all()                                # flat: exact zeros
    assert (a_np[pi[2, 0]:pi[2, 0] + n[2]] == 0).all()                                # rising: clamped
    x = o64.sigmoid_arg(sdf[pi[9, 0]:pi[9, 0] + n[9]], inv_s)
    assert (x > 17).all()                                                            # c == 1.0f on both sides of every interval
    # compression (the pack infos the render pass continues with)
    _, nidx, pinf, pidx = NF.neus_alpha_compress(_cuda(sdf), torch.tensor(inv_s, device="cuda"), _cuda(pi), EPS, thre)
    nidx_r, pinf_r = o64.compression(r["steps"])
    assert np.array_equal(nidx.cpu().numpy(), nidx_r) and np.array_equal(pinf.cpu().numpy(), pinf_r)
    assert np.array_equal(pidx.cpu().numpy(), np.nonzero(r["vis"])[0])
    # backward: random d_alpha with ~30 % zeros
    rng = np.random.default_rng(2)
    g = rng.standard_normal(sdf.shape[0]).astype(F32)
    g[rng.random(g.shape[0]) < 0.3] = 0
    (a * _cuda(g)).sum().backward()
    want = o64.alpha_backward(sdf, pi, inv_s, g)
    rd = _ratio(s.grad.cpu().numpy() - want["d_sdf"], want["d_sdf_scale"])
    ri = _inv_s_ratio(float(inv.grad), want)
    report(f"d_sdf[{thre},{inv_s}]", rd)
    report(f"d_inv_s[{thre},{inv_s}]", ri)
    assert rd <= C_DSDF and ri <= INV_S_REL, (rd, ri)


@pytest.mark.parametrize("estimate", [False, True])
def test_upsample_cdf_and_inverse_cdf_ladder(estimate):
    """k_upsample_cdf on the ladder (with packs whose weights are all zero: norm = 1e-5) and k_invert_cdf_shared_u on its cdf; empty
    packs get NaN samples.  Production never passes an empty pack: the up-sampler's packs are the hit rays of the march (>= 1 sample)."""
    from neuralsim_b200.graphics import neus_fused as NF
    pi, sdf, dep = _ladder_sdf(3)
    inv_s = 64.0
    cdf = NF.upsample_cdf(_cuda(sdf), _cuda(dep), _cuda(pi), inv_s, estimate, EPS, 0.0).cpu().numpy()
    cov = o64.pack_of(pi, sdf.shape[0]) >= 0
    if not estimate:
        _, _, a, _, _ = _alpha_fwd(sdf, pi, inv_s, 0.0)                 # the same neus_alpha_at: the cdf's alphas bit for bit
        r = o64.replay(a.detach().cpu().numpy(), pi, EPS, 0.0)
        want, scale = o64.upsample_cdf(r["w"], pi)
        ratio = _ratio((cdf - want)[cov], scale[cov], 1e-30)
        report("cdf_ulps", ratio)
        assert ratio <= C_CDF, ratio
    else:
        a64 = o64.upsample_alpha(sdf, dep, pi, inv_s)
        r = o64.replay(a64.astype(F32), pi, EPS, 0.0)
        T64, w64 = o64.transmittance(a64, r["vis"], pi)
        want, _ = o64.upsample_cdf(w64, pi)
        err = float(np.abs(cdf - want)[cov].max())
        report("cdf_est_abs", err)
        assert err <= EST_CDF, err
    flat = pi[7]
    assert np.array_equal(cdf[flat[0]:flat[0] + flat[1]], np.zeros(flat[1], F32))     # all weights 0: 0 / max(0, 1e-5)
    _check_invert(dep, cdf, pi, 33)


def _check_invert(dep, cdf, pi, n_s, packs=None):
    from neuralsim_b200.graphics import neus_fused as NF
    got = NF.sample_cdf_uniform(_cuda(dep), _cuda(cdf), _cuda(pi), n_s).cpu().numpy()
    u = np.linspace(0, 1, n_s + 2, dtype=F32)[1:-1]
    sel = np.arange(pi.shape[0]) if packs is None else packs
    want, scale = o64.invert_cdf(dep, cdf, u, pi[sel])
    g = got[sel]
    empty = pi[sel, 1] == 0
    assert np.isnan(g[empty]).all() and not np.isnan(g[~empty]).any()
    ratio = _ratio((g - want)[~empty], scale[~empty], 1e-30)
    report("invert_ulps", ratio)
    assert ratio <= C_INV, ratio
    return got


def _composite_inputs(alpha, pi, seed, n_rays=None):
    rng = np.random.default_rng(seed)
    S, P = alpha.shape[0], pi.shape[0]
    t = np.concatenate([np.sort(rng.uniform(0.5, 3.0, n)) for n in pi[:, 1]]).astype(F32) if S else np.zeros(0, F32)
    rgb, nab = rng.random((S, 3)).astype(F32), rng.standard_normal((S, 3)).astype(F32)
    R = P if n_rays is None else n_rays
    cot = dict(g_mask=rng.standard_normal(R), g_depth=rng.standard_normal(R), g_rgb=rng.standard_normal((R, 3)),
               g_nablas=rng.standard_normal((R, 3)), g_vw=rng.standard_normal(S))
    return t, rgb, nab, {k: v.astype(F32) for k, v in cot.items()}


def _run_composite(alpha, t, pi, rgb, nab, cot, normalize_depth, thre, ray_index=None, n_rays=None):
    from neuralsim_b200.graphics import neus_fused as NF
    a = _cuda(alpha).requires_grad_(True)
    r = _cuda(rgb).requires_grad_(True) if rgb is not None else None
    nb = _cuda(nab).requires_grad_(True) if nab is not None else None
    ri = _cuda(ray_index) if ray_index is not None else None
    vw, m, d, c, n_ = NF.composite(a, _cuda(t), _cuda(pi), rgb=r, nablas=nb, normalize_depth=normalize_depth, early_stop_eps=EPS,
                                   alpha_thre=thre, ray_index=ri, n_rays=n_rays)
    loss = (m * _cuda(cot["g_mask"])).sum() + (d * _cuda(cot["g_depth"])).sum() + (vw * _cuda(cot["g_vw"])).sum()
    if r is not None:
        loss = loss + (c * _cuda(cot["g_rgb"])).sum()
    if nb is not None:
        loss = loss + (n_ * _cuda(cot["g_nablas"])).sum()
    loss.backward()
    out = dict(vw=vw, mask=m, depth=d, rgb=c, nablas=n_, d_alpha=a.grad, d_rgb=None if r is None else r.grad,
               d_nablas=None if nb is None else nb.grad)
    return {k: (None if v is None else v.detach().cpu().numpy()) for k, v in out.items()}


def _check_composite(alpha, t, pi, rgb, nab, cot, normalize_depth, thre, got, ray_index=None, tag=""):
    """got: the kernel's outputs -> the largest bound ratios; asserts everything"""
    r = o64.replay(alpha, pi, EPS, thre)
    assert np.array_equal(got["vw"].view(np.int32), r["w"].view(np.int32))
    o = np.arange(pi.shape[0]) if ray_index is None else ray_index
    fw = o64.composite_forward(r["w"], t, pi, rgb, nab, normalize_depth)
    ratios = {}
    for k in ("mask", "depth", "rgb", "nablas"):
        if fw.get(k) is None or got[k] is None:
            continue
        ratios[k] = _ratio(got[k][o] - fw[k], fw[k + "_scale"])
    rb = o64.replay(alpha, pi, EPS, thre, backward=True)
    sl = lambda v: None if v is None else v[o]
    g = dict(g_mask=sl(cot["g_mask"]), g_depth=sl(cot["g_depth"]), g_vw=cot["g_vw"],
             g_rgb=sl(cot["g_rgb"]) if rgb is not None else None, g_nablas=sl(cot["g_nablas"]) if nab is not None else None)
    bw = o64.composite_backward(alpha, t, pi, r["w"], rb["T"], rb["vis"], got["mask"][o], got["depth"][o], rgb=rgb, nablas=nab,
                                normalize_depth=normalize_depth, **g)
    assert (got["d_alpha"][~rb["vis"]] == 0).all()                                # zero where the backward does not visit
    ratios["d_alpha"] = _ratio(got["d_alpha"] - bw["d_alpha"], bw["d_alpha_scale"])
    for k in ("d_rgb", "d_nablas"):
        if got[k] is not None:
            ratios[k] = _ratio(got[k] - bw[k], bw[k + "_scale"])
    for k, v in ratios.items():
        report(f"{tag}{k}", v)
    bound = dict(d_alpha=C_DALPHA)
    bad = {k: v for k, v in ratios.items() if v > bound.get(k, C_SUM)}
    assert not bad, bad
    return r, rb


@pytest.mark.parametrize("thre", [0.0, 0.01])
@pytest.mark.parametrize("normalize_depth", [True, False])
def test_composite_replay_edges(thre, normalize_depth):
    """k_composite_fwd / _bwd on hand-built alphas at every edge of replay_chunk, with rgb and nablas"""
    alpha, pi, names = _alpha_edges(thre)
    t, rgb, nab, cot = _composite_inputs(alpha, pi, 5)
    got = _run_composite(alpha, t, pi, rgb, nab, cot, normalize_depth, thre)
    r, rb = _check_composite(alpha, t, pi, rgb, nab, cot, normalize_depth, thre, got, tag=f"edges[{thre},{normalize_depth}].")
    _assert_alpha_edges(r, pi, names, alpha, thre)
    tie = (alpha == F32(thre)) & rb["vis"]
    assert tie.any() and not r["vis"][tie].any() and (got["d_alpha"][tie] != 0).all()    # the backward visits alpha == thre


@pytest.mark.parametrize("present", ["rgb", "nablas", "none"])
def test_composite_ray_index_and_optional_inputs(present):
    """per-pack outputs scattered to image slots (ray_index), with rgb / nablas absent; the slots no pack writes stay zero"""
    alpha, pi, _ = _alpha_edges(0.0)
    P = pi.shape[0]
    n_rays = 3 * P + 5
    ray_index = np.random.default_rng(7).permutation(n_rays)[:P].astype(np.int64)
    t, rgb, nab, cot = _composite_inputs(alpha, pi, 6, n_rays)
    rgb = rgb if present == "rgb" else None
    nab = nab if present == "nablas" else None
    got = _run_composite(alpha, t, pi, rgb, nab, cot, True, 0.0, ray_index=ray_index, n_rays=n_rays)
    _check_composite(alpha, t, pi, rgb, nab, cot, True, 0.0, got, ray_index=ray_index, tag=f"ray_index[{present}].")
    free = np.setdiff1d(np.arange(n_rays), ray_index)
    for k in ("mask", "depth", "rgb", "nablas"):
        if got[k] is not None:
            assert (got[k][free] == 0).all(), k


def _big_packs(seed):
    """>= 3 packs per warp of a pack_grid launch, lengths 0..96 (the ladder covers long packs), a mix of every sdf kind"""
    W = _warps()
    P = 3 * W + W // 3 + 17
    rng = np.random.default_rng(seed)
    n = rng.integers(0, 97, P)
    kinds_pool = ["cross", "cross", "cross", "flat", "rise", "sat", ("drop", 3), ("drop", 31)]
    kinds = [kinds_pool[i] for i in rng.integers(0, len(kinds_pool), P)]
    kinds = [("drop", min(k[1], max(int(m) - 1, 0))) if isinstance(k, tuple) else k for k, m in zip(kinds, n)]
    pi, sdf, dep = _sdf_packs(kinds, n, seed)
    return W, pi, sdf, dep


def test_grid_stride_every_warp_loops():
    """every stage kernel at >= 3 packs per warp: alpha forward (all packs bit for bit / per element), alpha backward (d_sdf per element,
    d_inv_s over all packs: the per-warp acc_invs), composite forward / backward (all packs), upsample cdf (all packs), inverse cdf on a
    sample of packs p = w + i W over all i (W warps) that covers every loop iteration of its own launch"""
    W, pi, sdf, dep = _big_packs(21)
    P, S = pi.shape[0], sdf.shape[0]
    assert P >= 3 * W
    inv_s = 256.0
    s, inv, a, sel, steps = _alpha_fwd(sdf, pi, inv_s, 0.0)
    r, ratio = _check_alpha_fwd(sdf, pi, inv_s, 0.0, a, sel, steps)
    report("big.alpha_ulps", ratio)
    assert (r["cross"] >= 0).sum() > P // 10
    rng = np.random.default_rng(22)
    g = rng.standard_normal(S).astype(F32)
    g[rng.random(S) < 0.3] = 0
    (a * _cuda(g)).sum().backward()
    want = o64.alpha_backward(sdf, pi, inv_s, g)
    rd = _ratio(s.grad.cpu().numpy() - want["d_sdf"], want["d_sdf_scale"])
    ri = _inv_s_ratio(float(inv.grad), want)
    report("big.d_sdf", rd)
    report("big.d_inv_s", ri)
    assert rd <= C_DSDF and ri <= INV_S_REL, (rd, ri)
    # composite on the kernel's alphas of every pack
    alpha = a.detach().cpu().numpy()
    t, rgb, nab, cot = _composite_inputs(alpha, pi, 23)
    got = _run_composite(alpha, t, pi, rgb, nab, cot, True, 0.0)
    _check_composite(alpha, t, pi, rgb, nab, cot, True, 0.0, got, tag="big.")
    # upsample cdf (same alphas) and the inverse cdf over a warp sample
    from neuralsim_b200.graphics import neus_fused as NF
    cdf = NF.upsample_cdf(_cuda(sdf), _cuda(dep), _cuda(pi), inv_s, False, EPS, 0.0).cpu().numpy()
    wc, sc = o64.upsample_cdf(r["w"], pi)
    rc = _ratio(cdf - wc, sc)
    report("big.cdf_ulps", rc)
    assert rc <= C_CDF, rc
    n_s = 33
    warps = np.array([0, 1, 31, 32, W // 2, W - 1])
    packs = np.concatenate([np.arange(w, P, W) for w in warps])
    stride = 8 * 8 * _sms() * 256                                          # threads of the inverse-cdf launch at the grid-stride limit
    iters = -(-P * n_s // stride)
    hit = np.unique((packs[:, None] * n_s + np.arange(n_s)[None, :]) // stride)
    assert iters >= 3 and np.array_equal(hit, np.arange(iters)), (iters, hit)
    assert all(len(np.arange(w, P, W)) >= 3 for w in warps)
    _check_invert(dep, cdf, pi, n_s, packs)


def test_training_chain_against_float64():
    """compress -> gather -> composite (ray_index) -> backward as one training step runs it (neus_alpha_compact + composite), against
    float64 of the same chain along the kernel's decisions: the image, d_sdf and d_inv_s"""
    from neuralsim_b200.graphics import neus_fused as NF
    kinds = ["cross"] * 40 + ["flat", "rise", "sat", ("drop", 31), ("drop", 0)] * 4
    rng = np.random.default_rng(31)
    lengths = rng.integers(1, 200, len(kinds))
    pi, sdf, dep = _sdf_packs(kinds, lengths, 31)
    P, S = pi.shape[0], sdf.shape[0]
    inv_s = 128.0
    n_rays = 2 * P
    rays_inds = _cuda(np.arange(P, dtype=np.int64) * 2)
    ridx_all = _cuda(np.repeat(np.arange(P), pi[:, 1]).astype(np.int64))
    s = _cuda(sdf).requires_grad_(True)
    inv = torch.tensor(inv_s, device="cuda", requires_grad=True)
    out = NF.neus_alpha_compact(s, inv, _cuda(pi), ridx_all, _cuda(dep), rays_inds, EPS, 0.0)
    K = out["alpha"].shape[0]
    rgb = rng.random((K, 3)).astype(F32)
    cot = dict(g_mask=rng.standard_normal(n_rays), g_depth=rng.standard_normal(n_rays), g_rgb=rng.standard_normal((n_rays, 3)))
    vw, m, d, c, _ = NF.composite(out["alpha"], out["t"], out["pack_infos"], rgb=_cuda(rgb), normalize_depth=True, early_stop_eps=EPS,
                                  ray_index=out["rays_inds_hit"], n_rays=n_rays)
    loss = (m * _cuda(cot["g_mask"].astype(F32))).sum() + (d * _cuda(cot["g_depth"].astype(F32))).sum() + (c * _cuda(cot["g_rgb"].astype(F32))).sum()
    loss.backward()
    # float64 chain along the kernel's decisions
    a_k = out["alpha"].detach().cpu().numpy()
    a_kernel = NF._NeusAlpha.apply(_cuda(sdf), torch.tensor(inv_s, device="cuda"), _cuda(pi), EPS, 0.0)[0]
    rf = o64.replay(a_kernel.cpu().numpy(), pi, EPS, 0.0)
    nidx, pinf = o64.compression(rf["steps"])
    assert np.array_equal(out["nidx"].cpu().numpy(), nidx) and np.array_equal(out["pack_infos"].cpu().numpy(), pinf)
    pidx = np.nonzero(rf["vis"])[0]
    assert np.array_equal(out["pidx"].cpu().numpy(), pidx)
    a64 = o64.neus_alpha(sdf, pi, inv_s)[0]
    vis_k = np.ones(K, bool)
    T64, w64 = o64.transmittance(a64[pidx], vis_k, pinf)
    t_k = dep[pidx].astype(np.float64)
    o = nidx * 2
    fw = o64.composite_forward(w64, t_k, pinf, rgb.astype(np.float64), None, True)
    img = np.zeros(n_rays)
    img[o] = fw["depth"]
    assert np.abs(m.detach().cpu().numpy()[o] - fw["mask"]).max() <= 1e-5
    e_img = float(np.linalg.norm(d.detach().cpu().numpy() - img) / np.linalg.norm(img))
    bw = o64.composite_backward(a64[pidx], t_k, pinf, w64, T64, vis_k, fw["mask"], fw["depth"], rgb=rgb, g_mask=cot["g_mask"][o],
                                g_depth=cot["g_depth"][o], g_rgb=cot["g_rgb"][o])
    ga = np.zeros(S)
    ga[pidx] = bw["d_alpha"]
    want = o64.alpha_backward(sdf, pi, inv_s, ga)
    e_sdf = float(np.linalg.norm(s.grad.cpu().numpy() - want["d_sdf"]) / np.linalg.norm(want["d_sdf"]))
    e_inv = abs(float(inv.grad) - want["d_inv_s"]) / abs(want["d_inv_s"])
    report("chain.depth_rel", e_img)
    report("chain.d_sdf_rel", e_sdf)
    report("chain.d_inv_s_rel", e_inv)
    assert e_img <= CHAIN_REL and e_sdf <= CHAIN_REL and e_inv <= CHAIN_REL, (e_img, e_sdf, e_inv)
    assert a_k.shape[0] == pidx.shape[0]


# ============================================================================================================== count-bound launches
def _bound_call(fn, what, cnt, *args):
    from neuralsim_b200.graphics.neus_static import _call
    _call(fn, what, cnt, 0, None, *args)


def test_count_bound_launches():
    """every stage kernel with a device count below the capacity: packs past the count name an extra, in-range region of samples whose
    cotangents are NaN; the outputs there keep their sentinels, num_steps between count and capacity is zero, and everything else equals
    the count-sized call (bit for bit; d_inv_s to summation order)"""
    from neuralsim_b200 import _lib as L
    lib = L.lib()
    pi_l, sdf_l, dep_l = _ladder_sdf(41)
    n_live, S_live = pi_l.shape[0], sdf_l.shape[0]
    extra_pi, extra_sdf, extra_dep = _sdf_packs(["cross"] * 20, [40] * 20, 42)
    pi = np.concatenate([pi_l, extra_pi + np.array([S_live, 0])])
    sdf, dep = np.concatenate([sdf_l, extra_sdf]), np.concatenate([dep_l, extra_dep])
    P, S = pi.shape[0], sdf.shape[0]
    cnt = torch.zeros(4, dtype=torch.int64, device="cuda")
    cnt[0] = n_live
    P_ = L.ptr
    SENT = -12345.0
    d_sdf_, d_pi, d_dep = _cuda(sdf), _cuda(pi), _cuda(dep)
    inv = torch.tensor([64.0], device="cuda")
    res = {}
    for mode in ("bound", "sized"):
        n_arg = P if mode == "bound" else n_live
        call = (lambda fn, what, *a: _bound_call(fn, what, cnt, *a)) if mode == "bound" else (lambda fn, what, *a: L.check(fn(*a), what))
        alpha = torch.full((S,), SENT, device="cuda")
        selb = torch.full((S,), 7, dtype=torch.uint8, device="cuda")
        steps = torch.full((P,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        call(lib.nsb_neus_alpha_forward, "alpha_fwd", P_(d_sdf_), P_(d_pi), L.c_i64(n_arg), P_(inv), L.c_f32(EPS), L.c_f32(0.0), P_(alpha),
             P_(selb), P_(steps), L.stream_ptr())
        g = torch.randn(S, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
        g[S_live:] = float("nan")
        d_sdf = torch.full((S,), SENT, device="cuda")
        d_inv = torch.zeros(1, device="cuda")
        call(lib.nsb_neus_alpha_backward, "alpha_bwd", P_(d_sdf_), P_(d_pi), L.c_i64(n_arg), P_(inv), P_(g), P_(d_sdf), P_(d_inv), L.stream_ptr())
        cdf = torch.full((S,), SENT, device="cuda")
        call(lib.nsb_neus_upsample_cdf, "cdf", P_(d_sdf_), P_(d_dep), P_(d_pi), L.c_i64(n_arg), L.c_f32(64.0), ctypes.c_int(0), L.c_f32(EPS),
             L.c_f32(0.0), P_(cdf), L.stream_ptr())
        u = torch.linspace(0, 1, 11, device="cuda")[1:-1].contiguous()
        fine = torch.full((P, 9), SENT, device="cuda")
        call(lib.nsb_packed_invert_cdf_shared_u, "invert", P_(d_dep), P_(cdf), P_(u), P_(d_pi), L.c_i64(n_arg), L.c_i32(9), P_(fine), L.stream_ptr())
        a_in = alpha.clone()
        a_in[S_live:] = 0.5
        ray_index = torch.arange(P, device="cuda") * 2
        R = 2 * P
        vw = torch.full((S,), SENT, device="cuda")
        outs = [torch.full((R,), SENT, device="cuda") for _ in range(2)] + [torch.full((R, 3), SENT, device="cuda") for _ in range(2)]
        rgb = torch.rand(S, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
        call(lib.nsb_composite_forward, "comp_fwd", P_(a_in), P_(d_dep), P_(rgb), P_(rgb), P_(d_pi), L.c_i64(n_arg), L.c_f32(EPS), L.c_f32(0.0),
             ctypes.c_int(1), P_(ray_index), P_(vw), *[P_(x) for x in outs], L.stream_ptr())
        gm = [torch.randn(x.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(5 + i)) for i, x in enumerate(outs)]
        for x in gm:
            x[1::2] = float("nan")                                 # odd slots: no live pack writes there
        for x in gm:
            x[2 * n_live:] = float("nan")
        gv = torch.randn(S, device="cuda", generator=torch.Generator("cuda").manual_seed(9))
        gv[S_live:] = float("nan")
        mask_in, depth_in = outs[0].clone(), outs[1].clone()
        d_alpha = torch.full((S,), SENT, device="cuda")
        d_rgb, d_nab = torch.full((S, 3), SENT, device="cuda"), torch.full((S, 3), SENT, device="cuda")
        call(lib.nsb_composite_backward, "comp_bwd", P_(a_in), P_(d_dep), P_(rgb), P_(rgb), P_(vw), P_(d_pi), L.c_i64(n_arg), L.c_f32(EPS),
             L.c_f32(0.0), ctypes.c_int(1), P_(mask_in), P_(depth_in), *[P_(x) for x in gm], P_(gv), P_(ray_index), P_(d_alpha), P_(d_rgb),
             P_(d_nab), L.stream_ptr())
        torch.cuda.synchronize()
        res[mode] = dict(alpha=alpha, sel=selb, steps=steps, d_sdf=d_sdf, d_inv=d_inv, cdf=cdf, fine=fine, vw=vw, mask=outs[0], depth=outs[1],
                         rgb=outs[2], nab=outs[3], d_alpha=d_alpha, d_rgb=d_rgb, d_nab=d_nab)
    b, z = res["bound"], res["sized"]
    assert (b["steps"][n_live:] == 0).all()                            # zero-filled between count and capacity
    for k in ("alpha", "d_sdf", "cdf", "vw", "d_alpha", "d_rgb", "d_nab"):
        assert (b[k][S_live:] == SENT).all(), k
    assert (b["sel"][S_live:] == 7).all() and (b["fine"][n_live:] == SENT).all()
    for k in ("mask", "depth", "rgb", "nab"):
        assert (b[k][2 * n_live:] == SENT).all() and (b[k][1::2] == SENT).all(), k
    for k in ("alpha", "sel", "d_sdf", "cdf", "vw", "d_alpha", "d_rgb", "d_nab"):
        assert torch.equal(b[k][:S_live], z[k][:S_live]), k
    assert torch.equal(b["steps"][:n_live], z["steps"][:n_live]) and torch.equal(b["fine"][:n_live].isnan(), z["fine"][:n_live].isnan())
    live_fine = ~z["fine"][:n_live].isnan()
    assert torch.equal(b["fine"][:n_live][live_fine], z["fine"][:n_live][live_fine])
    for k in ("mask", "depth", "rgb", "nab"):
        assert torch.equal(b[k][:2 * n_live], z[k][:2 * n_live]), k
    e = abs(float(b["d_inv"]) - float(z["d_inv"])) / max(abs(float(z["d_inv"])), 1e-30)
    report("count.d_inv_s_rel", e)
    assert torch.isfinite(b["d_inv"]).all() and e <= 1e-5, e
