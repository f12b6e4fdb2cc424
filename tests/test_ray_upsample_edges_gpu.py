"""The persistent up-sampling kernel (csrc/ray_upsample.cu: k_upsample_persistent) at its capacity, group and tie edges.

Its per-ray bodies warp_upsample_cdf, invert_cdf_one and warp_merge (csrc/neus_device.cuh) are the ones k_upsample_cdf, k_invert_cdf_shared_u
and k_merge_vals call, here on a ray's samples in shared memory or scratch, and its own logic carries state from one 4-ray group to the next
(cur, the p_t / p_sdf / p_cdf pointers, s_n, the ray's scratch slice).  Every case here is checked two ways:
  A  bit for bit against the stage-kernel chain fused_sdf_rays -> upsample_cdf -> sample_cdf_uniform -> merge_sorted_vals (and, with
     sample collection on, the occupancy evidence against the chain's and against OccGridEma.collect_samples on the evaluated points);
  B  per stage against float64 (oracle/neus64.py), teacher-forced on the chain's merged t, sdf and fp32 cdf: the cdf within C_CDF / EST_CDF
     and the kernel's samples within C_INV 2^-24 (|b0| + |b1 - b0|), the bounds of tests/test_neus_stages64_gpu.py.

Inputs are marched samples placed by hand on rays through (or past) the sphere of `make_pair`, so that each ray's length and the index of
its surface crossing are chosen.  Lengths run 0, 1, 2, 31, 32, 33, 127, 128, 129, room - 1, room, room + 1, 192, the scratch limit
long_cap - merged (and one past it), max_steps and the wrapper's long_cap - merged, in groups whose marched lengths sum to 128, 129 and 512
and in groups that mix shared-memory, scratch and flagged rays; room = kCap - (samples of every merged stage).  Stage layouts: [9, 9, 33],
one stage, two stages (an odd number of merges), four stages (kMaxStage) with n_fine 1, 32, 33 and 64, and merged = 191 (room = 1).
Every test asserts from the oracle's replay and inverse-cdf positions that its input reaches the edges it names."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import neus64 as o64
from test_neus_stages64_gpu import C_CDF, C_INV, EPS, EST_CDF
from util import make_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
KCAP, KG, KCTAS_PER_SM = 192, 4, 5            # csrc/ray_upsample.cu
INV_S = 64.0
MAX_STEPS = 4096
SENT, SENT_I = -12345.0, 5

# name -> (n_fine per stage, factor of INV_S per stage); the first factor stays 1 so that the placed crossings keep their lanes
LAYOUTS = {
    "prod": ([9, 9, 33], [1, 4, 16]),
    "one": ([33], [1]),
    "two": ([17, 33], [1, 8]),
    "four": ([1, 32, 64, 33], [1, 2, 4, 16]),
    "room1": ([64, 64, 63, 1], [1, 2, 4, 8]),
}


def report(name, value):
    print(f"METRIC {name} {value:.4g}")


def _ratio(err, scale, floor=1e-30):
    return float((np.abs(err) / (o64.U32 * np.maximum(scale, floor))).max()) if np.size(err) else 0.0


@pytest.fixture(scope="module")
def model(cuda):
    _, m = make_pair(cuda)
    occ = m.accel.occ
    occ.should_collect_samples = True
    occ.register_buffer("_occ_val_grid_pcl", torch.zeros_like(occ.occ_val_grid), persistent=False)
    return m.train()


# ============================================================================================================== inputs
class Rays:
    """hand-placed marched samples: rays_o / rays_d [R, 3], t [M], pack_infos [R, 2], one name per ray"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.o, self.d, self.t, self.n, self.names = [], [], [], [], []

    def _geom(self, h):
        """a ray (origin 3 before its closest approach to the centre, at distance h from it) in a direction near +x"""
        rng = self.rng
        d = np.array([1.0, *rng.uniform(-0.03, 0.03, 2)])
        d /= np.linalg.norm(d)
        a = np.cross(d, [0.0, 0.0, 1.0])
        a /= np.linalg.norm(a)
        b = np.cross(d, a)
        phi = rng.uniform(0, 2 * np.pi)
        return h * (np.cos(phi) * a + np.sin(phi) * b) - 3.0 * d, d

    def add(self, kind, n, name=None):
        """kind: 'hit' (n samples across the surface, random spread), ('cross', K) (K + 1 samples 0.4 .. 0.2 outside the surface, the rest
        0.2 .. 0.4 inside: at inv_s 64 T falls below eps at sample K), 'miss' (passes 0.35 from the surface: every alpha is 0), 'dup'
        (samples across the surface with two t values repeated: zero-weight interior bins), 'empty' (n = 0)"""
        rng = self.rng
        h = 0.85 if kind == "miss" else rng.uniform(0.0, 0.25 if kind == "hit" else 0.1)
        t_in = 3.0 - np.sqrt(max(0.25 - h * h, 0.0))
        if kind == "empty":
            t = np.zeros(0)
        elif kind == "miss":
            t = np.sort(rng.uniform(3.0 - 0.85, 3.0 + 0.85, n))
        elif kind == "hit":
            t = np.sort(rng.uniform(t_in - rng.uniform(0.03, 0.4), t_in + rng.uniform(0.03, 0.4), n))
        elif kind == "dup":
            base = np.linspace(t_in - 0.12, t_in + 0.12, n - 4)
            m = base.shape[0] // 2
            t = np.sort(np.concatenate([base, np.repeat(base[m - 3], 2), np.repeat(base[m + 2], 2)]))
        else:
            K = kind[1]
            assert n >= K + 2
            t = np.concatenate([np.linspace(t_in - 0.4, t_in - 0.2, K + 1), np.linspace(t_in + 0.2, t_in + 0.4, n - K - 1)])
        o, d = self._geom(h)
        self.o.append(o)
        self.d.append(d)
        self.t.append(t.astype(F32))
        self.n.append(int(n))
        self.names.append(name)
        return len(self.n) - 1

    def tensors(self):
        n = np.asarray(self.n, np.int64)
        pi = np.stack([np.cumsum(n) - n, n], 1)
        t = np.concatenate(self.t).astype(F32) if n.sum() else np.zeros(0, F32)
        c = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x)).cuda() if dt is None else torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()
        return dict(o=c(np.stack(self.o), F32), d=c(np.stack(self.d), F32), t=c(t), pi=c(pi), n=n, ridx_hit=c(np.arange(len(n), dtype=np.int64)))

    def index(self, name):
        return self.names.index(name)


def _sub(rt, rows):
    """the rays `rows` of a ray set as their own pack list (the chain is run on the rays the kernel works on)"""
    rows = torch.as_tensor(rows, dtype=torch.int64, device="cuda")
    pi = rt["pi"][rows]
    ridx = torch.repeat_interleave(rows, pi[:, 1])
    off = torch.repeat_interleave(pi[:, 0], pi[:, 1])
    pos = torch.arange(ridx.shape[0], device="cuda") - torch.repeat_interleave(torch.cumsum(pi[:, 1], 0) - pi[:, 1], pi[:, 1])
    t = rt["t"][off + pos].contiguous()
    npi = torch.stack([torch.cumsum(pi[:, 1], 0) - pi[:, 1], pi[:, 1]], 1).contiguous()
    return dict(ridx_hit=rows.contiguous(), ridx=ridx.contiguous(), t=t, pi=npi)


# ============================================================================================================== the two computations
def _chain(surf, rt, rows, layout, *, ml, est, thre, collect=None):
    """the stage kernels on the rays `rows`: -> (fine [len(rows), sum n_fine], per stage (t, sdf, pack_infos, cdf), sdf of the marched
    samples, [new samples, their sdf] of every merged stage)"""
    from neuralsim_b200.graphics import neus_fused as NF
    nf, fac = LAYOUTS[layout]
    s = _sub(rt, rows)
    o, d = rt["o"], rt["d"]
    sdf = surf.fused_sdf_rays(s["ridx"], s["t"], o, d, max_level=ml, collect=collect)
    sdf0 = sdf
    depth, pi, stages, per_stage, fine_pts = s["t"], s["pi"], [], [], []
    for i in range(len(nf)):
        cdf = NF.upsample_cdf(sdf, depth, pi, INV_S * fac[i], est, EPS, thre)
        fine = NF.sample_cdf_uniform(depth, cdf, pi, nf[i])
        per_stage.append((depth, sdf, pi, cdf))
        stages.append(fine)
        if i + 1 < len(nf):
            sdf_f = surf.fused_sdf_rays(s["ridx_hit"], fine, o, d, max_level=ml, collect=collect).contiguous()
            fine_pts.append((fine, sdf_f))
            depth, sdf, pi = NF.merge_sorted_vals(depth, sdf, pi, fine, sdf_f)
    return torch.cat(stages, -1), per_stage, (s, sdf0), fine_pts


def _kernel(surf, rt, layout, *, ml, est, thre, entry, long_cap=None, count=None, collect=None):
    """k_upsample_persistent through the C ABI into sentinel-filled buffers.  entry: 'persistent' (nsb_upsample_persistent, no scratch),
    'abi' (nsb_upsample_rays with an explicit long_cap, optionally a device count and collection) or 'wrapper' (graphics.neus_fused.upsample_rays:
    long_cap sized from max_steps).  -> (fine_all, overflow)"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics import neus_fused as NF
    nf, fac = LAYOUTS[layout]
    grid16, dec = surf._fused_state()
    if entry == "wrapper":
        return NF.upsample_rays(surf.encoding.meta, grid16, dec, rt["ridx_hit"], rt["pi"], rt["t"], rt["o"], rt["d"], [INV_S * f for f in fac], nf,
                                max_level=ml, max_steps=MAX_STEPS, use_estimate_alpha=est, early_stop_eps=EPS, alpha_thre=thre, collect=collect)
    lib = L.lib()
    n_hit, S = rt["n"].shape[0], len(nf)
    us = [NF._quantiles(n, torch.device("cuda")) for n in nf]
    fine = torch.full((n_hit, sum(nf)), SENT, device="cuda")
    ovf = torch.full((n_hit,), SENT_I, dtype=torch.int32, device="cuda")
    P = L.ptr
    args = (surf.encoding.meta.c_ref, P(grid16, "f16"), ctypes.byref(dec), P(rt["o"], "f32"), P(rt["d"], "f32"), P(rt["t"], "f32"), P(rt["pi"], "i64"),
            P(rt["ridx_hit"], "i64"), L.c_i64(n_hit), L.c_i32(ml), L.c_i32(S), (ctypes.c_int32 * S)(*nf), (ctypes.c_float * S)(*[INV_S * f for f in fac]),
            (ctypes.c_void_p * S)(*[u.data_ptr() for u in us]), L.c_i32(int(est)), L.c_f32(EPS), L.c_f32(thre), P(fine), P(ovf))
    if entry == "persistent":
        L.check(lib.nsb_upsample_persistent(*args, L.stream_ptr()), "upsample_persistent")
    else:
        lib.nsb_upsample_rays_scratch_floats.restype = ctypes.c_int64
        scratch = torch.empty(int(lib.nsb_upsample_rays_scratch_floats(L.c_i64(n_hit), L.c_i32(long_cap))), device="cuda")
        cnt = None
        if count is not None:
            cnt = torch.tensor([count], dtype=torch.int64, device="cuda")
            lib.nsb_bind_device_counts(ctypes.c_void_p(cnt.data_ptr()), None)
        L.check(lib.nsb_upsample_rays(*args, P(scratch), L.c_i32(long_cap), ctypes.byref(collect) if collect is not None else None, L.stream_ptr()),
                "upsample_rays")
    torch.cuda.synchronize()
    return fine, ovf


def _float64(surf, per_stage, fine_rows, layout, *, est, thre, sel=None, tag=""):
    """reference B: for every stage, float64 alphas / replay / cdf on the chain's merged t and sdf, and float64 inverse-cdf samples on the
    chain's fp32 cdf, against the kernel's samples `fine_rows` [rows of the chain].  -> per stage dict(r (replay), a (fp32 alphas), pos
    [sel, n_fine] (bins of the inverse cdf), cdf, t, pi) for the census"""
    from neuralsim_b200.graphics import neus_fused as NF
    nf, fac = LAYOUTS[layout]
    got_all = fine_rows.cpu().numpy()
    out, off = [], 0
    for i, (dep_t, sdf_t, pi_t, cdf_t) in enumerate(per_stage):
        dep, sdf, pi, cdf = (x.cpu().numpy() for x in (dep_t, sdf_t, pi_t, cdf_t))
        inv_s = INV_S * fac[i]
        cov = o64.pack_of(pi, sdf.shape[0]) >= 0
        if est:
            a64 = o64.upsample_alpha(sdf, dep, pi, inv_s)
            r = o64.replay(a64.astype(F32), pi, EPS, thre)
            _, w64 = o64.transmittance(a64, r["vis"], pi)
            want, _ = o64.upsample_cdf(w64, pi)
            # EST_CDF (measured at inv_s 64) grows with inv_s (the rounding of the fp32 sigmoid argument); and each fp32 sigmoid near 1 is
            # rounded by up to 2^-25, so alpha_k carries up to 2^-24 absolute (fp32 rounds both sigmoids of a far-outside interval to 1:
            # alpha 0), summed over the samples before k and divided by the norm (its 1e-5 floor on rays that miss the surface)
            pk = np.maximum(o64.pack_of(pi, sdf.shape[0]), 0)
            k1 = np.arange(sdf.shape[0]) - pi[pk, 0] + 1                                 # samples up to and including k
            w_pack = np.bincount(pk[cov], weights=w64[cov], minlength=pi.shape[0])
            w_last = np.where(pi[:, 1] > 0, w64[np.maximum(pi[:, 0] + pi[:, 1] - 1, 0)], 0.0)
            norm = np.maximum(w_pack - w_last, 1e-5)[pk]                                 # max(last exclusive cdf, 1e-5)
            bound = EST_CDF * max(1.0, inv_s / 64.0) + 2 * o64.U32 * k1 / norm
            ratio = float((np.abs(cdf - want) / bound)[cov].max()) if cov.any() else 0.0
            report(f"{tag}cdf_est_over_bound[{i}]", ratio)
            assert ratio <= 1.0, (i, ratio)
        else:
            a64 = o64.neus_alpha(sdf, pi, inv_s)[0]
            a32 = NF._NeusAlpha.apply(sdf_t, torch.tensor(inv_s, device="cuda"), pi_t, EPS, thre)[0].cpu().numpy()
            r = o64.replay(a32, pi, EPS, thre)
            want, scale = o64.upsample_cdf(r["w"], pi)
            ratio = _ratio((cdf - want)[cov], scale[cov])
            report(f"{tag}cdf_ulps[{i}]", ratio)
            assert ratio <= C_CDF, (i, ratio)
        rows = np.arange(pi.shape[0]) if sel is None else np.asarray(sel)
        u = np.linspace(0, 1, nf[i] + 2, dtype=F32)[1:-1]
        want_s, scale_s, pos = o64.invert_cdf(dep, cdf, u, pi[rows], return_pos=True)
        got = got_all[rows, off:off + nf[i]]
        ratio = _ratio(got - want_s, scale_s)
        report(f"{tag}invert_ulps[{i}]", ratio)
        assert ratio <= C_INV, (i, ratio)
        out.append(dict(r=r, a=a64, pos=pos, rows=rows, cdf=cdf, t=dep, pi=pi))       # (k_neus_alpha_fwd zeroes alphas after the stop)
        off += nf[i]
    return out


# ============================================================================================================== census helpers
def _lane_of_cross(st, p):
    return int(st[0]["r"]["cross"][p])


def _pmf_at(st, p):
    """(pos, pmf) of the stage-0 inverse-cdf samples of pack p (the float64 check ran on every pack)"""
    pi, cdf = st[0]["pi"], st[0]["cdf"]
    b = pi[p, 0]
    pos = st[0]["pos"][p]
    c1 = cdf[b + pos]
    c0 = np.where(pos > 0, cdf[b + np.maximum(pos - 1, 0)], F32(0))
    return pos, (c1 - c0).astype(F32)


def _ties(chain_fine, per_stage, layout):
    """new samples of each merged stage equal to an existing sample of their ray (the merge's upper / lower bound decides their order)"""
    nf, _ = LAYOUTS[layout]
    fine = chain_fine.cpu().numpy()
    ties, off = 0, 0
    for i in range(len(nf) - 1):
        dep, pi = per_stage[i][0].cpu().numpy(), per_stage[i][2].cpu().numpy()
        for p, (b, n) in enumerate(pi):
            ties += int(np.isin(fine[p, off:off + nf[i]], dep[b:b + n]).sum())
        off += nf[i]
    return ties


# ============================================================================================================== the ladder
CASES = [("prod", True, 0.0, None), ("prod", False, 0.01, 7), ("one", True, 0.01, None), ("two", False, 0.0, None), ("two", True, 0.01, 7),
         ("four", True, 0.0, 7), ("room1", False, 0.01, None), ("room1", True, 0.0, None)]


def _ladder(layout, seed, tail):
    """one ray set per layout: the length ladder, the numeric edges, the composed groups; `tail` extra rays set n_hit % 4"""
    nf, _ = LAYOUTS[layout]
    merged = sum(nf[:-1])
    room = KCAP - merged
    cap = merged + 300                              # the explicit long_cap of the 'abi' entry: scratch rays up to 300 marched samples
    R = Rays(seed)
    for n in (32, 32, 32, 32, 32, 32, 32, 33):     # groups 0, 1: marched lengths sum to 128 (one full tile) and 129
        R.add("hit", n)
    for _ in range(4):                              # group 2: 512
        R.add("hit", 128)
    R.add("hit", min(40, room), "g3_smem")          # group 3: shared memory, scratch, flagged (abi entry), and n = 2
    R.add("hit", min(room + 1, 300), "g3_scratch")
    R.add("hit", 301, "g3_flag")
    R.add("hit", 2)
    R.add("hit", 300, "cap_fits")                   # group 4: exactly the abi scratch limit, an empty pack, a miss, n = 1
    R.add("empty", 0, "empty")
    R.add("miss", 40, "miss40")
    R.add("hit", 1, "n1")
    R.add(("cross", 0), 40, "cross0")
    R.add(("cross", 31), 52, "cross31")
    R.add(("cross", 32), 43, "cross32")
    R.add("miss", 1, "miss1")
    R.add("miss", 2, "miss2")
    R.add("miss", 200, "miss200")
    R.add("dup", 40, "dup40")
    R.add("dup", 90, "dup90")
    R.add("hit", 1, "n1b")
    for n in (1, 2, 31, 32, 33, 127, 128, 129, room - 1, room, room + 1, 192):
        if n >= 1:
            R.add("hit", n, f"len{n}")
    R.add("hit", MAX_STEPS, "max_steps")
    R.add("hit", MAX_STEPS + 64, "wrapper_cap")     # the wrapper's long_cap - merged
    while (len(R.n) % 4) != tail % 4:
        R.add("hit", int(R.rng.integers(1, 60)))
    return R, room, cap


@pytest.mark.parametrize("layout,est,thre,max_level", CASES)
def test_ladder_against_stage_kernels_and_float64(model, layout, est, thre, max_level):
    surf = model.implicit_surface
    ml = surf._ml(max_level)
    ci = CASES.index((layout, est, thre, max_level))
    R, room, cap = _ladder(layout, 100 + ci, 1 + ci % 3)
    nf, _ = LAYOUTS[layout]
    merged = sum(nf[:-1])
    # rays past the device count: long enough to be flagged if the count were ignored
    n_live = len(R.n)
    for _ in range(5):
        R.add("hit", cap - merged + 7)
    rt_all = R.tensors()
    live = np.arange(n_live)
    rt = {k: (v[:n_live] if k in ("o", "d", "n", "ridx_hit") else v) for k, v in rt_all.items()}
    rt["pi"] = rt_all["pi"][:n_live].contiguous()
    n = rt["n"]
    nonempty = live[n > 0]
    with torch.no_grad():
        ref, per_stage, _, _ = _chain(surf, rt, nonempty, layout, ml=ml, est=est, thre=thre)
        got_w, ovf_w = _kernel(surf, rt, layout, ml=ml, est=est, thre=thre, entry="wrapper")
        got_p, ovf_p = _kernel(surf, rt, layout, ml=ml, est=est, thre=thre, entry="persistent")
        got_a, ovf_a = _kernel(surf, rt_all, layout, ml=ml, est=est, thre=thre, entry="abi", long_cap=cap, count=n_live)
    ne = torch.as_tensor(nonempty, device="cuda")
    # --- A: the wrapper (long_cap from max_steps): every ray fits, every row equals the chain
    assert int(ovf_w.sum()) == 0
    assert torch.equal(got_w[ne], ref)
    # --- A: no scratch: exactly the rays beyond the shared-memory room are flagged; their rows and the empty pack's row are not written
    flag_p = n > room
    assert np.array_equal(ovf_p.cpu().numpy(), np.where(flag_p, 1, SENT_I)) and flag_p.any() and (n == room + 1).any()
    keep = nonempty[~flag_p[nonempty]]
    pos_in_chain = {r: k for k, r in enumerate(nonempty)}
    kc = torch.as_tensor([pos_in_chain[r] for r in keep], device="cuda")
    assert torch.equal(got_p[torch.as_tensor(keep, device="cuda")], ref[kc])
    untouched = torch.as_tensor(live[flag_p | (n == 0)], device="cuda")
    assert bool((got_p[untouched] == SENT).all())
    # --- A: explicit long_cap and a device count: rays beyond long_cap - merged are flagged, the rest (scratch or not) equal the chain;
    # the rows and overflow entries past the count keep their sentinels
    flag_a = n > cap - merged
    ovf_a = ovf_a.cpu().numpy()
    assert np.array_equal(ovf_a[:n_live], np.where(flag_a, 1, SENT_I)) and (ovf_a[n_live:] == SENT_I).all()
    assert (n == cap - merged).any() and (n == cap - merged + 1).any()
    keep = nonempty[~flag_a[nonempty]]
    kc = torch.as_tensor([pos_in_chain[r] for r in keep], device="cuda")
    assert torch.equal(got_a[torch.as_tensor(keep, device="cuda")], ref[kc])
    assert bool((got_a[torch.as_tensor(live[flag_a | (n == 0)], device="cuda")] == SENT).all()) and bool((got_a[n_live:] == SENT).all())
    # --- B: float64 per stage on every ray the chain ran
    st = _float64(surf, per_stage, got_w[ne], layout, est=est, thre=thre, tag=f"{layout}.")
    # --- census: the input reaches every edge this test names
    assert len(R.n) - 5 == n_live and n_live % 4 == 1 + ci % 3                 # a partial last group
    assert {1, 2, 31, 32, 33, 127, 128, 129, room, room + 1, 192, MAX_STEPS, MAX_STEPS + 64} <= set(n.tolist())
    assert room - 1 < 1 or room - 1 in set(n.tolist())
    sums = n[:4 * (n_live // 4)].reshape(-1, 4).sum(1)
    assert {128, 129, 512} <= set(sums.tolist())
    g3 = R.index("g3_smem") // 4
    kinds = ["smem" if m <= room else ("scratch" if m <= cap - merged else "flag") for m in n[4 * g3:4 * g3 + 4]]
    assert {"smem", "scratch", "flag"} <= set(kinds), kinds
    row = lambda name: pos_in_chain[R.index(name)]
    for K in (0, 31, 32):
        assert _lane_of_cross(st, row(f"cross{K}")) == K, (K, st[0]["r"]["cross"][row(f"cross{K}")])
    p = row("cross31")
    b = st[0]["pi"][p, 0]
    assert (st[0]["a"][b + 32:b + st[0]["pi"][p, 1]] > thre).any()            # live samples in the chunk after the crossing
    for name in ("miss1", "miss2", "miss40", "miss200"):
        p = row(name)
        b, m = st[0]["pi"][p]
        assert (st[0]["cdf"][b:b + m] == 0).all()                               # every fp32 weight 0: the norm at its 1e-5 floor
        assert est or (st[0]["r"]["w"][b:b + m] == 0).all()                      # (the replay of est runs on float64 alphas)
        pos, pmf = _pmf_at(st, p)
        assert (pos == m - 1).all() and (m == 1 or (pmf < 1e-5).all())
    for name in ("n1", "n1b", "miss1"):
        assert (st[0]["pos"][row(name)] == 0).all()
    for name in ("dup40", "dup90"):
        p = row(name)
        b, m = st[0]["pi"][p]
        t, c, vis = st[0]["t"][b:b + m], st[0]["cdf"][b:b + m], st[0]["r"]["vis"][b:b + m]
        assert (np.diff(t) == 0).sum() >= 2                                      # duplicate marched t
        # an interior flat stretch: two unvisited (zero-weight) samples between live ones (flat to the warp scan's rounding: each lane
        # sums its prefix in its own order)
        flat = ~vis[1:-1] & ~vis[2:] & (c[1:-1] > 0.01) & (c[2:] < 0.99)
        assert flat.any()
    if len(nf) > 1:
        assert _ties(ref, per_stage, layout) > 0


# ============================================================================================================== grid-stride groups
@pytest.mark.parametrize("layout,est,thre", [("prod", True, 0.0), ("two", False, 0.01)])
def test_every_cta_runs_three_groups_with_collection(model, layout, est, thre):
    """n_hit >= 3 grid 4: every CTA runs >= 3 groups, and one CTA's warp slots go scratch -> scratch (shorter: stale data past it) -> shared
    memory and scratch -> shared memory -> scratch; two scratch rays share a group; empty packs and flagged rays sit in later groups of many
    CTAs.  Sample collection on: the evidence equals the chain's and OccGridEma.collect_samples on the evaluated points."""
    surf = model.implicit_surface
    occ = model.accel.occ
    ml = surf._ml(None)
    nf, _ = LAYOUTS[layout]
    merged = sum(nf[:-1])
    room = KCAP - merged
    cap = merged + 320
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = KCTAS_PER_SM * sms
    n_hit = 3 * grid * KG + 2
    b = 1
    special = {
        4 * b + 0: ("hit", 300), 4 * b + 1: ("empty", 0), 4 * b + 2: ("hit", 260), 4 * b + 3: ("hit", 20),
        4 * (b + grid) + 0: ("hit", 220), 4 * (b + grid) + 1: ("hit", cap - merged + 1), 4 * (b + grid) + 2: ("hit", 40), 4 * (b + grid) + 3: ("miss", 30),
        4 * (b + 2 * grid) + 0: ("hit", 40), 4 * (b + 2 * grid) + 1: ("hit", 20), 4 * (b + 2 * grid) + 2: ("hit", 200), 4 * (b + 2 * grid) + 3: ("empty", 0),
    }
    for c in range(3, grid, 7):
        special[4 * (c + grid) + 3] = ("empty", 0)
        special[4 * (c + 2 * grid) + 1] = ("hit", cap - merged + 1)
    R = Rays(7 + len(nf))
    for j in range(n_hit):
        kind, m = special.get(j, (None, None))
        if kind is None:
            u = R.rng.random()
            kind, m = ("miss", int(R.rng.integers(1, 40))) if u < 0.1 else (("dup", int(R.rng.integers(12, 48))) if u < 0.15 else ("hit", int(R.rng.integers(1, 48))))
        R.add(kind, m)
    rt = R.tensors()
    n = rt["n"]
    flag = n > cap - merged
    valid = np.nonzero((n > 0) & ~flag)[0]
    with torch.no_grad():
        coll = occ.collect_struct()
        assert coll is not None
        occ._occ_val_grid_pcl.zero_()
        ref, per_stage, (s0, sdf0), fine_pts = _chain(surf, rt, valid, layout, ml=ml, est=est, thre=thre, collect=coll)
        pcl_chain = occ._occ_val_grid_pcl.clone()
        occ._occ_val_grid_pcl.zero_()
        got, ovf = _kernel(surf, rt, layout, ml=ml, est=est, thre=thre, entry="abi", long_cap=cap, collect=coll)
        pcl_kernel = occ._occ_val_grid_pcl.clone()
        # the points the kernel evaluated, through the torch restatement of the collection
        occ._occ_val_grid_pcl.zero_()
        o, d = rt["o"], rt["d"]
        pts = [torch.addcmul(o[s0["ridx"]], d[s0["ridx"]], s0["t"][:, None])]
        vals = [sdf0]
        for fine, sdf_f in fine_pts:
            r = s0["ridx_hit"][:, None].expand(fine.shape).reshape(-1)
            pts.append(torch.addcmul(o[r], d[r], fine.reshape(-1)[:, None]))
            vals.append(sdf_f.reshape(-1))
        occ.collect_samples(torch.cat(pts), val=torch.cat(vals))
        pcl_points = occ._occ_val_grid_pcl.clone()
        occ._occ_val_grid_pcl.zero_()
    assert np.array_equal(ovf.cpu().numpy(), np.where(flag, 1, SENT_I))
    vt = torch.as_tensor(valid, device="cuda")
    assert torch.equal(got[vt], ref)
    assert bool((got[torch.as_tensor(np.nonzero((n == 0) | flag)[0], device="cuda")] == SENT).all())
    assert float(pcl_chain.max()) > 0 and torch.equal(pcl_kernel, pcl_chain) and torch.equal(pcl_kernel, pcl_points)
    # float64 on the special CTA's rows and a sample of the others
    rows_b = [k for k, r in enumerate(valid) if (r // 4) % grid == b]
    sel = np.unique(np.concatenate([rows_b, np.arange(0, valid.shape[0], 41)]))
    _float64(surf, per_stage, got[vt], layout, est=est, thre=thre, sel=sel, tag=f"grid.{layout}.")
    # census: every CTA runs >= 3 groups; the special slots are what their names say
    groups = -(-n_hit // KG)
    assert groups >= 3 * grid and grid == min(groups, KCTAS_PER_SM * sms)
    where = lambda j: "empty" if n[j] == 0 else ("smem" if n[j] <= room else ("scratch" if n[j] <= cap - merged else "flag"))
    slots = [[where(4 * (b + k * grid) + w) for k in range(3)] for w in range(KG)]
    assert slots[0] == ["scratch", "scratch", "smem"] and n[4 * b] > n[4 * (b + grid)]
    assert slots[2] == ["scratch", "smem", "scratch"] and slots[1] == ["empty", "flag", "smem"]
    assert flag.sum() > grid // 7 and (n == 0).sum() > grid // 7 and n_hit % KG == 2
