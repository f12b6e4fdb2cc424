"""The warp-merged table-gradient scatter of k_sdf_bwd_tc (csrc/fused_tc.cu) and k_color_sdf_bwd (csrc/color_tc.cu) against the float64
reference (oracle/fused64.py) and against the kernels themselves in an order where nothing merges.

warp_merge_updates (csrc/lotd_device.cuh) sums the updates of consecutive lanes whose points lie in the same cell of a level
(resolution <= 1024 per axis) with a segmented shuffle scan, and only a run's first lane issues the 8 reductions; with more than
24 run heads in a warp every lane issues its own.  It runs only where neighbouring lanes share cells: on samples in ray order, as
the training step produces them.  The inputs here are such samples (marched steps and boundary-query patterns, packs that cross warp
and tile boundaries), the same points shuffled (the no-merge reference), and hand-built warps with the run structures at the edges of
the merge (one run, 32 heads, 24 and 25 heads, a run that starts at lane 31, A A B A A keys, zero cotangents on a head and inside a
run).  Every test asserts with tests/util.py:merge_census that its inputs do (or do not) exercise the merge, so an edit to the inputs
cannot silently stop covering it.  The graph step's calls are covered too: nsb_fused_sdf_bwd_indexed over a device-built keep list,
and the backward and colour kernels under a device-resident count smaller than their capacity (tests/test_wide_scatter_gpu.py runs the
same bodies on the 17-level street table, the 48-column kernels).

The table gradient is compared per level (a whole-table rel-L2 lets the dominant levels hide one level).  Bounds are about 3x the
errors measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); DESIGN.md §4 lists them."""
import ctypes

import numpy as np
import pytest
import torch

import test_tc_kernels_gpu as tk
from oracle import fused64, lotd as olotd
from util import MERGE_MAX_HEADS, merge_census

pytestmark = pytest.mark.gpu

CFG = olotd.gen_ngp_cfg()
META = olotd.LoDMeta(3, **CFG)
CASES = [tk.PRODUCTION, ((64, 64, 4), 7)]
CASE_IDS = [f"w{c[0]}-r{c[1]}-a{c[2]}-ml{m}" for c, m in CASES]
SDF_KEYS = ("grid", "W1", "b1", "W2", "b2")
MID_LEVEL = 5                     # the mid level whose run structure the hand-built warps fix besides level 0 (res 80, dense)

# Bounds (rel-L2).  Table gradient per level against float64 on ray-ordered inputs, every cotangent or ~30 % zero (the other gradients
# keep tk.BWD_REL);
LEVEL_REL = 1e-4                    # measured <= 3.1e-5
# one hand-built warp (32 points) against float64: a single fp16 value of one point that rounds the other way is a larger share of a
# 32-point sum than of a tile's (the other gradients keep tk.TILE_REL)
HAND_REL = 4.5e-4                   # measured <= 1.4e-4 (k_color_sdf_bwd, head_at_31), all others <= 1.9e-5
# the kernel against itself (shuffled order, no-merge layout, count-bound call): only the fp32 summation order differs
ORDER_LEVEL_REL = 1.5e-6            # table gradient per level, measured <= 4.5e-7
ORDER_REL = 3e-6                    # every other gradient, measured <= 9.2e-7


# ===================================================================================================================== inputs
def _slab(o, d, lim):
    """entry and exit t of the ray o + d t through [-lim, lim]^3"""
    with np.errstate(divide="ignore"):
        a, b = (-lim - o) / d, (lim - o) / d
    return float(np.minimum(a, b).max()), float(np.maximum(a, b).min())


def _ray_samples(n, n_appear, seed):
    """n samples of a few hundred rays through the box, in ray order with t ascending: rays alternate between marched samples
    (step 0.005) and a boundary-query pattern (65 coarse samples + 64 fine samples clustered around a surface).  No pack length is a
    multiple of 32.  The last ray ends with 5 samples in [0, 1e-4]^3, the cell of table-space 0.5 that an invalid lane (x = 0) loads."""
    rng = np.random.default_rng(seed)
    os_, ds, ts = [], [], []
    total = 0
    while True:
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        o = rng.uniform(-0.6, 0.6, 3) - 2.5 * d
        t0, t1 = _slab(o, d, 0.995)
        if len(ts) % 2 == 0:
            t = t0 + rng.uniform(0, 0.005) + np.arange(int((t1 - t0) / 0.005)) * 0.005
        else:
            ts_ = rng.uniform(t0 + 0.2 * (t1 - t0), t1 - 0.2 * (t1 - t0))
            t = np.sort(np.concatenate([np.linspace(t0, t1, 65), np.clip(ts_ + rng.normal(0, 0.004, 64), t0, t1)]))
        if len(t) % 32 == 0:
            t = t[:-1]
        if total + len(t) > n - 150:
            break
        os_.append(o), ds.append(d), ts.append(t)
        total += len(t)
    m = n - total
    if m % 32 == 0:                       # shorten a ray whose length then stays off a multiple of 32
        j = next(j for j, t in enumerate(ts) if len(t) % 32 != 1)
        ts[j] = ts[j][:-1]
        m += 1
    d = np.abs(rng.normal(size=3)) + 0.2
    d /= np.linalg.norm(d)
    step = 0.9 / (d.max() * m)
    os_.append(-2.5 * d), ds.append(d)
    ts.append(np.concatenate([2.5 - step * np.arange(m - 5, 0, -1), 2.5 + 5e-6 + 2e-5 * np.arange(5)]))
    lens = np.array([len(t) for t in ts])
    assert lens.sum() == n and (lens % 32 != 0).all()
    o = torch.tensor(np.stack(os_), dtype=torch.float32)
    d = torch.tensor(np.stack(ds), dtype=torch.float32)
    t = torch.tensor(np.concatenate(ts), dtype=torch.float32)
    ridx = torch.from_numpy(np.repeat(np.arange(len(ts)), lens))
    x = (d.double()[ridx] * t.double()[:, None] + o.double()[ridx]).float()        # the kernels' fma(d, t, o)
    assert float(x.abs().max()) < 1.0 and (x[-5:] >= 0).all() and (x[-5:] <= 1e-4).all()
    g = torch.Generator().manual_seed(seed)
    ha = torch.randn(len(ts), n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    # ~30 % zero cotangents: runs of 2..16 samples and isolated ones
    zero = torch.rand(n, generator=g) < 0.1
    for s in np.flatnonzero(rng.random(n) < 0.025):
        zero[s:s + rng.integers(2, 17)] = True
    return dict(x=x, o=o, d=d, t=t, ridx=ridx, v=d.clone(), ha=ha, cot=cot, zero=zero, perm=torch.from_numpy(rng.permutation(n)))


_CACHE = {}


def _case(case):
    """model, ray-ordered inputs and float64 reference for one configuration (built once)"""
    if case not in _CACHE:
        (width, rw, n_appear), max_level = case
        full = case == tk.PRODUCTION
        n = tk._size("color_fwd", 3 if full else 2)
        model = tk._model(width, rw, n_appear, seed=width + 3 * rw + n_appear + 1)
        model.max_level = max_level
        inp = _ray_samples(n, n_appear, seed=17 if full else 23)
        ref = fused64.Fused64.from_model(model, max_level=max_level)
        for k in [k for k in _CACHE if k != tk.PRODUCTION]:
            del _CACHE[k]
        _CACHE[case] = dict(model=model, inp=inp, ref=ref)
    return _CACHE[case]


def _color_fwd64(c):
    if "fwd" not in c:
        inp = c["inp"]
        c["fwd"] = c["ref"].color_forward(inp["x"].numpy(), inp["v"][inp["ridx"]].numpy(), inp["ha"][inp["ridx"]].numpy())
    return c["fwd"]


def _masked(cot, zero):
    keep = (~zero).float()
    return tuple(v * keep.view(-1, *[1] * (v.dim() - 1)) for v in cot)


def _assert_ray_order_merges(x, max_level=None):
    """census of the ray order: the merge runs on most warps of the coarse levels, somewhere on every level 5..12, and some warps are
    one run on level 0"""
    c = merge_census(x, CFG, max_level=max_level)
    frac = (c["heads"] <= MERGE_MAX_HEADS).mean(0)
    print("METRIC census ray order: fraction of warps that merge per level "
          + " ".join(f"L{l}={f:.2f}" for l, f, m in zip(c["levels"], frac, c["mergeable"]) if m))
    assert (frac[:5] >= 0.5).all(), frac
    assert all(frac[l] > 0 for l in range(5, min(12, c["levels"][-1]) + 1)), frac
    assert (c["heads"][:, 0] == 1).any()
    assert not c["mergeable"][13:].any() and frac[c["mergeable"]].min() > 0
    # the last valid lanes share every cell with the invalid lanes (x = 0) after them
    n = x.shape[0]
    if n % 32:
        for cell in c["cells"]:
            assert (cell[n - 1] == cell[n:]).all()


def _assert_no_merge(x, order):
    c = merge_census(x, CFG, order=order)
    assert (c["heads"] > MERGE_MAX_HEADS).all(), int(c["heads"].min())


# ===================================================================================================================== kernel calls
def _sdf_bwd(model, max_level, d_sdf, *, x=None, rays=None, keep=None, n=None, count=None):
    """nsb_fused_sdf_bwd_indexed over n work items (default: all of d_sdf): points x, or rays = (o, d, ridx, t); keep: optional index
    list; count = (cnt, slot): bind the device-resident count cnt[slot] (the graph step's call)"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.neus_static import _call
    s = model.implicit_surface
    grid16, dec = s._fused_state()
    p = tk._params(model)
    g = {k: torch.zeros(p[k].shape, dtype=torch.float32, device="cuda") for k in SDF_KEYS}
    if x is not None:
        src = (L.ptr(x, "f32"), None, None, None, None)
    else:
        o, d, ridx, t = rays
        src = (None, L.ptr(o, "f32"), L.ptr(d, "f32"), L.ptr(ridx, "i64"), L.ptr(t, "f32"))
    n = d_sdf.shape[0] if n is None else n
    args = (s.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), *src, L.ptr(d_sdf, "f32"), L.ptr(keep, "i64", allow_none=True),
            L.c_i64(n), L.c_i32(s._ml(max_level)), *[L.ptr(g[k]) for k in SDF_KEYS], L.stream_ptr())
    if count is None:
        L.check(L.lib().nsb_fused_sdf_bwd_indexed(*args), "fused_sdf_bwd")
    else:
        _call(L.lib().nsb_fused_sdf_bwd_indexed, "fused_sdf_bwd", count[0], count[1], None, *args)
    return g


def _rays_cuda(inp, perm=None):
    ridx, t = (inp["ridx"], inp["t"]) if perm is None else (inp["ridx"][perm], inp["t"][perm])
    return inp["o"].cuda(), inp["d"].cuda(), ridx.cuda(), t.cuda()


def _color_fwd(model, inp, perm=None):
    o, d, ridx, t = _rays_cuda(inp, perm)
    ha = inp["ha"].cuda() if model.use_h_appear else None
    return model.forward_on_rays(ridx, t, o, d, inp["v"].cuda(), ha)


# ===================================================================================================================== comparisons
def _level_slices(max_level=None, meta=META):
    top = meta.n_levels - 1 if max_level is None else max_level
    return [(l, slice(meta.level_offsets[l], meta.level_offsets[l + 1]), l <= top) for l in range(meta.n_levels)]


def _np(v):
    return v.detach().double().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, dtype=np.float64)


def _compare(got, want, what, level_bound, weight_bounds, max_level=None, fails=None, meta=META):
    """per-level rel-L2 of the table gradient of the table `meta` (levels above max_level must be exactly zero in `got`) and rel-L2 of
    every other gradient.  Prints one METRIC line; appends failures to `fails` (asserts right away when it is None)."""
    own = fails is None
    fails = [] if own else fails
    g, w = _np(got["grid"]), _np(want["grid"])
    lv = {}
    for l, sl, on in _level_slices(max_level, meta):
        if on:
            if not np.abs(w[sl]).max() > 0:
                fails.append((what, "level has no reference gradient", l))
            lv[l] = tk._rel(g[sl], w[sl])
        elif np.any(g[sl] != 0):
            fails.append((what, "gradient above max_level", l, int(np.count_nonzero(g[sl]))))
    errs = {k: tk._rel(_np(got[k]), _np(want[k])) for k in want if k != "grid"}
    print(f"METRIC {what} grid per level max={max(lv.values()):.2e} " + " ".join(f"L{l}={e:.1e}" for l, e in lv.items()) + " | "
          + " ".join(f"{k}={e:.2e}" for k, e in errs.items()))
    fails += [(what, f"L{l}", e, level_bound) for l, e in lv.items() if not e < level_bound]
    for k, e in errs.items():
        if not np.abs(_np(want[k])).max() > 0:
            fails.append((what, k, "no reference gradient"))
        if not e < weight_bounds[k]:
            fails.append((what, k, e, weight_bounds[k]))
    if own:
        assert not fails, fails


def _all_finite(grads):
    return all(bool(torch.isfinite(v).all()) for v in grads.values())


# ===================================================================================================================== 1. order invariance
def test_sdf_forward_order_invariant():
    """k_fused_sdf_tc: a point's sdf does not depend on the order of the points (modes 0 and 1)"""
    c = _case(tk.PRODUCTION)
    model, inp = c["model"], c["inp"]
    s, perm = model.implicit_surface, inp["perm"].cuda()
    x = inp["x"].cuda()
    o, d, ridx, t = _rays_cuda(inp)
    with torch.no_grad():
        a = dict(points=s.fused_sdf(x), rays=s.fused_sdf_rays(ridx, t, o, d))
        b = dict(points=s.fused_sdf(x[perm]), rays=s.fused_sdf_rays(ridx[perm], t[perm], o, d))
    for k in a:
        assert torch.equal(a[k][perm], b[k]), (k, int((a[k][perm] != b[k]).sum()))


def _order_grads(route, model, inp, perm):
    """sdf backward with every cotangent set (route points / rays) or with the zero gaps compacted away (route indexed), in the given
    order of the work items"""
    p = tk._params(model)
    cot = inp["cot"][0].cuda()
    if route == "indexed":
        o, d, ridx, t = _rays_cuda(inp)
        c = torch.where(inp["zero"].cuda(), torch.zeros_like(cot), cot)
        keep = torch.nonzero(c).flatten()
        if perm is not None:
            keep = keep[torch.from_numpy(np.random.default_rng(5).permutation(keep.shape[0])).cuda()]
        return _sdf_bwd(model, None, c, rays=(o, d, ridx, t), keep=keep, n=keep.shape[0])
    q = torch.arange(cot.shape[0], device="cuda") if perm is None else perm.cuda()
    s = model.implicit_surface
    if route == "points":
        sdf = s.fused_sdf_autograd(inp["x"].cuda()[q])
    else:
        o, d, ridx, t = _rays_cuda(inp)
        sdf = s.fused_sdf_rays_autograd(ridx[q], t[q], o, d)
    return dict(zip(SDF_KEYS, torch.autograd.grad((sdf * cot[q]).sum(), [p[k] for k in SDF_KEYS])))


@pytest.mark.parametrize("route", ["points", "rays", "indexed"])
def test_sdf_backward_order_invariant(route):
    """k_sdf_bwd_tc on ray-ordered samples (the merge runs) against the same samples shuffled (nothing merges)"""
    c = _case(tk.PRODUCTION)
    model, inp = c["model"], c["inp"]
    x, perm = inp["x"].numpy(), inp["perm"].numpy()
    _assert_ray_order_merges(x)
    _assert_no_merge(x, perm)
    a = _order_grads(route, model, inp, None)
    b = _order_grads(route, model, inp, inp["perm"])
    assert _all_finite(a) and _all_finite(b)
    _compare(b, a, f"order sdf_bwd {route}", ORDER_LEVEL_REL, {k: ORDER_REL for k in SDF_KEYS})


def test_color_order_invariant():
    """k_color_fwd per point and k_color_rad_bwd + k_color_sdf_bwd on ray-ordered samples against the same samples shuffled"""
    c = _case(tk.PRODUCTION)
    model, inp = c["model"], c["inp"]
    perm = inp["perm"].cuda()
    _assert_ray_order_merges(inp["x"].numpy())
    _assert_no_merge(inp["x"].numpy(), inp["perm"].numpy())
    a, b = _color_fwd(model, inp), _color_fwd(model, inp, inp["perm"])
    assert torch.equal(a["x"].cpu(), inp["x"])
    for k in ("sdf", "nablas", "rgb", "x"):
        assert torch.equal(a[k][perm], b[k]), (k, int((a[k][perm] != b[k]).sum()))
    ga = tk._color_grads(model, a, inp["cot"])
    gb = tk._color_grads(model, b, tuple(v[inp["perm"]] for v in inp["cot"]))
    assert _all_finite(ga) and _all_finite(gb)
    _compare(gb, ga, "order color_bwd", ORDER_LEVEL_REL, {k: ORDER_REL for k in tk.BWD_REL})


# ===================================================================================================================== 2. float64, ray order
@pytest.fixture(scope="module", params=CASES, ids=CASE_IDS)
def case(request):
    return request.param


@pytest.mark.parametrize("zeros", [False, True], ids=["all", "zero30"])
def test_sdf_backward_ray_order_float64(case, zeros):
    """k_sdf_bwd_tc over every ray-ordered sample (a zero cotangent makes a lane inactive in the merge)"""
    c = _case(case)
    model, inp, ref = c["model"], c["inp"], c["ref"]
    max_level = case[1]
    n = inp["x"].shape[0]
    tk._assert_multi_tile("sdf_bwd", n, 3 if case == tk.PRODUCTION else 2)
    cot = _masked(inp["cot"], inp["zero"])[0] if zeros else inp["cot"][0]
    if zeros:
        assert 0.2 < float((cot == 0).float().mean()) < 0.4
    _assert_ray_order_merges(inp["x"].numpy(), max_level)
    got = _sdf_bwd(model, max_level, cot.cuda(), rays=_rays_cuda(inp))
    _compare(got, ref.sdf_backward(inp["x"].numpy(), cot.numpy()), f"f64 sdf_bwd rays {case} zeros={zeros}", LEVEL_REL, tk.BWD_REL, max_level)


@pytest.mark.parametrize("zeros", [False, True], ids=["all", "zero30"])
def test_color_backward_ray_order_float64(case, zeros):
    c = _case(case)
    model, inp, ref = c["model"], c["inp"], c["ref"]
    max_level = case[1]
    tk._assert_multi_tile("color_bwd", inp["x"].shape[0], 3)
    cot = _masked(inp["cot"], inp["zero"]) if zeros else inp["cot"]
    out = _color_fwd(model, inp)
    assert torch.equal(out["x"].cpu(), inp["x"])
    got = tk._color_grads(model, out, cot)
    want = ref.color_backward(_color_fwd64(c), *(v.numpy() for v in cot))
    _compare(got, want, f"f64 color_bwd rays {case} zeros={zeros}", LEVEL_REL, tk.BWD_REL, max_level)


# ===================================================================================================================== 3. hand-built warps
def _runs(lengths):
    return [j for j, m in enumerate(lengths) for _ in range(m)]


def _hand_structures():
    """name -> (run label per lane, lanes with a zero cotangent, heads on level 0 and MID_LEVEL for k_sdf_bwd_tc / k_color_sdf_bwd).
    Lanes with the same label share their cells on both levels, lanes with different labels do not."""
    rng = np.random.default_rng(7)
    h24, h25 = [2] * 8 + [1] * 16, [2] * 7 + [1] * 18
    rng.shuffle(h24), rng.shuffle(h25)
    return {
        "one_run": ([0] * 32, [], 1, 1),
        "32_heads": (list(range(32)), [], 32, 32),
        "24_heads": (_runs(h24), [], 24, 24),
        "25_heads": (_runs(h25), [], 25, 25),
        "16+16": (_runs([16, 16]), [], 2, 2),
        "1,2,3,..": (_runs([1, 2, 3, 4, 5, 6, 7, 4]), [], 8, 8),
        "A_B_A": ([0] * 12 + [1] * 4 + [0] * 16, [], 3, 3),
        "head_at_31": (_runs([31, 1]), [], 2, 2),
        "zero_on_head": (_runs([8, 8, 16]), [8], 4, 3),
        "zero_in_run": ([0] * 32, [13], 3, 1),
    }


def _label_centre(label, which):
    """table-space centre of a level-0 cell (14 cells per axis, cell k centred on k / 14) that is also a cell centre of MID_LEVEL"""
    k = np.array([2 + label % 10, 2 + (label // 10) % 10, 2 + which % 8], dtype=np.float64)
    sc = CFG["lod_res"][MID_LEVEL] - 2
    return np.round(k / 14 * sc) / sc


def _hand_layouts():
    """Two launches of the same hand-built points, one tile per structure.  merged: lanes 0..31 of tile k are structure k; nomerge:
    its 32 points sit in lanes 0, 2, .., 62 with filler between.  Filler (zero cotangent) fills the rest; it lies in level-0 cell
    (12, 12, 12), away from every hand-built cell, so no two consecutive lanes of the nomerge layout share a cell on any level.
    -> names, x [P, 3] (the hand-built points first, then filler), order of each layout [K * 128], zero-cotangent mask [P]"""
    structs = _hand_structures()
    names = list(structs)
    pts, zero = [], []
    for k, name in enumerate(names):
        labels, zl = structs[name][:2]
        for lane, lab in enumerate(labels):
            xs = _label_centre(lab, k) + np.array([3e-5, 2e-5, -2.5e-5]) * lane
            pts.append(2 * xs - 1)
            zero.append(lane in zl)
    nh = len(pts)
    n_fill = 96
    for j in range(n_fill):
        pts.append(2 * (np.full(3, 12 / 14) + np.array([1e-4, -1e-4, 2e-4]) * (j - n_fill / 2) / n_fill) - 1)
        zero.append(True)
    K = len(names)
    merged, nomerge = np.empty((K, 128), dtype=np.int64), np.empty((K, 128), dtype=np.int64)
    fill = nh + np.arange(n_fill)
    for k in range(K):
        hand = k * 32 + np.arange(32)
        merged[k] = np.concatenate([hand, fill])
        nomerge[k, 0:64:2], nomerge[k, 1:64:2], nomerge[k, 64:] = hand, fill[:32], fill[32:]
    return names, np.stack(pts).astype(np.float32), dict(merged=merged.ravel(), nomerge=nomerge.ravel()), np.array(zero)


@pytest.mark.parametrize("kernel", ["sdf", "color"])
def test_hand_built_warps(kernel):
    """one hand-built warp's cotangent at a time: the table gradient is exactly that warp's sum, against float64 (per level) and
    against the same 32 points in a layout where nothing merges (fp32 order)"""
    c = _case(tk.PRODUCTION)
    model, ref = c["model"], c["ref"]
    names, x, orders, zero = _hand_layouts()
    structs = _hand_structures()
    g = torch.Generator().manual_seed(29)
    P = x.shape[0]
    cot_all = (torch.randn(P, generator=g), torch.randn(P, 3, generator=g) * 0.05, torch.randn(P, 3, generator=g))
    cot_all = _masked(cot_all, torch.from_numpy(zero))
    v_all = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    ha_all = torch.randn(P, 4, generator=g) * 0.5
    # census: the designed run structures on level 0 and MID_LEVEL in the merged layout, no merge at all in the nomerge layout
    for k, name in enumerate(names):
        lanes = orders["merged"][k * 128:(k + 1) * 128]
        active = ~zero[lanes] if kernel == "sdf" else None
        heads = merge_census(x, CFG, order=lanes, active=active)["heads"][0]
        want = structs[name][2] if kernel == "sdf" else structs[name][3]
        assert heads[0] == want and heads[MID_LEVEL] == want, (name, heads[0], heads[MID_LEVEL], want)
    nm = merge_census(x, CFG, order=orders["nomerge"])["heads"].reshape(len(names), 4, -1)[:, :2]
    assert (nm > MERGE_MAX_HEADS).all(), int(nm.min())

    launch = {}                           # layout -> (point of each lane, the points on the device | the colour forward over them)
    for lay, order in orders.items():
        q, xx = torch.from_numpy(order), torch.from_numpy(x[order])
        if kernel == "sdf":
            launch[lay] = (q, xx.cuda())
        else:
            n = order.shape[0]
            inp = dict(ridx=torch.arange(n), t=torch.zeros(n), o=xx, d=torch.tensor([[0.6, 0.0, 0.8]]).repeat(n, 1), v=v_all[q],
                       ha=ha_all[q])
            out = tk._color_fwd(model, inp)
            assert torch.equal(out["x"].cpu(), xx)
            launch[lay] = (q, out)
    fails = []
    for k, name in enumerate(names):
        rows = np.arange(k * 32, (k + 1) * 32)
        mask = torch.zeros(P, dtype=torch.bool)
        mask[rows] = True
        cot = _masked(cot_all, ~mask)
        got = {}
        for lay, (q, obj) in launch.items():
            cq = tuple(v[q] for v in cot)
            if kernel == "sdf":
                got[lay] = _sdf_bwd(model, None, cq[0].cuda(), x=obj)
            else:
                got[lay] = tk._color_grads(model, obj, cq, retain=True)
        if kernel == "sdf":
            want = ref.sdf_backward(x[rows], cot[0].numpy()[rows])
            keys = SDF_KEYS
        else:
            f = ref.color_forward(x[rows], v_all.numpy()[rows], ha_all.numpy()[rows])
            want = ref.color_backward(f, *(v.numpy()[rows] for v in cot))
            keys = tuple(tk.BWD_REL)
        _compare(got["merged"], want, f"hand {kernel} {name} vs f64", HAND_REL, {k_: tk.TILE_REL[k_] for k_ in keys}, fails=fails)
        _compare(got["merged"], got["nomerge"], f"hand {kernel} {name} vs nomerge", ORDER_LEVEL_REL, {k_: ORDER_REL for k_ in keys},
                 fails=fails)
    assert not fails, fails


# ===================================================================================================================== 4. the graph step's calls
def _count_block(slot, value):
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[slot] = value
    return cnt


def _bench_graph_case():
    """the graph-step calls' case on the bench table: the production model on its ray-ordered samples.  tests/test_wide_scatter_gpu.py
    builds the same dict for the 17-level street table (the 48-column kernels)."""
    c = _case(tk.PRODUCTION)
    return dict(name="bench16", model=c["model"], inp=c["inp"], ref=c["ref"], cfg=CFG, meta=META, bwd_rel=tk.BWD_REL,
                merge_levels=list(range(5)))


def test_indexed_sdf_backward_keep_list_and_device_count():
    """nsb_fused_sdf_bwd_indexed as _StaticSDF.backward (graphics/neus_static.py) calls it: the samples with a non-zero cotangent
    compacted by nsb_flag_nonzero + a scan into a keep list; once with the count on the host, once with the count device-resident
    and the capacity larger.  Slots past the counts hold in-range indices of samples whose cotangent is NaN."""
    indexed_sdf_backward_keep_list_and_device_count(_bench_graph_case())


def indexed_sdf_backward_keep_list_and_device_count(c):
    """the body of the test above for a case dict(name, model, inp, ref, cfg, meta, bwd_rel, merge_levels): merge_levels are the levels
    on which the census of the kept samples must show the merge on most warps"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _call, _scan
    name, model, inp, ref, meta = c["name"], c["model"], c["inp"], c["ref"], c["meta"]
    n, extra = inp["x"].shape[0], 1000
    cap = n + extra
    cot = _masked(inp["cot"], inp["zero"])[0]
    o, d, ridx, t = _rays_cuda(inp)
    g = torch.Generator().manual_seed(31)
    ridx_c = torch.cat([ridx, torch.randint(0, o.shape[0], (extra,), generator=g).cuda()])
    t_c = torch.cat([t, t[:extra]])
    d_c = torch.cat([cot.cuda(), torch.full((extra,), float("nan"), device="cuda")])
    cnt = _count_block(CNT_SLOTS["boundary"], n)
    flag = torch.empty(cap, dtype=torch.int32, device="cuda")
    _call(L.lib().nsb_flag_nonzero, "flag_nonzero", cnt, CNT_SLOTS["boundary"], None, L.ptr(d_c, "f32"), L.c_i64(cap), L.ptr(flag), L.stream_ptr())
    keep = torch.empty(cap, dtype=torch.int64, device="cuda")
    _scan(flag, cnt, CNT_SLOTS["nonzero"], index=keep)
    K = int(cnt[CNT_SLOTS["nonzero"]])
    kept = torch.nonzero(cot).flatten()
    assert K == kept.shape[0] and torch.equal(keep[:K].cpu(), kept)
    c_k = merge_census(inp["x"].numpy(), c["cfg"], order=kept.numpy())
    frac = (c_k["heads"] <= MERGE_MAX_HEADS).mean(0)
    assert (frac[c["merge_levels"]] >= 0.5).all(), frac
    rays = (o, d, ridx_c, t_c)
    a = _sdf_bwd(model, None, d_c, rays=rays, keep=keep[:K].clone(), n=K)
    _compare(a, ref.sdf_backward(inp["x"].numpy()[kept], cot.numpy()[kept]), f"f64 sdf_bwd indexed {name}", LEVEL_REL, c["bwd_rel"], meta=meta)
    keep[K:] = n + torch.arange(cap - K, device="cuda") % extra          # in range; the samples they name carry NaN cotangents
    b = _sdf_bwd(model, None, d_c, rays=rays, keep=keep, n=cap, count=(cnt, CNT_SLOTS["nonzero"]))
    assert _all_finite(b)
    _compare(b, a, f"sdf_bwd indexed count-bound vs count-sized {name}", ORDER_LEVEL_REL, {k: ORDER_REL for k in SDF_KEYS}, meta=meta)


def test_color_device_count():
    """nsb_fused_color_fwd / nsb_fused_color_bwd as _StaticColor calls them: capacity larger than the device-resident count; slots past
    the count hold in-range ray indices and NaN cotangents, and the outputs there must stay untouched"""
    color_device_count(_bench_graph_case())


def color_device_count(c):
    """the body of the test above for a case dict as indexed_sdf_backward_keep_list_and_device_count takes it"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.fields.fused_color import h_tile_cols
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _call
    name, model, inp = c["name"], c["model"], c["inp"]
    n, extra = inp["x"].shape[0], 1000
    cap = n + extra
    P = L.ptr
    grid16, net, _alive = model._fused_color_state()
    meta = model.implicit_surface.encoding.meta
    o, d, ridx, t = _rays_cuda(inp)
    g = torch.Generator().manual_seed(37)
    ridx_c = torch.cat([ridx, torch.randint(0, o.shape[0], (extra,), generator=g).cuda()])
    t_c = torch.cat([t, t[:extra]])
    v, ha = inp["v"].cuda(), inp["ha"].cuda()
    nan = float("nan")
    cot = [torch.cat([x.cuda(), torch.full((extra, *x.shape[1:]), nan, device="cuda")]) for x in inp["cot"]]
    SENT = -12345.0
    cnt = _count_block(CNT_SLOTS["kept"], n)
    ps = tk._params(model)

    def run(m, count):
        out = dict(sdf=torch.full((m,), SENT, device="cuda"), nab=torch.full((m, 3), SENT, device="cuda"),
                   rgb=torch.full((m, 3), SENT, device="cuda"), x=torch.full((m, 3), SENT, device="cuda"))
        acts = torch.empty(4, int(L.lib().nsb_color_act_bytes(L.c_i64(m), meta.n_pseudo_levels)), dtype=torch.uint8, device="cuda")
        fwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o, "f32"), P(d, "f32"), P(ridx_c, "i64"), P(t_c, "f32"), P(v, "f32"),
               P(ha, "f32"), L.c_i64(m), L.c_i32(model.implicit_surface._ml(None)), P(out["sdf"]), P(out["nab"]), P(out["rgb"]), P(out["x"]),
               *[P(acts[k]) for k in range(4)], None, L.stream_ptr())
        grads = {k: torch.zeros(p.shape, dtype=torch.float32, device="cuda") for k, p in ps.items()}
        dh = torch.empty(m, h_tile_cols(meta.n_pseudo_levels), dtype=torch.float32, device="cuda")
        cm = [x[:m].contiguous() for x in cot]
        bwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o, "f32"), P(d, "f32"), P(ridx_c, "i64"), P(t_c, "f32"), L.c_i64(m),
               L.c_i32(model.implicit_surface._ml(None)), *[P(acts[k]) for k in range(4)], P(out["rgb"]), P(cm[0]), P(cm[1]), P(cm[2]), P(dh),
               *[P(grads[k]) for k in tk.BWD_REL], L.stream_ptr())
        for fn, what, args in ((L.lib().nsb_fused_color_fwd, "fused_color_fwd", fwd), (L.lib().nsb_fused_color_bwd, "fused_color_bwd", bwd)):
            if count:
                _call(fn, what, cnt, CNT_SLOTS["kept"], None, *args)
            else:
                L.check(fn(*args), what)
        return out, grads

    a_out, a = run(n, False)
    b_out, b = run(cap, True)
    for k in a_out:
        assert torch.equal(b_out[k][:n], a_out[k]), k
        assert bool((b_out[k][n:] == SENT).all()), k
    assert torch.equal(a_out["x"].cpu(), inp["x"])
    assert _all_finite(b)
    _compare(b, a, f"color_bwd count-bound vs count-sized {name}", ORDER_LEVEL_REL, {k: ORDER_REL for k in tk.BWD_REL}, meta=c["meta"])
