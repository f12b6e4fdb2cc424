"""The warp-merged table-gradient scatter of k_sdf_bwd_tc and k_color_sdf_bwd on EVERY level, the finest included.

warp_merge_updates (csrc/lotd_device.cuh) keys a lane's cell by its three integer cell coordinates, 21 bits each, so the merge runs on
levels with more than 1024 cells per axis too: the finest levels of the bench table (levels 13-15: 1073, 1483 and 2049 per axis) and
the cuboid levels of the cfg3 table where only one axis exceeds 1024.  Those are the levels where the samples of the last up-sampling
stage crowd together: 33 samples within a few thousandths of the surface, closer than a level-15 cell.  Covered here:
  - ray-ordered samples with such clusters, on the bench table and on the cfg3 table, where the census below shows the merge running on
    the levels above 1024 cells per axis: both kernels against float64 per level and against the same samples shuffled (nothing merges)
  - hand-built warps on level 15 at the edges of the merge (one run, 24 and 25 heads, a head at lane 31, A A B A A, zero cotangents)
  - the host rejection of a table whose resolution does not fit the key
  - the static step's single table gradient (SharedTableGrad) against the two nodes' separate buffers
The census here is the all-level rule; tests/util.py:merge_census keeps the coordinates, and its `mergeable` flag is not used.
Bounds are those of tests/test_tc_scatter_gpu.py (DESIGN.md §4)."""
import numpy as np
import pytest
import torch

import test_tc_geometry_gpu as tgeo
import test_tc_kernels_gpu as tk
import test_tc_scatter_gpu as ts
from oracle import fused64, lotd as olotd
from util import MERGE_MAX_HEADS, merge_census

pytestmark = pytest.mark.gpu

CFG = ts.CFG
FINE = (13, 14, 15)                 # the bench table's levels with more than 1024 cells per axis
LEVEL_REL, HAND_REL, ORDER_LEVEL_REL, ORDER_REL = ts.LEVEL_REL, ts.HAND_REL, ts.ORDER_LEVEL_REL, ts.ORDER_REL
SDF_KEYS = ts.SDF_KEYS
# a level-15 hand-built warp against its no-merge layout: on the coarse levels all 32 lanes share one cell, so the level's gradient is
# a 32-term fp32 sum of cotangents of either sign, in two orders (measured <= 2.1e-6, head_at_31 level 4; float64 keeps HAND_REL)
HAND_ORDER_LEVEL_REL = 6e-6


# ===================================================================================================================== census
def census(x, cfg, order=None, active=None):
    """The run structure every level's merge sees (all levels merge).  -> dict(heads [W/32, L] run heads per warp (inactive lanes
    count), issues [L] the 8-reduction issues per level: a warp issues one per active run head, or one per active lane when it has more
    than MERGE_MAX_HEADS heads, active [L] the active lanes)"""
    c = merge_census(x, cfg, order=order, active=active)
    act = c["valid"].copy()
    if active is not None:
        act[:len(active)] &= np.asarray(active, dtype=bool)
    act = act.reshape(-1, 32)
    prev = np.zeros_like(act)
    prev[:, 1:] = act[:, :-1]
    issues = []
    for l, cell in enumerate(c["cells"]):
        cw = cell.reshape(-1, 32, 3)
        differs = np.ones(act.shape, dtype=bool)
        differs[:, 1:] = (cw[:, 1:] != cw[:, :-1]).any(-1)
        head = ~act | ~prev | differs
        assert (head.sum(1) == c["heads"][:, l]).all()
        per_warp = np.where(head.sum(1) > MERGE_MAX_HEADS, act.sum(1), (act & head).sum(1))
        issues.append(int(per_warp.sum()))
    return dict(heads=c["heads"], issues=np.array(issues), active=int(act.sum()), levels=c["levels"])


# ===================================================================================================================== inputs
def _box_beam(rng):
    """a ray through the box from outside it -> (o, d, view direction, entry t, exit t)"""
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    o = rng.uniform(-0.6, 0.6, 3) - 2.5 * d
    return (o, d, d, *ts._slab(o, d, 0.99))


def _cluster_rays(n, n_appear, seed, beam=_box_beam, half=0.003):
    """n samples of rays (beam(rng) -> o, d, view direction, entry and exit t) in ray order, t ascending: 8..14 coarse samples over the
    ray's interval and, around a surface point inside it, 33 samples within +-half (the last up-sampling stage at inv_s 1024 places them
    within +-0.003 in the unit box), then 0..3 more coarse samples.  No ray length is a multiple of 32; ~30 % of the sdf cotangents are
    zero (runs and isolated)."""
    rng = np.random.default_rng(seed)
    os_, ds, vs, ts_, total = [], [], [], [], 0
    while total < n:
        o, d, v, t0, t1 = beam(rng)
        s = rng.uniform(t0 + 0.2 * (t1 - t0), t1 - 0.3 * (t1 - t0))
        near = np.sort(s + rng.uniform(-half, half, 33))
        a = np.linspace(t0, s - 0.01, rng.integers(8, 15))
        b = np.linspace(s + 0.01, t1, 4)[:rng.integers(0, 4)]
        t = np.concatenate([a, near, b])
        if len(t) % 32 == 0:
            t = t[1:]
        t = t[:n - total]
        os_.append(o), ds.append(d), vs.append(v), ts_.append(t)
        total += len(t)
    lens = np.array([len(t) for t in ts_])
    o = torch.tensor(np.stack(os_), dtype=torch.float32)
    d = torch.tensor(np.stack(ds), dtype=torch.float32)
    t = torch.tensor(np.concatenate(ts_), dtype=torch.float32)
    ridx = torch.from_numpy(np.repeat(np.arange(len(ts_)), lens))
    x = (d.double()[ridx] * t.double()[:, None] + o.double()[ridx]).float()        # the kernels' fma(d, t, o)
    assert float(x.abs().max()) < 1.0
    g = torch.Generator().manual_seed(seed)
    ha = torch.randn(len(ts_), n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    zero = torch.rand(n, generator=g) < 0.1
    for s in np.flatnonzero(rng.random(n) < 0.025):
        zero[s:s + rng.integers(2, 17)] = True
    return dict(x=x, o=o, d=d, t=t, ridx=ridx, v=torch.tensor(np.stack(vs), dtype=torch.float32), ha=ha, cot=cot, zero=zero,
                perm=torch.from_numpy(rng.permutation(n)))


def _assert_merges_on(x, cfg, levels, what, zero=None):
    """the merge runs on most warps of `levels` and saves at least a third of their reductions; shuffled, nothing merges"""
    c = census(x, cfg, active=None if zero is None else ~zero)
    frac = (c["heads"] <= MERGE_MAX_HEADS).mean(0)
    share = c["issues"] / c["active"]
    print(f"METRIC census {what}: merging warps / issues per active lane " + " ".join(f"L{l}={f:.2f}/{s:.2f}" for l, f, s in zip(c["levels"], frac, share)))
    assert all(frac[l] >= 0.5 and share[l] <= 0.67 for l in levels), (frac, share)
    sh = census(x, cfg, order=np.random.default_rng(3).permutation(x.shape[0]))
    assert (sh["heads"] > MERGE_MAX_HEADS).all(), int(sh["heads"].min())


_CACHE = {}


def _case(table):
    """model, ray-ordered cluster samples and the float64 reference on the bench table ('cubic') or the cfg3 table ('cuboid')"""
    if table not in _CACHE:
        n = tk._size("color_fwd", 2)
        if table == "cubic":
            model, cfg = tk._model(64, 64, 4, seed=71), CFG
        else:
            cfg = tgeo._cfg()
            model = tgeo._model(cfg, seed=73)
        inp = _cluster_rays(n, 4, seed=79 if table == "cubic" else 83)
        _CACHE.clear()
        _CACHE[table] = dict(model=model, cfg=cfg, meta=olotd.LoDMeta(3, **cfg), inp=inp, ref=fused64.Fused64.from_model(model))
    return _CACHE[table]


def _over_1024(cfg):
    """-> (the levels with more than 1024 cells on exactly one axis, on two or three axes)"""
    n = (np.array(olotd.LoDMeta(3, **cfg).level_res_multidim) > 1024).sum(1)
    return [l for l in range(len(n)) if n[l] == 1], [l for l in range(len(n)) if n[l] > 1]


def _merge_levels(table):
    """the levels over 1024 cells per axis on which the census must show the merge: the bench table's finest three, the cfg3 table's
    levels with one such axis (its finest cells are smaller than the clusters' spacing)"""
    return list(FINE) if table == "cubic" else _over_1024(tgeo._cfg())[0]


def _compare_f64(c, got, want, what):
    """per level at LEVEL_REL, the other gradients at tk.BWD_REL (b2 at the cfg3 table's bound: the plain fp32 sum of the cotangents)"""
    if c["cfg"] is CFG:
        ts._compare(got, want, what, LEVEL_REL, tk.BWD_REL)
    else:
        tgeo._per_level(c["meta"], got["grid"], want["grid"], what, LEVEL_REL)
        tgeo._others(got, want, what)


# ===================================================================================================================== ray order
TABLES = ["cubic", "cuboid"]


def test_tables_over_1024():
    assert _over_1024(CFG) == ([], list(FINE))
    assert len(_over_1024(tgeo._cfg())[0]) >= 3


@pytest.mark.parametrize("table", TABLES)
@pytest.mark.parametrize("zeros", [False, True], ids=["all", "zero30"])
def test_sdf_backward_clusters_float64(table, zeros):
    """k_sdf_bwd_tc over ray-ordered cluster samples: per level against float64"""
    c = _case(table)
    model, inp, ref = c["model"], c["inp"], c["ref"]
    tk._assert_multi_tile("sdf_bwd", inp["x"].shape[0], 2)
    cot = ts._masked(inp["cot"], inp["zero"])[0] if zeros else inp["cot"][0]
    _assert_merges_on(inp["x"].numpy(), c["cfg"], _merge_levels(table), f"{table} sdf", inp["zero"].numpy() if zeros else None)
    got = ts._sdf_bwd(model, None, cot.cuda(), rays=ts._rays_cuda(inp))
    _compare_f64(c, got, ref.sdf_backward(inp["x"].numpy(), cot.numpy()), f"f64 sdf_bwd clusters {table} zeros={zeros}")


@pytest.mark.parametrize("table", TABLES)
def test_color_backward_clusters_float64(table):
    """k_color_rad_bwd + k_color_sdf_bwd over ray-ordered cluster samples: per level against float64"""
    c = _case(table)
    model, inp, ref = c["model"], c["inp"], c["ref"]
    _assert_merges_on(inp["x"].numpy(), c["cfg"], _merge_levels(table), f"{table} color")
    out = ts._color_fwd(model, inp)
    assert torch.equal(out["x"].cpu(), inp["x"])
    got = tk._color_grads(model, out, inp["cot"])
    want = ref.color_backward(ref.color_forward(inp["x"].numpy(), inp["v"][inp["ridx"]].numpy(), inp["ha"][inp["ridx"]].numpy()),
                              *(v.numpy() for v in inp["cot"]))
    _compare_f64(c, got, want, f"f64 color_bwd clusters {table}")


@pytest.mark.parametrize("route", ["points", "rays", "indexed"])
def test_sdf_backward_clusters_order_invariant(route):
    """k_sdf_bwd_tc on the cluster samples in ray order (the merge runs on every level) against the same samples shuffled"""
    c = _case("cubic")
    model, inp = c["model"], c["inp"]
    a = ts._order_grads(route, model, inp, None)
    b = ts._order_grads(route, model, inp, inp["perm"])
    assert ts._all_finite(a) and ts._all_finite(b)
    ts._compare(b, a, f"order sdf_bwd clusters {route}", ORDER_LEVEL_REL, {k: ORDER_REL for k in SDF_KEYS})


def test_color_backward_clusters_order_invariant():
    c = _case("cubic")
    model, inp = c["model"], c["inp"]
    perm = inp["perm"]
    a, b = ts._color_fwd(model, inp), ts._color_fwd(model, inp, perm)
    ga = tk._color_grads(model, a, inp["cot"])
    gb = tk._color_grads(model, b, tuple(v[perm] for v in inp["cot"]))
    assert ts._all_finite(ga) and ts._all_finite(gb)
    ts._compare(gb, ga, "order color_bwd clusters", ORDER_LEVEL_REL, {k: ORDER_REL for k in tk.BWD_REL})


# ===================================================================================================================== hand-built warps
def _hand_layouts(cfg, level):
    """ts._hand_layouts with the run structures set on `level` of the table `cfg` (level 15 of the bench table: 2049 cells per axis).
    Label j of structure k sits in cell (200 + 1024 (1 - j % 2) + 3 (j // 2), 600 + j % 2, 700 + 3 k) of the level: labels 2 m and 2 m + 1
    are cells (x + 1024, y) and (x, y + 1) with y even, whose keys coincide when packed with 10 bits per axis, so a narrower key would
    merge lanes that must stay apart.  Lanes are jittered by 1e-6 per lane in table space (a level-15 cell is ~4.9e-4 wide), or by an
    eighth of the smallest cell / 32 on a finer level, so lanes share a cell of the level exactly when they share a label.  The nomerge
    layout interleaves filler lanes in cells far away on every level."""
    structs = ts._hand_structures()
    names = list(structs)
    sc = np.array(olotd.LoDMeta(3, **cfg).level_res_multidim[level], dtype=np.float64) - 2
    jitter = min(1e-6, 0.125 / sc.max() / 32)
    pts, zero = [], []
    for k, name in enumerate(names):
        labels, zl = structs[name][:2]
        for lane, lab in enumerate(labels):
            cell = np.array([200 + 1024 * (1 - lab % 2) + 3 * (lab // 2), 600 + lab % 2, 700 + 3 * k])
            xs = cell / sc + jitter * lane
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


def hand_built_warps(model, ref, cfg, level, kernel, what):
    """one hand-built warp's cotangent at a time (_hand_layouts(cfg, level)): the table gradient is that warp's sum, against float64 (per
    level) and against the same 32 points in a layout where nothing merges"""
    meta = olotd.LoDMeta(3, **cfg)
    names, x, orders, zero = _hand_layouts(cfg, level)
    structs = ts._hand_structures()
    for k, name in enumerate(names):
        lanes = orders["merged"][k * 128:(k + 1) * 128]
        heads = census(x, cfg, order=lanes, active=~zero[lanes] if kernel == "sdf" else None)["heads"][0]
        want = structs[name][2] if kernel == "sdf" else structs[name][3]
        assert heads[level] == want, (name, heads[level], want)
    nm = census(x, cfg, order=orders["nomerge"])["heads"].reshape(len(names), 4, -1)[:, :2]
    assert (nm > MERGE_MAX_HEADS).all(), int(nm.min())
    # the 32-heads warp: lanes 2 m and 2 m + 1 are different cells of the level whose 10-bit-per-axis keys are equal
    k32 = names.index("32_heads")
    cell = merge_census(x, cfg, order=orders["merged"][k32 * 128:k32 * 128 + 32])["cells"][level].astype(np.int64)
    packed10 = cell[:, 0] | (cell[:, 1] << 10) | (cell[:, 2] << 20)
    assert (cell[0::2] != cell[1::2]).any(1).all() and (packed10[0::2] == packed10[1::2]).all() and (cell[0::2, 0] >= 1024).all()
    g = torch.Generator().manual_seed(89)
    P = x.shape[0]
    cot_all = ts._masked((torch.randn(P, generator=g), torch.randn(P, 3, generator=g) * 0.05, torch.randn(P, 3, generator=g)),
                         torch.from_numpy(zero))
    v_all = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    ha_all = torch.randn(P, 4, generator=g) * 0.5
    launch = {}
    for lay, order in orders.items():
        q, xx = torch.from_numpy(order), torch.from_numpy(x[order])
        if kernel == "sdf":
            launch[lay] = (q, xx.cuda())
        else:
            n = order.shape[0]
            inp = dict(ridx=torch.arange(n), t=torch.zeros(n), o=xx, d=torch.tensor([[0.6, 0.0, 0.8]]).repeat(n, 1), v=v_all[q], ha=ha_all[q])
            out = tk._color_fwd(model, inp)
            assert torch.equal(out["x"].cpu(), xx)
            launch[lay] = (q, out)
    fails = []
    for k, name in enumerate(names):
        rows = np.arange(k * 32, (k + 1) * 32)
        mask = torch.zeros(P, dtype=torch.bool)
        mask[rows] = True
        cot = ts._masked(cot_all, ~mask)
        got = {}
        for lay, (q, obj) in launch.items():
            cq = tuple(v[q] for v in cot)
            got[lay] = ts._sdf_bwd(model, None, cq[0].cuda(), x=obj) if kernel == "sdf" else tk._color_grads(model, obj, cq, retain=True)
        if kernel == "sdf":
            want, keys = ref.sdf_backward(x[rows], cot[0].numpy()[rows]), SDF_KEYS
        else:
            want = ref.color_backward(ref.color_forward(x[rows], v_all.numpy()[rows], ha_all.numpy()[rows]), *(v.numpy()[rows] for v in cot))
            keys = tuple(tk.BWD_REL)
        ts._compare(got["merged"], want, f"{what} {kernel} {name} vs f64", HAND_REL, {k_: tk.TILE_REL[k_] for k_ in keys}, fails=fails,
                    meta=meta)
        ts._compare(got["merged"], got["nomerge"], f"{what} {kernel} {name} vs nomerge", HAND_ORDER_LEVEL_REL, {k_: ORDER_REL for k_ in keys},
                    fails=fails, meta=meta)
    assert not fails, fails


@pytest.mark.parametrize("kernel", ["sdf", "color"])
def test_hand_built_warps_level15(kernel):
    c = _case("cubic")
    hand_built_warps(c["model"], c["ref"], CFG, 15, kernel, "hand L15")


# ===================================================================================================================== host rejection
@pytest.mark.parametrize("res", [2 ** 21, 2 ** 21 + 1])
def test_resolution_must_fit_the_cell_key(res):
    """a hashed level with `res` cells on one axis: 2^21 (the key's 21 bits) runs, one more is refused before any launch"""
    from neuralsim_b200.fields.neus import LoTDNeuS
    cfg = olotd.gen_ngp_cfg()
    cfg["lod_res"] = [[r, r, r] for r in cfg["lod_res"]]
    cfg["lod_res"][15][1] = res
    assert cfg["lod_types"][15] == "Hash"
    gen = torch.Generator("cuda").manual_seed(97)
    model = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=cfg)), radiance_cfg=dict(n_appear_embedding=4), device="cuda",
                     generator=gen)
    x = torch.rand(300, 3, device="cuda", generator=gen) * 2 - 1
    s = model.implicit_surface
    if res <= 2 ** 21:
        (s.fused_sdf_autograd(x) * 1.0).sum().backward()
        assert torch.isfinite(s.encoding.flattened_params.grad).all()
    else:
        with pytest.raises(RuntimeError, match="cells per axis"):
            with torch.no_grad():
                s.fused_sdf(x)


# ===================================================================================================================== static step
def test_static_step_one_table_gradient(cuda, monkeypatch):
    """the static step's boundary and colour backward nodes scatter into one buffer (SharedTableGrad): the table gradient equals the sum
    of the two nodes' separate buffers (fp32 atomics: order tolerance), and every other gradient as well -- also with a term on the table
    that is created after the render, whose gradient autograd may add to the table's before either node has run"""
    from neuralsim_b200.fields.fused_color import SharedTableGrad
    from neuralsim_b200.graphics.neus_static import render_static
    from oracle import scene as oscene
    from util import make_pair
    _, model = make_pair(cuda)
    model.train()
    table = model.implicit_surface.encoding.flattened_params
    key = "implicit_surface.encoding.flattened_params"
    ro, rd = oscene.pinhole_rays(36, 48, oscene.orbit_camera(1, 8, radius=3.0, elev_deg=25.0))
    ro, rd = ro.to(cuda), rd.to(cuda)
    ha = torch.zeros(ro.shape[0], 4, device=cuda)
    take = SharedTableGrad.take

    def run(w):
        model.zero_grad(set_to_none=True)
        rendered, cnt, _ = render_static(model, ro, rd, ha, near=0.01, march_cap=1 << 18, kept_cap=1 << 17, coherent=True)
        assert int(cnt[20]) == 0
        loss = sum(rendered[k].mean() for k in ("rgb_volume", "depth_volume", "normals_volume", "mask_volume"))
        if w is not None:
            loss = loss + (table * w).sum()
        loss.backward()
        return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    w = None
    for case in ("render", "render+table_term"):
        shared = []
        monkeypatch.setattr(SharedTableGrad, "take", lambda self, shape, device: shared.append(take(self, shape, device)) or shared[-1])
        one = run(w)
        assert len(shared) == 2 and shared[0] is shared[1]                 # both nodes ran and scatter into one buffer
        assert key in one and float(one[key].abs().sum()) > 0
        parts = []                                                          # a buffer per node; they never reach .grad
        monkeypatch.setattr(SharedTableGrad, "take", lambda self, shape, device: parts.append(torch.zeros(shape, device=device)) or parts[-1])
        two = run(w)
        assert len(parts) == 2 and (key in two) == (w is not None)
        two[key] = parts[0] + parts[1] + (two[key] if w is not None else 0)
        assert one.keys() == two.keys()
        for n in one:
            e = tk._rel(one[n].double().cpu().numpy(), two[n].double().cpu().numpy())
            bound = ORDER_LEVEL_REL if n == key else ORDER_REL
            assert e < bound, (case, n, e, bound)
        # the extra term: random, at the scale of the render's table gradient, so that losing either node's part shows
        w = torch.randn(table.shape, device=cuda, generator=torch.Generator(cuda).manual_seed(101)) * float(one[key].abs().mean())
