"""The fused wgmma kernels (k_fused_sdf_tc, k_sdf_bwd_tc, k_color_fwd, k_color_rad_bwd, k_color_sdf_bwd) against the float64
reference (oracle/fused64.py) at the geometry of the cfg3 street model: cuboid levels from the `ngp` auto config of a 40 x 150 x 15 m
aabb (bench_cfg3.py, here with a 2^16 table as tests/test_cfg3_gpu.py builds it) and sdf_scale 25, so that the nablas scale
fac = sdf_scale / radius differs on every axis.  tests/test_tc_kernels_gpu.py and tests/test_tc_scatter_gpu.py run the same
kernels on cubic tables only.

On this table levels 0-7 have every axis <= 1024 and the warp merge of the table-gradient scatter runs there; levels 8-14 have some
axes <= 1024 and some above, and the merge must stay off.  The inputs are random points, LiDAR-like samples in ray order (long rays,
0.2 m steps) and hand-built warps whose lanes alternate between two cells of level 8 that a cell key of fewer axes would not tell
apart.  A table with a hash size that is not a power of two covers the `h % size` addressing of the fused kernels.  Bounds are about
3x the errors measured on an H100 80GB HBM3 (132 SMs, 400 W power limit); DESIGN.md §4 lists them."""
import numpy as np
import pytest
import torch

import test_tc_kernels_gpu as tk
from oracle import fused64, lotd as olotd
from test_tc_scatter_gpu import _sdf_bwd
from util import MERGE_MAX_HEADS, merge_census

pytestmark = pytest.mark.gpu

AABB = [[-20., -75., -7.5], [20., 75., 7.5]]
RADIUS = np.array([20., 75., 7.5])
SDF_SCALE = 25.0
COLLIDE_LEVEL = 8                   # [319, 1197, 119]: x, z <= 1024 < y

# Bounds (measured values in DESIGN.md §4).  Forwards keep tk's per-element bounds; gradients other than the table keep tk.BWD_REL except
# b2, the plain fp32 sum of the sdf cotangents, which cancels to ~1/sqrt(n) of its terms (measured <= 5.6e-6 here).
LEVEL_REL = 1e-4                    # table gradient per level against float64, measured <= 3.2e-5
BWD_REL = dict(tk.BWD_REL, b2=2e-5)


def _cfg(hashmap_size=None):
    from neuralsim_b200.fields.encoding import auto_ngp_cfg
    cfg = auto_ngp_cfg([40., 150., 15.], 18 * 2 ** 17, dim=3, n_feats=2, log2_hashmap_size=16, min_res=16, max_num_levels=16)
    if hashmap_size:
        cfg["hashmap_size"] = hashmap_size
    return cfg


def _model(cfg, seed, **surface):
    from neuralsim_b200.fields.neus import LoTDNeuS
    gen = torch.Generator("cuda").manual_seed(seed)
    model = LoTDNeuS(surface_cfg=dict(aabb=AABB, sdf_scale=SDF_SCALE, encoding_cfg=dict(lotd_cfg=cfg), **surface),
                     radiance_cfg=dict(n_appear_embedding=4), device="cuda", generator=gen)
    with torch.no_grad():
        model.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=gen)
    assert model._color_fusable()
    return model


def _lidar_beam(rng):
    """a LiDAR beam (one of 64 elevations -17.6 .. 2.4 deg, random azimuth) from a sensor 2.2 m above z = -5.5 along the street
    -> (o, d) in network space (world / radius, so t is in metres), the unit world direction, and the t where the beam leaves the box"""
    elev = np.radians(rng.choice(np.linspace(-17.6, 2.4, 64)))
    az = rng.uniform(0, 2 * np.pi)
    dw = np.array([np.cos(elev) * np.sin(az), np.cos(elev) * np.cos(az), np.sin(elev)])
    ow = np.array([rng.uniform(-3, 3), rng.uniform(-60, 60), -3.3])
    o, d = ow / RADIUS, dw / RADIUS
    with np.errstate(divide="ignore"):
        a, b = (-0.995 - o) / d, (0.995 - o) / d
    return o, d, dw, float(np.maximum(a, b).min())


def _lidar_samples(n, seed):
    """n samples of LiDAR beams (_lidar_beam) in ray order with t ascending, 0.2 m apart from 1 m on, until the beam leaves the box.
    Network space: x = o / radius + (d / radius) t, t in metres."""
    rng = np.random.default_rng(seed)
    os_, ds, ts, total = [], [], [], 0
    while True:
        o, d, _, t1 = _lidar_beam(rng)
        t = 1.0 + rng.uniform(0, 0.2) + 0.2 * np.arange(int((t1 - 1.0) / 0.2))
        if total + len(t) >= n:
            t = t[:n - total]
        os_.append(o), ds.append(d), ts.append(t)
        total += len(t)
        if total == n:
            break
    lens = np.array([len(t) for t in ts])
    o = torch.tensor(np.stack(os_), dtype=torch.float32)
    d = torch.tensor(np.stack(ds), dtype=torch.float32)
    t = torch.tensor(np.concatenate(ts), dtype=torch.float32)
    ridx = torch.from_numpy(np.repeat(np.arange(len(ts)), lens))
    x = (d.double()[ridx] * t.double()[:, None] + o.double()[ridx]).float()        # the kernels' fma(d, t, o)
    assert float(x.abs().max()) < 1.0
    g = torch.Generator().manual_seed(seed)
    v = torch.nn.functional.normalize(d * torch.tensor(RADIUS, dtype=torch.float32), dim=-1)
    ha = torch.randn(len(ts), 4, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    pi = torch.stack([torch.from_numpy(np.cumsum(lens) - lens), torch.from_numpy(lens)], 1)
    return dict(x=x, o=o, d=d, t=t, ridx=ridx, v=v, ha=ha, cot=cot, pi=pi)


_CACHE = {}


def _case():
    if not _CACHE:
        cfg = _cfg()
        model = _model(cfg, seed=31)
        n = tk._size("color_fwd", 2)
        rnd = tk._inputs(n, 4, seed=41)
        ref = fused64.Fused64.from_model(model)
        _CACHE.update(cfg=cfg, meta=olotd.LoDMeta(3, **cfg), model=model, rnd=rnd, ref=ref, lidar=_lidar_samples(n, seed=43))
    return _CACHE


def _rays_fwd(model, inp):
    ridx, t, o, d = (inp[k].cuda() for k in ("ridx", "t", "o", "d"))
    return model.forward_on_rays(ridx, t, o, d, inp["v"].cuda(), inp["ha"].cuda())


def _ref_fwd(c, key):
    if key + "_fwd" not in c:
        inp = c[key]
        if key == "lidar":
            v, ha = inp["v"][inp["ridx"]], inp["ha"][inp["ridx"]]
        else:
            v, ha = inp["v"], inp["ha"]
        c[key + "_fwd"] = c["ref"].color_forward(inp["x"].numpy(), v.numpy(), ha.numpy())
    return c[key + "_fwd"]


def _per_level(meta, got, want, what, bound=LEVEL_REL):
    g = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
    errs = []
    for l in range(meta.n_levels):
        sl = slice(meta.level_offsets[l], meta.level_offsets[l + 1])
        assert np.abs(want[sl]).max() > 0, (what, l)
        errs.append(tk._rel(g[sl], want[sl]))
    print(f"METRIC {what} grid per level max={max(errs):.2e} " + " ".join(f"L{l}={e:.1e}" for l, e in enumerate(errs)))
    bad = [(l, e) for l, e in enumerate(errs) if not e < bound]
    assert not bad, (what, bad, bound)


def _others(got, want, what):
    rest = {k: v for k, v in want.items() if k != "grid"}
    tk._compare_grads({k: got[k] for k in rest}, rest, BWD_REL, what)


# ===================================================================================================================== geometry
def test_cfg3_geometry_and_merge_census():
    """the table is cuboid on every level, the nablas scale differs per axis, the merge is on for levels 0-7 and off for the levels
    where only some axes exceed 1024, and on the LiDAR samples it runs on most warps of the coarse levels"""
    c = _case()
    meta = c["meta"]
    res = np.array(meta.level_res_multidim)
    assert meta.n_levels == 16 and all(len(set(r)) == 3 for r in res.tolist())
    assert np.allclose(c["ref"].fac, SDF_SCALE / RADIUS, rtol=1e-6) and len(set(c["ref"].fac.tolist())) == 3
    mixed = [l for l in range(16) if (res[l] <= 1024).any() and (res[l] > 1024).any()]
    assert mixed == list(range(8, 15)) and (res[8:11, [0, 2]] <= 1024).all() and (res[8:11, 1] > 1024).all()
    cen = merge_census(c["lidar"]["x"].numpy(), c["cfg"])
    assert cen["mergeable"].tolist() == [True] * 8 + [False] * 8
    frac = (cen["heads"] <= MERGE_MAX_HEADS).mean(0)
    print("METRIC census lidar: fraction of warps that merge per level " + " ".join(f"L{l}={f:.2f}" for l, f in enumerate(frac)))
    assert (frac[:6] >= 0.5).all() and not frac[8:].any(), frac        # 0.2 m steps share cells up to level 5 (~0.3 m cells)


# ===================================================================================================================== forward
@pytest.mark.parametrize("inputs", ["random", "lidar"])
def test_sdf_forward(inputs):
    c = _case()
    model, ref = c["model"], c["ref"]
    s = model.implicit_surface
    if inputs == "random":
        n = tk._size("sdf_fwd", 2)
        tk._assert_multi_tile("sdf_fwd", n, 2)
        inp = tk._inputs(n, 4, seed=47)
        rows = tk._tile_rows(n)
    else:
        inp = c["lidar"]
        n = inp["x"].shape[0]
        rows = np.arange(n)
    x, ridx, t, o, d = tk._cuda(inp, "x", "ridx", "t", "o", "d")
    with torch.no_grad():
        got = dict(points=s.fused_sdf(x), rays=s.fused_sdf_rays(ridx, t, o, d))
        if inputs == "lidar":
            pi = inp["pi"].cuda()
            got["packs"] = s.fused_sdf_rays(ridx, t, o, d, packs=(pi, torch.arange(pi.shape[0], device="cuda")))
    want, scale = ref.sdf(inp["x"].numpy()[rows], with_scale=True)
    m = {k: tk._fp16_metrics(v.cpu().numpy()[rows], want, scale) for k, v in got.items()}
    print(f"METRIC cfg3 sdf_fwd {inputs} " + " ".join(f"{k}: flips={f:.2e} max_ulp={u:.2f}" for k, (f, u) in m.items()))
    for k, (frac, worst) in m.items():
        assert frac <= tk.SDF_FLIP_FRAC and worst <= tk.SDF_MAX_ULP, (k, frac, worst)


@pytest.mark.parametrize("inputs", ["rnd", "lidar"])
def test_color_forward_per_axis(inputs):
    c = _case()
    model, inp = c["model"], c[inputs]
    tk._assert_multi_tile("color_fwd", inp["x"].shape[0], 2)
    fwd = _ref_fwd(c, inputs)
    with torch.no_grad():
        got = _rays_fwd(model, inp) if inputs == "lidar" else tk._color_fwd(model, inp)
    sdf = tk._fp16_metrics(got["sdf"].cpu().numpy(), fwd["sdf"], fwd["sdf_scale"])
    rgb = tk._fp16_metrics(got["rgb"].cpu().numpy(), fwd["rgb"], 0.5)
    nab = np.abs(got["nablas"].cpu().numpy() - fwd["nablas"]) / (fwd["nablas_scale"] + 1e-30)
    print(f"METRIC cfg3 color_fwd {inputs} sdf: flips={sdf[0]:.2e} max_ulp={sdf[1]:.2f} rgb: flips={rgb[0]:.2e} max_ulp={rgb[1]:.2f} "
          f"nablas max_rel per axis=" + ",".join(f"{v:.2e}" for v in nab.max(0)))
    assert 0.01 < float((np.abs(fwd["nablas"]) < 1).mean())
    assert sdf[0] <= tk.SDF_FLIP_FRAC and sdf[1] <= tk.SDF_MAX_ULP, sdf
    assert rgb[0] <= tk.RGB_FLIP_FRAC and rgb[1] <= tk.RGB_MAX_ULP, rgb
    for ax in range(3):
        assert float(nab[:, ax].max()) <= tk.NAB_MAX_REL and float((nab[:, ax] > 1e-5).mean()) <= tk.NAB_FRAC_1E5, ax


# ===================================================================================================================== backward
@pytest.mark.parametrize("inputs", ["rnd", "lidar"])
def test_sdf_backward(inputs):
    c = _case()
    model, inp, meta = c["model"], c[inputs], c["meta"]
    tk._assert_multi_tile("sdf_bwd", inp["x"].shape[0], 2)
    d_sdf = inp["cot"][0].cuda()
    if inputs == "lidar":
        got = _sdf_bwd(model, None, d_sdf, rays=(inp["o"].cuda(), inp["d"].cuda(), inp["ridx"].cuda(), inp["t"].cuda()))
    else:
        p = tk._params(model)
        keys = ("grid", "W1", "b1", "W2", "b2")
        sdf = model.implicit_surface.fused_sdf_autograd(inp["x"].cuda())
        got = dict(zip(keys, torch.autograd.grad((sdf * d_sdf).sum(), [p[k] for k in keys])))
    want = c["ref"].sdf_backward(inp["x"].numpy(), inp["cot"][0].numpy())
    _per_level(meta, got["grid"], want["grid"], f"cfg3 sdf_bwd {inputs}")
    _others(got, want, f"cfg3 sdf_bwd {inputs}")


@pytest.mark.parametrize("cots", ["all", "lidar_no_rgb"])
@pytest.mark.parametrize("inputs", ["rnd", "lidar"])
def test_color_backward(inputs, cots):
    """k_color_rad_bwd + k_color_sdf_bwd with every cotangent set, and as LiDAR rays use it: sdf and nablas only (g_rgb = None)"""
    c = _case()
    model, inp, meta = c["model"], c[inputs], c["meta"]
    tk._assert_multi_tile("color_bwd", inp["x"].shape[0], 2)
    out = _rays_fwd(model, inp) if inputs == "lidar" else tk._color_fwd(model, inp)
    g_sdf, g_nab, g_rgb = (v.cuda() for v in inp["cot"])
    loss = (out["sdf"] * g_sdf).sum() + (out["nablas"] * g_nab).sum()
    if cots == "all":
        loss = loss + (out["rgb"] * g_rgb).sum()
    p = tk._params(model)
    keys = [k for k in p if cots == "all" or k[0] not in "Rr"]
    got = dict(zip(keys, torch.autograd.grad(loss, [p[k] for k in keys])))
    fwd = _ref_fwd(c, inputs)
    want = c["ref"].color_backward(fwd, inp["cot"][0].numpy(), inp["cot"][1].numpy(), inp["cot"][2].numpy() if cots == "all" else None)
    _per_level(meta, got["grid"], want["grid"], f"cfg3 color_bwd {inputs} {cots}")
    _others(got, {k: v for k, v in want.items() if k in keys}, f"cfg3 color_bwd {inputs} {cots}")


# ===================================================================================================================== merge edge
def _collision_warps(meta, n_warps, seed):
    """warps whose lanes alternate between cell A = (i, j, k) and cell B = (i, j - 1024, k + 1) of COLLIDE_LEVEL, k even: packed into
    10-bit fields, A's y field would carry into z and the two keys would be equal.  Network-space points [32 n_warps, 3]."""
    rng = np.random.default_rng(seed)
    scale = np.array(meta.level_res_multidim[COLLIDE_LEVEL]) - 2
    xs = np.empty((n_warps, 32, 3))
    for w in range(n_warps):
        i, j, k = rng.integers(1, scale[0] - 1), rng.integers(1024, scale[1]), 2 * rng.integers(1, (scale[2] - 2) // 2)
        cells = np.array([[i, j, k], [i, j - 1024, k + 1]] * 16, dtype=np.float64)
        xs[w] = (cells - 0.5 + rng.uniform(0.15, 0.85, (32, 3))) / scale
    x = (xs.reshape(-1, 3) * 2 - 1).astype(np.float32)
    cell, _ = olotd.pos_fract(fused64.Fused64.xs_of(x), scale.astype(np.float32))
    packed = cell[:, 0] | (cell[:, 1] << 10) | (cell[:, 2] << 20)
    a, b = cell[0::2], cell[1::2]
    assert (packed[0::2] == packed[1::2]).all() and (a[:, 1] - b[:, 1] == 1024).all() and (b[:, 2] - a[:, 2] == 1).all()
    return x


@pytest.mark.parametrize("kernel", ["sdf", "color"])
def test_merge_off_where_only_y_exceeds_1024(kernel):
    """the hand-built warps against float64, per level: each lane's update must land in its own cell"""
    c = _case()
    model, meta, ref = c["model"], c["meta"], c["ref"]
    x = _collision_warps(meta, 64, seed=5)
    n = x.shape[0]
    cen = merge_census(x, c["cfg"])
    assert not cen["mergeable"][COLLIDE_LEVEL] and (cen["heads"][:, COLLIDE_LEVEL] == 32).all()
    g = torch.Generator().manual_seed(6)
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    xt = torch.from_numpy(x)
    if kernel == "sdf":
        got = _sdf_bwd(model, None, cot[0].cuda(), x=xt.cuda())
        want = ref.sdf_backward(x, cot[0].numpy())
    else:
        inp = dict(x=xt, o=xt, d=torch.zeros(n, 3), t=torch.zeros(n), ridx=torch.arange(n),
                   v=torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1), ha=torch.randn(n, 4, generator=g) * 0.5)
        out = _rays_fwd(model, inp)
        p = tk._params(model)
        loss = sum((out[k] * v.cuda()).sum() for k, v in zip(("sdf", "nablas", "rgb"), cot))
        got = dict(grid=torch.autograd.grad(loss, [p["grid"]])[0])
        want = ref.color_backward(ref.color_forward(x, inp["v"].numpy(), inp["ha"].numpy()), *(v.numpy() for v in cot))
    _per_level(meta, got["grid"], want["grid"], f"cfg3 collision warps {kernel}")


# ===================================================================================================================== h % size
def test_hash_size_not_a_power_of_two():
    """the cfg3 table with 12289 hash cells: sdf forward per element and the sdf backward per level"""
    cfg = _cfg(12289)
    model = _model(cfg, seed=37)
    meta = olotd.LoDMeta(3, **cfg)
    ref = fused64.Fused64.from_model(model)
    n = tk._size("sdf_bwd", 2)
    inp = tk._inputs(n, 4, seed=53)
    s = model.implicit_surface
    x = inp["x"].cuda()
    with torch.no_grad():
        sdf = s.fused_sdf(x).cpu().numpy()
    want, scale = ref.sdf(inp["x"].numpy(), with_scale=True)
    frac, worst = tk._fp16_metrics(sdf, want, scale)
    print(f"METRIC cfg3 hash12289 sdf_fwd flips={frac:.2e} max_ulp={worst:.2f}")
    assert frac <= tk.SDF_FLIP_FRAC and worst <= tk.SDF_MAX_ULP
    got = _sdf_bwd(model, None, inp["cot"][0].cuda(), x=x)
    _per_level(meta, got["grid"], ref.sdf_backward(inp["x"].numpy(), inp["cot"][0].numpy())["grid"], "cfg3 hash12289 sdf_bwd")
