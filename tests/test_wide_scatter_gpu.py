"""The 48-column wgmma kernels (LoTD tables of 17..24 levels) against the float64 reference in the 48-column layout (tests/fused64_wide.py)
at the street geometry, on ray-ordered samples where the warp-merged table-gradient scatter runs on the wide levels 16..L-1.

Tables (bench_cfg3's box, 40 x 150 x 15 m, sdf_scale 25, so every level is cuboid and the nablas scale differs per axis):
  street17   the shipped camera models' table: auto_ngp_cfg with a 2^20 hashmap and 32 * 2^20 parameters, 17 levels (2 dense,
             15 hashed), the finest 8541 x 32030 x 3203
  street24   a 2^16 hashmap and 40 * 2^17 parameters: 24 levels (1 dense, 23 hashed), the finest 40916 x 153436 x 15343
  street17h  street17 with a hash size that is not a power of two (the `h % size` addressing on the wide levels)
Samples: LiDAR-like beams along the street (tests/test_tc_geometry_gpu.py:_lidar_beam) in ray order, each with 8..14 coarse samples and
33 samples within +-1 mm of a surface point (tests/test_tc_scatter_all_levels_gpu.py:_cluster_rays): 1 mm is below the finest cell of
both tables (~4.7 mm and ~1 mm on every axis), so consecutive samples share cells on every wide level and the merge runs there; the
same samples shuffled merge nowhere.  Every test asserts that census.
Covered: k_sdf_bwd_tc<., ., 48> from points, from rays and over a keep list; k_color_rad_bwd + k_color_sdf_bwd at 48 columns with every
cotangent, with ~30 % zero cotangents and without g_rgb; max_level None, 15 (every wide level gets exact zeros) and L - 3; the colour
forward per element; ray order against shuffled; hand-built warps on level 16 of street17 and level 21 of street24; the ray, view and
code gradients (k_sdf_bwd_tc<true, true, 48>, k_color_rad_bwd<A, R, 48>, k_color_sdf_bwd<true, 48>) against tests/rays64.py and
tests/appear64.py; the graph step's calls at 48 columns (the bodies of tests/test_tc_scatter_gpu.py's keep-list and device-count tests).
Bounds are those of tests/test_tc_geometry_gpu.py and tests/test_tc_scatter_gpu.py; DESIGN.md §4 lists the measured errors."""
import numpy as np
import pytest
import torch

import test_appear_grad_gpu as ag
import test_ray_grad_gpu as rg
import test_tc_geometry_gpu as tgeo
import test_tc_kernels_gpu as tk
import test_tc_scatter_all_levels_gpu as tsa
import test_tc_scatter_gpu as ts
from fused64_wide import Fused64Wide
from oracle import lotd as olotd
from rays64 import color_rows, ray_grads, sdf_rows

pytestmark = pytest.mark.gpu

LEVEL_REL, BWD_REL = tgeo.LEVEL_REL, tgeo.BWD_REL
ORDER_LEVEL_REL, ORDER_REL = ts.ORDER_LEVEL_REL, ts.ORDER_REL
# ray order against shuffled: b2 is the plain fp32 sum of the sdf cotangents, which cancels to ~1/sqrt(n) of its terms, so two summation
# orders differ by more than ORDER_REL of it (measured 5.1e-6 on street24); it keeps its float64 bound (BWD_REL["b2"]), as in
# tests/test_tc_geometry_gpu.py
ORDER_BOUNDS = {k: BWD_REL["b2"] if k == "b2" else ORDER_REL for k in tk.BWD_REL}
HALF = 1e-3                         # half width of a surface cluster in metres (t is in metres on these beams)
KEY_BITS = 21                       # cell_key3 (csrc/lotd_device.cuh): bits per axis
HAND_LEVEL = dict(street17=16, street24=21)


# ===================================================================================================================== tables
def _cfg(table):
    from neuralsim_b200.fields.encoding import auto_ngp_cfg
    if table == "street24":
        return auto_ngp_cfg([40., 150., 15.], 40 * 2 ** 17, dim=3, n_feats=2, log2_hashmap_size=16, min_res=16, max_num_levels=24)
    cfg = auto_ngp_cfg([40., 150., 15.], 32 * 2 ** 20, dim=3, n_feats=2, log2_hashmap_size=20, min_res=16, max_num_levels=24)
    if table == "street17h":
        cfg["hashmap_size"] = 3 * 2 ** 18 + 1
    return cfg


def _assert_table(table, cfg, ref):
    """level count, dense / hashed ladder, cuboid levels, fac per axis, every resolution inside the cell key"""
    meta = olotd.LoDMeta(3, **cfg)
    res = np.array(meta.level_res_multidim)
    L, dense = (24, 1) if table == "street24" else (17, 2)
    assert meta.n_levels == L and cfg["lod_types"] == ["Dense"] * dense + ["Hash"] * (L - dense), cfg["lod_types"]
    assert all(len(set(r)) == 3 for r in res.tolist()) and (res < 2 ** KEY_BITS).all()
    assert res[-1].tolist() == ([40916, 153436, 15343] if table == "street24" else [8541, 32030, 3203])
    size = cfg["hashmap_size"]
    assert (size & (size - 1) == 0) == (table != "street17h"), size
    assert np.allclose(ref.fac, tgeo.SDF_SCALE / tgeo.RADIUS, rtol=1e-6) and len(set(ref.fac.tolist())) == 3


def _street_beam(rng):
    o, d, dw, t1 = tgeo._lidar_beam(rng)
    return o, d, dw, 1.0, t1


_CACHE = {}


def _case(table):
    """model (max_fused_levels=24), ray-ordered street samples and their shuffle, built once per table"""
    if table not in _CACHE:
        cfg = _cfg(table)
        seed = dict(street17=131, street24=137, street17h=139)[table]
        model = tgeo._model(cfg, seed=seed, max_fused_levels=24)
        s = model.implicit_surface
        assert s.encoding.meta.n_pseudo_levels > 16 and s._fusable()
        inp = tsa._cluster_rays(tk._size("color_fwd", 2), 4, seed=seed + 1, beam=_street_beam, half=HALF)
        _CACHE[table] = dict(name=table, cfg=cfg, meta=olotd.LoDMeta(3, **cfg), model=model, inp=inp, refs={})
    return _CACHE[table]


def _ref(c, max_level):
    """Fused64Wide of the case's model at max_level, and its colour forward on the samples (built on first use, one max_level at a time)"""
    if max_level not in c["refs"]:
        c["refs"].clear()
        c["refs"][max_level] = dict(ref=Fused64Wide.from_model(c["model"], max_level=max_level))
    return c["refs"][max_level]["ref"]


def _fwd64(c, max_level):
    r = _ref(c, max_level)
    e = c["refs"][max_level]
    if "fwd" not in e:
        inp = c["inp"]
        e["fwd"] = r.color_forward(inp["x"].numpy(), inp["v"][inp["ridx"]].numpy(), inp["ha"][inp["ridx"]].numpy())
    return e["fwd"]


def _wide_levels(c):
    return list(range(16, c["meta"].n_levels))


def _assert_census(c, zero=None):
    """in ray order the merge runs on most warps of every wide level (and saves a third of their reductions); shuffled, nowhere"""
    tsa._assert_merges_on(c["inp"]["x"].numpy(), c["cfg"], _wide_levels(c), c["name"] + (" zero30" if zero is not None else ""), zero)


# ===================================================================================================================== geometry
@pytest.mark.parametrize("table", ["street17", "street24", "street17h"])
def test_street_tables_and_census(table):
    c = _case(table)
    _assert_table(table, c["cfg"], _ref(c, None))
    _assert_census(c)
    _assert_census(c, c["inp"]["zero"].numpy())


# ===================================================================================================================== float64
ML_CASES = [("street17", None), ("street17", 15), ("street17", 14), ("street24", None), ("street24", 15), ("street24", 21),
            ("street17h", None)]
ML_IDS = [f"{t}-ml{m}" for t, m in ML_CASES]


@pytest.mark.parametrize("table,max_level", ML_CASES, ids=ML_IDS)
def test_sdf_backward_float64(table, max_level):
    """k_sdf_bwd_tc<., ., 48> per level against float64: from points and from rays with every cotangent, from rays with ~30 % zero
    cotangents, and over the keep list of the non-zero ones (nsb_fused_sdf_bwd_indexed)"""
    c = _case(table)
    model, inp, meta = c["model"], c["inp"], c["meta"]
    ref = _ref(c, max_level)
    n = inp["x"].shape[0]
    tk._assert_multi_tile("sdf_bwd", n, 2)
    _assert_census(c, inp["zero"].numpy())
    cot = inp["cot"][0]
    zcot = ts._masked(inp["cot"], inp["zero"])[0]
    assert 0.2 < float((zcot == 0).float().mean()) < 0.4
    rays = ts._rays_cuda(inp)
    keep = torch.nonzero(zcot).flatten().cuda()
    got = dict(points=ts._sdf_bwd(model, max_level, cot.cuda(), x=inp["x"].cuda()), rays=ts._sdf_bwd(model, max_level, cot.cuda(), rays=rays),
               rays_zero30=ts._sdf_bwd(model, max_level, zcot.cuda(), rays=rays),
               indexed=ts._sdf_bwd(model, max_level, zcot.cuda(), rays=rays, keep=keep, n=keep.shape[0]))
    want = dict(all=ref.sdf_backward(inp["x"].numpy(), cot.numpy()), zero30=ref.sdf_backward(inp["x"].numpy(), zcot.numpy()))
    fails = []
    for route, g in got.items():
        w = want["all"] if route in ("points", "rays") else want["zero30"]
        ts._compare(g, w, f"wide f64 sdf_bwd {table} ml={max_level} {route}", LEVEL_REL, BWD_REL, max_level, fails, meta)
    assert not fails, fails


@pytest.mark.parametrize("table,max_level", ML_CASES, ids=ML_IDS)
def test_color_backward_float64(table, max_level):
    """k_color_rad_bwd + k_color_sdf_bwd at 48 columns per level against float64: every cotangent set, ~30 % zero cotangents (runs and
    isolated), and sdf and nablas only (g_rgb = None, as LiDAR rays use them)"""
    c = _case(table)
    model, inp, meta = c["model"], c["inp"], c["meta"]
    model.max_level = max_level
    try:
        tk._assert_multi_tile("color_bwd", inp["x"].shape[0], 2)
        _assert_census(c)
        out = ts._color_fwd(model, inp)
        assert torch.equal(out["x"].cpu(), inp["x"])
        ref, fwd = _ref(c, max_level), _fwd64(c, max_level)
        p = tk._params(model)
        fails = []
        for cots in ("all", "zero30", "no_rgb"):
            cot = ts._masked(inp["cot"], inp["zero"]) if cots == "zero30" else inp["cot"]
            g_sdf, g_nab, g_rgb = (v.cuda() for v in cot)
            loss = (out["sdf"] * g_sdf).sum() + (out["nablas"] * g_nab).sum()
            if cots != "no_rgb":
                loss = loss + (out["rgb"] * g_rgb).sum()
            keys = [k for k in p if cots != "no_rgb" or k[0] not in "Rr"]
            got = dict(zip(keys, torch.autograd.grad(loss, [p[k] for k in keys], retain_graph=True)))
            want = ref.color_backward(fwd, cot[0].numpy(), cot[1].numpy(), None if cots == "no_rgb" else cot[2].numpy())
            ts._compare(got, {k: v for k, v in want.items() if k in keys}, f"wide f64 color_bwd {table} ml={max_level} {cots}", LEVEL_REL,
                        BWD_REL, max_level, fails, meta)
        assert not fails, fails
    finally:
        model.max_level = None


def test_color_forward_per_element_street17():
    """k_color_fwd<true, 48> per element against float64, the nablas per axis"""
    c = _case("street17")
    model, inp = c["model"], c["inp"]
    tk._assert_multi_tile("color_fwd", inp["x"].shape[0], 2)
    fwd = _fwd64(c, None)
    with torch.no_grad():
        got = ts._color_fwd(model, inp)
    sdf = tk._fp16_metrics(got["sdf"].cpu().numpy(), fwd["sdf"], fwd["sdf_scale"])
    rgb = tk._fp16_metrics(got["rgb"].cpu().numpy(), fwd["rgb"], 0.5)
    nab = np.abs(got["nablas"].cpu().numpy() - fwd["nablas"]) / (fwd["nablas_scale"] + 1e-30)
    print(f"METRIC wide color_fwd street17 sdf: flips={sdf[0]:.2e} max_ulp={sdf[1]:.2f} rgb: flips={rgb[0]:.2e} max_ulp={rgb[1]:.2f} "
          f"nablas max_rel per axis=" + ",".join(f"{v:.2e}" for v in nab.max(0)))
    assert sdf[0] <= tk.SDF_FLIP_FRAC and sdf[1] <= tk.SDF_MAX_ULP, sdf
    assert rgb[0] <= tk.RGB_FLIP_FRAC and rgb[1] <= tk.RGB_MAX_ULP, rgb
    for ax in range(3):
        assert float(nab[:, ax].max()) <= tk.NAB_MAX_REL and float((nab[:, ax] > 1e-5).mean()) <= tk.NAB_FRAC_1E5, ax


# ===================================================================================================================== ray order
@pytest.mark.parametrize("table", ["street17", "street24"])
def test_ray_order_against_shuffled(table):
    """the three sdf routes and the colour pair on the ray-ordered samples (the merge runs on every wide level) against the same samples
    shuffled (nothing merges): only the fp32 summation order differs"""
    c = _case(table)
    model, inp, meta = c["model"], c["inp"], c["meta"]
    _assert_census(c)
    perm = inp["perm"]
    fails = []
    for route in ("points", "rays", "indexed"):
        a = ts._order_grads(route, model, inp, None)
        b = ts._order_grads(route, model, inp, perm)
        assert ts._all_finite(a) and ts._all_finite(b)
        ts._compare(b, a, f"wide order sdf_bwd {table} {route}", ORDER_LEVEL_REL, ORDER_BOUNDS, fails=fails, meta=meta)
    a, b = ts._color_fwd(model, inp), ts._color_fwd(model, inp, perm)
    for k in ("sdf", "nablas", "rgb", "x"):
        assert torch.equal(a[k][perm.cuda()], b[k]), k
    ga = tk._color_grads(model, a, inp["cot"])
    gb = tk._color_grads(model, b, tuple(v[perm] for v in inp["cot"]))
    assert ts._all_finite(ga) and ts._all_finite(gb)
    ts._compare(gb, ga, f"wide order color_bwd {table}", ORDER_LEVEL_REL, ORDER_BOUNDS, fails=fails, meta=meta)
    assert not fails, fails


# ===================================================================================================================== hand-built warps
@pytest.mark.parametrize("kernel", ["sdf", "color"])
@pytest.mark.parametrize("table", ["street17", "street24"])
def test_hand_built_warps_on_a_wide_level(table, kernel):
    """the ten run structures of tests/test_tc_scatter_gpu.py on level 16 of street17 and level 21 of street24, one warp's cotangent at
    a time, against float64 and against the same points interleaved with filler"""
    c = _case(table)
    level = HAND_LEVEL[table]
    tsa.hand_built_warps(c["model"], _ref(c, None), c["cfg"], level, kernel, f"wide hand {table} L{level}")


# ===================================================================================================================== the graph step's calls
def _graph_case():
    """street17 as the graph-step bodies of tests/test_tc_scatter_gpu.py take a case; the kept samples must merge on the coarse levels
    and on the wide level"""
    c = _case("street17")
    return dict(name="street17", model=c["model"], inp=c["inp"], ref=_ref(c, None), cfg=c["cfg"], meta=c["meta"], bwd_rel=BWD_REL,
                merge_levels=list(range(5)) + _wide_levels(c))


def test_indexed_sdf_backward_keep_list_and_device_count_street17():
    """nsb_fused_sdf_bwd_indexed at 48 columns over the keep list built by nsb_flag_nonzero and the scan, count on the host and
    device-resident"""
    ts.indexed_sdf_backward_keep_list_and_device_count(_graph_case())


def test_color_device_count_street17():
    """nsb_fused_color_fwd / nsb_fused_color_bwd at 48 columns under a device count below the capacity: NaN cotangents past the count,
    outputs there untouched"""
    ts.color_device_count(_graph_case())


# ===================================================================================================================== ray and code gradients
@pytest.mark.parametrize("table", ["street17", "street24"])
def test_ray_view_and_code_grads_float64(table):
    """the entry points of tests/test_ray_grad_gpu.py (nsb_fused_color_bwd_grads with and without rgb, nsb_fused_sdf_bwd_rays) and of
    tests/test_appear_grad_gpu.py (nsb_fused_color_bwd_appear) on the ray-ordered street samples against tests/rays64.py and
    tests/appear64.py in the 48-column layout"""
    c = _case(table)
    model, inp = c["model"], c["inp"]
    _assert_census(c)
    e = dict(inp, R=inp["o"].shape[0])
    ml = model.implicit_surface._ml(None)
    ref, fwd = _ref(c, None), _fwd64(c, None)
    ridx, t = inp["ridx"].numpy(), inp["t"].numpy()
    v = inp["v"].numpy()[ridx]
    cot = [x.numpy() for x in inp["cot"]]
    R = e["R"]
    outs, _ = rg._entry(model, e, ml)
    g_x, g_v = color_rows(ref, fwd, v, *cot)
    rg._check_entry(f"wide colour {table}", outs, ray_grads(g_x, t, ridx, R, g_v), e)
    outs, _ = rg._entry(model, e, ml, rgb=False)
    g_x, _ = color_rows(ref, fwd, v, cot[0], cot[1])
    rg._check_entry(f"wide geometry {table}", outs, ray_grads(g_x, t, ridx, R), e)
    outs, _ = rg._entry(model, e, ml, sdf=True)
    rg._check_entry(f"wide sdf {table}", outs, ray_grads(sdf_rows(ref, inp["x"].numpy(), cot[0]), t, ridx, R), e)
    got = ag._direct(model, e)
    ag._check_against_f64(model, e, got, f"wide {table}", ref=ref, fwd=fwd)
    assert torch.equal(got["dh"], ag._direct(model, e, appear=False)["dh"])
