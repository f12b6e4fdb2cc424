"""The five LoTD kernels of csrc/lotd.cu against the float64 oracle (oracle/lotd.py) at the table geometries the cfg3 street model
trains on, and at the ones the other instantiations see:

  G1  the shipped cfg3 table: auto_ngp_cfg([40, 150, 15], 32 Mi, 2^20), 17 cuboid levels (2 dense, 15 hashed), 17 pseudo levels
  G2  the same with max_num_levels=16 (the table of the fused path and of `bench.py --workload cfg3`)
  G3  the 4-D table of the distant model (tests/test_distant.py) plus a dense level that is cuboid in x / y / z
  G4  mixed widths 2 / 4: the 4-wide levels split into two pseudo levels that share a cell row
  G5  a hash table of 12289 cells (not a power of two: `h % size`)
  G6  the (D, F) = (3, 4) and (2, 2) instantiations

The kernels are called through the C ABI, so the table gradients are read as the kernels' fp32 accumulators (bindings._lotd rounds
them to the table dtype) and compared per pseudo level.  G1 and G2 run more than 8 waves of work items, so every thread of every
kernel walks its grid-stride loop; the oracle then runs on a sample of rows that spans every loop iteration, and the cotangents are
non-zero only on that sample while the kernels run over all points.  The inputs put points on cell boundaries, at the clamp limits,
and ~30 % of the cotangent rows at zero.

Also here: the autograd glue of fields/encoding.py (loss scale, `x/2+0.5`) at 17 levels, and the reference project's own kernels at
the cuboid and 4-D geometries (tests/golden/ref__lotd_geometry.npz, recorded from oracle/_ref/_lotd as tests/refgold.py describes).
Bounds are about 3x the errors measured on an H100 80GB HBM3 (132 SMs, 400 W power limit); DESIGN.md §4 lists them."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import lotd as olotd
from refgold import Golden

pytestmark = pytest.mark.gpu

BLOCK, CTAS_PER_SM, MAX_WAVES = 256, 4, 8          # wave_grid(n, 256, 4) of every lotd.cu launch (csrc/nsb_common.cuh)


def _cfg3(max_num_levels):
    from neuralsim_b200.fields.encoding import auto_ngp_cfg
    return auto_ngp_cfg([40., 150., 15.], 32 * 2 ** 20, dim=3, n_feats=2, log2_hashmap_size=20, min_res=16, max_num_levels=max_num_levels)


def _distant_plus_cuboid():
    from test_distant import _cfg
    c = _cfg()
    return dict(lod_res=c["lod_res"] + [[7, 11, 5, 4]], lod_n_feats=c["lod_n_feats"] + [2], lod_types=c["lod_types"] + ["Dense"],
                hashmap_size=c["hashmap_size"])


# id -> (n_dims, LoTD configuration, points; 0: enough for every thread to loop, the oracle on a row sample)
GEOMS = {
    "G1": (3, lambda: _cfg3(None), 0),
    "G2": (3, lambda: _cfg3(16), 0),
    "G3": (4, _distant_plus_cuboid, 20000),
    "G4": (3, lambda: dict(lod_res=[[6, 9, 5], [9, 13, 7], [13, 19, 10], [19, 28, 14], [28, 41, 21], [41, 60, 30]],
                           lod_n_feats=[2, 4, 2, 4, 2, 4], lod_types=["Dense"] * 3 + ["Hash"] * 3, hashmap_size=2 ** 13), 20000),
    "G5": (3, lambda: dict(lod_res=[[8, 12, 5], [12, 18, 7], [18, 27, 10], [27, 40, 15], [40, 60, 22], [60, 90, 33], [90, 135, 50]],
                           lod_n_feats=[2] * 7, lod_types=["Dense"] * 2 + ["Hash"] * 5, hashmap_size=12289), 20000),
    "G6a": (3, lambda: dict(lod_res=[[6, 10, 4], [10, 17, 6], [17, 29, 9], [29, 49, 15], [49, 83, 25]], lod_n_feats=[4] * 5,
                            lod_types=["Dense"] * 2 + ["Hash"] * 3, hashmap_size=2 ** 12), 20000),
    "G6b": (2, lambda: dict(lod_res=[[5, 9], [9, 17], [17, 33], [33, 65], [65, 129], [129, 257]], lod_n_feats=[2] * 6,
                            lod_types=["Dense"] * 3 + ["Hash"] * 3, hashmap_size=2 ** 11), 20000),
}
SAMPLE = 6000                # oracle rows of G1 / G2

# Bounds, rel-L2 per pseudo level of the fp32 kernel result against float64 (measured values in DESIGN.md §4).  The table gradients of
# G1 / G2 sum few points per table entry (6000 sample rows over 2^20 cells per level); the small tables sum tens to hundreds, so their
# fp32 atomics round more often.
GRID_REL = dict(G1=1.5e-7, G2=1.5e-7)   # bwd_grid and bwd_bwd_grid table gradients, measured <= 4.6e-8
GRID_REL_SMALL = 2.5e-6                 # the same on G3..G6, measured <= 8.3e-7
INPUT_REL = 2e-7                        # dL_dx per axis, dL_d(dL_dy) per pseudo level, measured <= 5.9e-8


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stride(work_items):
    """threads of a lotd.cu launch over `work_items` (wave_grid): the grid-stride loop's stride"""
    wave = _sms() * CTAS_PER_SM
    need = -(-work_items // BLOCK)
    blocks = need if need <= wave else min(-(-need // wave), MAX_WAVES) * wave
    return blocks * BLOCK


def _boundary_points(rng, meta, n):
    """points with x (res-2) + 0.5 an integer, exactly in fp32, on one axis of some level (a cell boundary: frac = 0)"""
    D = meta.n_dims_to_encode
    x = rng.uniform(0.05, 0.95, (n, D)).astype(np.float32)
    for i in range(n):
        l, d = rng.integers(meta.n_levels), rng.integers(D)
        s = meta.level_res_multidim[l][d] - 2
        x[i, d] = np.float32((rng.integers(1, s) - 0.5) / s)
    return x


def _clamp_points(D):
    """every combination of the two clamp limits and the centre over the axes"""
    v = np.array([1e-6, 1 - 1e-6, 0.5], dtype=np.float32)
    g = np.stack(np.meshgrid(*[v] * D, indexing="ij"), -1).reshape(-1, D)
    return g.astype(np.float32)


class Geom:
    def __init__(self, gid):
        from neuralsim_b200.bindings import _lotd
        self.gid = gid
        D, make, n = GEOMS[gid]
        self.D, self.cfg = D, make()
        self.om = olotd.LoDMeta(D, **self.cfg)
        self.gm = _lotd.LoDMeta(D, self.cfg["lod_res"], self.cfg["lod_n_feats"], self.cfg["lod_types"], self.cfg["hashmap_size"])
        om, gm = self.om, self.gm
        assert (gm.n_params, gm.level_offsets, gm.level_sizes, gm.map_levels, gm.map_cnt, gm.level_res_multidim) == \
               (om.n_params, om.level_offsets, om.level_sizes, om.map_levels, om.map_cnt, om.level_res_multidim)
        rng = np.random.default_rng(sum(map(ord, gid)))
        self.p16 = rng.uniform(-0.5, 0.5, om.n_params).astype(np.float16)
        big = n == 0
        if big:        # more than 8 waves of points: every thread of every launch loops at least twice
            s = _stride(1 << 40)
            n = 2 * s + s // 3 + 77
        self.n = n
        x = rng.uniform(1e-6, 1 - 1e-6, (n, D)).astype(np.float32)
        self.rows = np.unique(np.concatenate([rng.choice(n, SAMPLE, replace=False), [0, n - 1]])) if big else np.arange(n)
        S = len(self.rows)
        special = np.concatenate([_clamp_points(D), _boundary_points(rng, om, S // 5)])
        at = rng.choice(S, len(special), replace=False)
        x[self.rows[at]] = special
        self.x = x
        self.xr = x[self.rows]
        # cotangents on the sample rows only, ~30 % of those rows zero
        g = (rng.normal(size=(S, om.n_encoded_dims)) * 0.1).astype(np.float16)
        g[rng.random(S) < 0.3] = 0
        gin = rng.normal(size=(S, D)).astype(np.float32)
        gin[rng.random(S) < 0.3] = 0
        self.g, self.gin = g, gin
        self.ml_mid = om.n_levels // 2 - 1

    def check_layout(self):
        """the input layout the comparisons rely on, asserted"""
        om, xr = self.om, self.xr
        frac0 = 0
        for l in range(om.n_levels):
            _, fr = olotd.pos_fract(xr, (np.array(om.level_res_multidim[l]) - 2).astype(np.float32))
            frac0 += int((fr == 0).any(1).sum())
        assert frac0 >= len(xr) // 5, frac0
        lim = np.float32(1 - 1e-6)
        assert ((xr == np.float32(1e-6)).all(1).any() and (xr == lim).all(1).any() and ((xr == lim) & (np.roll(xr, 1, 1) == np.float32(1e-6))).any())
        zero = (self.g == 0).all(1).mean()
        assert 0.2 < zero < 0.4, zero
        if self.n > len(self.rows):
            for items, per in ((self.n, 1), (self.n * om.n_pseudo_levels, om.n_pseudo_levels), (self.n * om.n_encoded_dims, om.n_encoded_dims)):
                s = _stride(items)
                iters = -(-items // s)
                assert iters >= 2 and s == MAX_WAVES * _sms() * CTAS_PER_SM * BLOCK, (items, s)
                hit = np.unique((self.rows[:, None] * per + np.arange(per)[None, :]) // s)
                assert np.array_equal(hit, np.arange(iters)), (per, iters, hit.size)

    # ------------------------------------------------------------------ kernels through the C ABI
    def fwd(self, params, ml, dydx=True):
        from neuralsim_b200 import _lib as L
        n, F, D = self.n, self.gm.n_encoded_dims, self.D
        y = torch.empty((n, F), dtype=params.dtype, device="cuda")
        d = torch.empty((n, F * D), dtype=torch.float32, device="cuda") if dydx else None
        L.check(L.lib().nsb_lotd_fwd(self.gm.c_ref, L.ptr(self.xg, "f32"), L.ptr(params), ctypes.c_int(params.dtype == torch.float16),
                                     L.c_i64(n), L.c_i32(ml), L.ptr(y), L.ptr(d, "f32", allow_none=True), L.stream_ptr()), "lod_fwd")
        return y, d

    def full(self, rows_val, dtype):
        out = torch.zeros((self.n,) + rows_val.shape[1:], dtype=dtype)
        out[torch.from_numpy(self.rows)] = torch.from_numpy(rows_val).to(dtype)
        return out.cuda()

    def bwd(self, ml, dy_dx):
        from neuralsim_b200 import _lib as L
        n, gm = self.n, self.gm
        g = self.full(self.g, torch.float16)
        acc = torch.zeros(gm.n_params, dtype=torch.float32, device="cuda")
        dx = torch.empty((n, self.D), dtype=torch.float32, device="cuda")
        L.check(L.lib().nsb_lotd_bwd_grid(gm.c_ref, L.ptr(g), 1, L.ptr(self.xg, "f32"), L.c_i64(n), L.c_i32(ml), L.c_f32(1.0), L.ptr(acc),
                                          L.stream_ptr()), "bwd_grid")
        L.check(L.lib().nsb_lotd_bwd_input(L.ptr(g), 1, L.ptr(dy_dx, "f32"), L.c_i64(n), L.c_i32(gm.n_encoded_dims), L.c_i32(self.D),
                                           L.c_f32(1.0), L.ptr(dx), L.stream_ptr()), "bwd_input")
        gin = self.full(self.gin, torch.float32)
        ddy = torch.empty((n, gm.n_encoded_dims), dtype=torch.float32, device="cuda")
        acc2 = torch.zeros(gm.n_params, dtype=torch.float32, device="cuda")
        L.check(L.lib().nsb_lotd_bwd_bwd_input(gm.c_ref, L.ptr(gin, "f32"), L.ptr(g), 1, L.ptr(self.xg, "f32"), L.ptr(dy_dx, "f32"),
                                               L.c_i64(n), L.c_i32(ml), L.c_f32(1.0), L.ptr(ddy), L.ptr(acc2), L.stream_ptr()), "bwd_bwd")
        return acc, dx, ddy, acc2

    # ------------------------------------------------------------------ per pseudo level views
    def pseudo_slices(self):
        """pseudo level -> (level, index array of its table elements, output columns)"""
        om, F = self.om, self.om.n_feat_per_pseudo_lvl
        out = []
        for p in range(om.n_pseudo_levels):
            l = om.map_levels[p]
            nf = om.level_n_feats[l]
            base = om.level_offsets[l] + om.map_cnt[p] * F
            idx = (base + np.arange(om.level_sizes[l])[:, None] * nf + np.arange(F)[None, :]).ravel()
            out.append((l, idx, slice(p * F, (p + 1) * F)))
        return out


_GEOMS = {}


@pytest.fixture(scope="module", params=list(GEOMS))
def geom(request):
    """module scope: the tests of one geometry run together and build it once"""
    gid = request.param
    if gid not in _GEOMS:
        _GEOMS.clear()
        G = Geom(gid)
        G.xg = torch.from_numpy(G.x).cuda()
        G.pg16 = torch.from_numpy(G.p16).cuda()
        _GEOMS[gid] = G
    return _GEOMS[gid]


def _rel(got, want):
    got, want = np.asarray(got, dtype=np.float64).ravel(), np.asarray(want, dtype=np.float64).ravel()
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-300))


def _levels(G):
    """max_level values: all levels, only the last level masked, a middle level"""
    return [G.om.n_levels, G.om.n_levels - 2, G.ml_mid]


# ===================================================================================================================== forward
def test_geometry_layout(geom):
    G = geom
    G.check_layout()
    cuboid = [l for l, r in enumerate(G.om.level_res_multidim) if len(set(r[:3])) == 3]
    dense_cuboid = [l for l in cuboid if G.om.level_types[l] == olotd.DENSE]
    if G.gid in ("G1", "G2"):
        assert cuboid == list(range(G.om.n_levels)) and dense_cuboid == [0, 1]
        assert G.om.n_pseudo_levels == (17 if G.gid == "G1" else 16)
    elif G.gid == "G3":
        assert dense_cuboid == [4] and G.D == 4
    elif G.gid == "G4":
        assert G.om.n_pseudo_levels == 9 and G.om.n_feat_per_pseudo_lvl == 2
    elif G.gid == "G5":
        assert G.om.level_sizes[-1] == 12289 and dense_cuboid == [0, 1]
    elif G.gid == "G6a":
        assert G.om.n_feat_per_pseudo_lvl == 4
    else:
        assert G.D == 2


def test_forward_fp16(geom):
    """y bit-exact, dy_dx to ~1e-6; levels above max_level exactly zero"""
    G = geom
    F = G.om.n_feat_per_pseudo_lvl
    for ml in _levels(G):
        y, d = G.fwd(G.pg16, ml)
        y_ref, d_ref = olotd.lod_fwd(G.om, G.xr, G.p16, max_level=ml, need_input_grad=True)
        rows = torch.from_numpy(G.rows).cuda()
        yr, dr = y[rows].cpu().numpy(), d[rows].view(len(G.rows), -1, G.D).cpu().numpy()
        assert np.array_equal(yr.view(np.uint16), y_ref.view(np.uint16)), (ml, int((yr.view(np.uint16) != y_ref.view(np.uint16)).sum()))
        err = np.abs(dr - d_ref) / (np.abs(d_ref) + 1e-7)
        print(f"METRIC lotd_fwd {G.gid} ml={ml} dy_dx max rel={err.max():.2e}")
        assert np.allclose(dr, d_ref, rtol=1e-6, atol=1e-7), (ml, err.max())
        off = [p for p, l in enumerate(G.om.map_levels) if l > ml]
        if off:
            cols = np.concatenate([np.arange(p * F, (p + 1) * F) for p in off])
            assert float(y[:, cols].abs().max()) == 0 and float(d.view(G.n, -1, G.D)[:, cols].abs().max()) == 0


def test_forward_fp32(geom):
    G = geom
    p32 = (G.p16.astype(np.float32) + np.float32(1e-4) * np.sign(G.p16)).astype(np.float32)     # values that fp16 cannot hold
    for ml in (G.om.n_levels, G.ml_mid):
        y, _ = G.fwd(torch.from_numpy(p32).cuda(), ml, dydx=False)
        y_ref, _ = olotd.lod_fwd(G.om, G.xr, p32, max_level=ml)
        yr = y[torch.from_numpy(G.rows).cuda()].cpu().numpy()
        print(f"METRIC lotd_fwd32 {G.gid} ml={ml} max abs={np.abs(yr - y_ref).max():.2e}")
        assert y.dtype == torch.float32 and np.allclose(yr, y_ref, rtol=1e-6, atol=1e-7), ml


# ===================================================================================================================== backward
def test_backward_per_pseudo_level(geom):
    """bwd_grid, bwd_input, ddLdy and bwd_bwd_grid against float64, per pseudo level; nothing above max_level"""
    G = geom
    om = G.om
    rows = torch.from_numpy(G.rows).cuda()
    slices = G.pseudo_slices()
    fails = []
    for ml in (om.n_levels, G.ml_mid):
        _, d = G.fwd(G.pg16, ml)
        acc, dx, ddy, acc2 = G.bwd(ml, d)
        _, J = olotd.lod_fwd(om, G.xr, G.p16, max_level=ml, need_input_grad=True)
        gp_ref = olotd.lod_bwd_grid(om, G.g, G.xr, om.n_params, ml)
        dx_ref = olotd.lod_bwd_input(G.g, J)
        ddy_ref, gp2_ref, _ = olotd.lod_bwd_bwd_input(om, G.gin, G.g, G.xr, G.p16, J, ml)
        a, a2 = acc.double().cpu().numpy(), acc2.double().cpu().numpy()
        ddy_r = ddy[rows].cpu().numpy()
        errs = dict(grid=[], bwd_bwd=[], ddLdy=[])
        for p, (l, idx, cols) in enumerate(slices):
            if l > ml:
                if np.any(a[idx] != 0) or np.any(a2[idx] != 0) or np.any(ddy_r[:, cols] != 0):
                    fails.append((ml, "non-zero above max_level", p))
                continue
            for k, got, want in (("grid", a[idx], gp_ref[idx]), ("bwd_bwd", a2[idx], gp2_ref[idx]), ("ddLdy", ddy_r[:, cols], ddy_ref[:, cols])):
                if not np.abs(want).max() > 0:
                    fails.append((ml, k, p, "no reference gradient"))
                e = _rel(got, want)
                errs[k].append(e)
                if not e < (GRID_REL.get(G.gid, GRID_REL_SMALL) if k != "ddLdy" else INPUT_REL):
                    fails.append((ml, k, p, e))
        dx_r = dx[rows].cpu().numpy()
        errs["dL_dx"] = [_rel(dx_r[:, k], dx_ref[:, k]) for k in range(G.D)]
        fails += [(ml, "dL_dx", k, e) for k, e in enumerate(errs["dL_dx"]) if not e < INPUT_REL]
        # points off the sample carry zero cotangents: nothing may reach them
        mask = torch.ones(G.n, dtype=torch.bool, device="cuda")
        mask[rows] = False
        if float(dx[mask].abs().max() if mask.any() else 0) != 0 or float(ddy[mask].abs().max() if mask.any() else 0) != 0:
            fails.append((ml, "output on a row without cotangent"))
        print(f"METRIC lotd_bwd {G.gid} ml={ml} " + " ".join(f"{k}: max={max(v):.2e}" for k, v in errs.items())
              + " | grid per pseudo level " + " ".join(f"{e:.1e}" for e in errs["grid"]))
    assert not fails, fails


def test_bindings_dtype_and_shapes(geom):
    """the same kernels through bindings._lotd: shapes, dtypes (gradients rounded to the table dtype) and the fp16 forward"""
    from neuralsim_b200.bindings import _lotd
    G = geom
    om = G.om
    rows = torch.from_numpy(G.rows).cuda()
    xs = G.xg[rows].contiguous()
    y, d = _lotd.lod_fwd(G.gm, xs, G.pg16, None, None, None, None, True)
    assert y.dtype == torch.float16 and y.shape == (len(G.rows), om.n_encoded_dims) and d.shape == (len(G.rows), om.n_encoded_dims * G.D)
    y_ref, _ = olotd.lod_fwd(om, G.xr, G.p16)
    assert np.array_equal(y.cpu().numpy().view(np.uint16), y_ref.view(np.uint16))
    g = torch.from_numpy(G.g).cuda()
    gx, gp = _lotd.lod_bwd(G.gm, g, xs, G.pg16, d, None, None, None, None, True, True)
    assert gx.dtype == torch.float32 and gx.shape == (len(G.rows), G.D) and gp.dtype == torch.float16 and gp.shape == (om.n_params,)
    ref = olotd.lod_bwd_grid(om, G.g, G.xr, om.n_params)
    absum = olotd.lod_bwd_grid(om, np.abs(G.g), G.xr, om.n_params)        # sum of the magnitudes of each entry's terms (weights >= 0)
    got = gp.double().cpu().numpy()
    # one fp16 rounding of the fp32 sum, whose own rounding error is a small multiple of 2^-24 of its terms' magnitudes (hundreds of
    # terms per entry on the coarse levels of the small tables)
    assert np.all(np.abs(got - ref) <= 2.0 ** -11 * np.abs(ref) + 2.0 ** -18 * absum + 2.0 ** -24)
    a, b, c = _lotd.lod_bwd_bwd_input(G.gm, torch.from_numpy(G.gin).cuda(), g, xs, G.pg16, d, None, None, None, None, True, True, False)
    assert c is None and a.dtype == torch.float16 and a.shape == (len(G.rows), om.n_encoded_dims) and b.dtype == torch.float16


# ===================================================================================================================== glue
def test_encoding_autograd_glue_17_levels(cuda):
    """LoTDEncoding.forward_dydx -> backward_dydx -> autograd at G1: the loss scale 128 on the fp16 dL_dy, the division by it after
    the fp16 table gradient and the `x/2+0.5` chain rule, against float64 with the same factors written out"""
    from neuralsim_b200.fields.encoding import LoTDEncoding
    cfg = _cfg3(None)
    om = olotd.LoDMeta(3, **cfg)
    gen = torch.Generator("cuda").manual_seed(3)
    enc = LoTDEncoding(3, lotd_cfg=cfg, device=cuda, generator=gen)
    with torch.no_grad():
        enc.flattened_params.uniform_(-0.5, 0.5, generator=gen)
    assert enc.lotd.loss_scale == 128.0 and om.n_levels == 17
    rng = np.random.default_rng(4)
    n = 20000
    x = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    x[:4] = [[-1, -1, -1], [1, 1, 1], [1, -1, 0.3], [-0.99, 0.999, -0.5]]
    # magnitudes of a training step: fp16 values of dL_dy times 128, and of the second-order table gradient (the finest level scales
    # by res - 2 = 32028), stay well inside the fp16 range
    dLdy = (rng.normal(size=(n, om.n_encoded_dims)) * 1e-3).astype(np.float16)
    cot_y = rng.normal(size=(n, om.n_encoded_dims)).astype(np.float32)
    cot_n = (rng.normal(size=(n, 3)) * 0.1).astype(np.float32)
    xg = torch.from_numpy(x).cuda()
    dLdy_g = torch.from_numpy(dLdy).cuda().requires_grad_(True)
    y, dydx = enc.forward_dydx(xg)
    nablas = enc.backward_dydx(dLdy_g, dydx, xg)
    loss = (y.float() * torch.from_numpy(cot_y).cuda()).sum() + (nablas * torch.from_numpy(cot_n).cuda()).sum()
    g_table, g_dLdy = torch.autograd.grad(loss, [enc.flattened_params, dLdy_g])

    # float64, the factors of fields/encoding.py written out
    s = 128.0
    p16 = enc.flattened_params.detach().half().cpu().numpy()
    xs = np.clip((x * np.float32(0.5) + np.float32(0.5)).astype(np.float32), np.float32(1e-6), np.float32(1 - 1e-6))
    y_ref, J = olotd.lod_fwd(om, xs, p16, need_input_grad=True)
    assert np.array_equal(y.detach().cpu().numpy().view(np.uint16), y_ref.view(np.uint16))
    scaled = (dLdy.astype(np.float32) * np.float32(s)).astype(np.float16)
    nab_ref = olotd.lod_bwd_input(scaled, J).astype(np.float64) / s / 2.0
    nab_scale = np.einsum("nf,nfd->nd", np.abs(scaled.astype(np.float64)), np.abs(J.astype(np.float64))) / s / 2.0
    gin = cot_n / np.float32(2.0)                                              # d nablas / d(dL_dx): 1/2
    a = olotd.lod_bwd_grid(om, (cot_y.astype(np.float16).astype(np.float32) * np.float32(s)).astype(np.float16), xs, om.n_params) / s
    _, b, _ = olotd.lod_bwd_bwd_input(om, gin, scaled, xs, p16, J, need_dLdy=False)
    b = b / s
    ddLdy_ref = np.einsum("nd,nfd->nf", gin.astype(np.float64), J.astype(np.float64))
    ddLdy_scale = np.einsum("nd,nfd->nf", np.abs(gin.astype(np.float64)), np.abs(J.astype(np.float64)))       # fp32 sum over 3 axes
    nab_err = np.abs(nablas.detach().double().cpu().numpy() - nab_ref) / (nab_scale + 1e-30)
    got_t = g_table.double().cpu().numpy()
    tab_err = np.abs(got_t - (a + b)) / (2.0 ** -10 * (np.abs(a) + np.abs(b)) + 2.0 ** -23)
    got_y = g_dLdy.double().cpu().numpy()
    y_err = np.abs(got_y - ddLdy_ref) / (2.0 ** -10 * np.abs(ddLdy_ref) + 2.0 ** -22 * ddLdy_scale + 2.0 ** -24)
    print(f"METRIC lotd_glue nablas max err / scale={nab_err.max():.2e} table max err / bound={tab_err.max():.2e} "
          f"dL_dy max err / bound={y_err.max():.2e}")
    assert nab_err.max() < 1e-5
    assert np.isfinite(got_t).all() and tab_err.max() <= 1.0 and np.abs(a).max() > 0 and np.abs(b).max() > 0
    assert y_err.max() <= 1.0


# ===================================================================================================================== reference kernels
# sizes of what the golden file keeps per geometry (rows of dense outputs, entries of the sparse gradient samples): enough for the
# comparisons' statistics, small enough for a test vector
D_ROWS, GX_ROWS, A_ROWS, N_SAMPLE = 100, 1000, 500, 3000


def _rows(t, n):
    return t.detach().reshape(t.shape[0], -1)[:n].cpu()


def _support_sample(t, n, seed):
    nz = torch.nonzero(t.detach().reshape(-1).float() != 0).squeeze(-1).cpu()
    g = torch.Generator().manual_seed(seed)
    return nz[torch.randperm(nz.numel(), generator=g)[:n]].sort().values.int()


def test_against_reference_kernels(cuda):
    """the reference project's own _lotd kernels on the cuboid 3-D (G1) and the 4-D (G3) table: y bit-exact, dy_dx rows, gradient
    samples (the reference accumulates in fp16 atomics, so those keep the tolerance of test_ref_parity_gpu.py)"""
    G = Golden("_lotd_geometry", "_lotd")
    for gid in ("G1", "G3"):
        _against_reference(cuda, G, gid)
    G.save()


def _against_reference(cuda, G, gid):
    from neuralsim_b200.bindings import _lotd as ours
    D, make, _ = GEOMS[gid]
    cfg = make()
    rmeta = lambda ref: ref.LoDMeta(D, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"], False)
    om = ours.LoDMeta(D, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"])
    sizes = G.value(f"{gid}.meta", lambda ref: torch.tensor([rmeta(ref).n_params] + list(rmeta(ref).level_offsets) + list(rmeta(ref).level_sizes)))
    assert sizes.tolist() == [om.n_params] + list(om.level_offsets) + list(om.level_sizes)
    rng = np.random.default_rng(7)
    n = 60000
    p = torch.from_numpy(rng.uniform(-0.5, 0.5, om.n_params).astype(np.float16)).to(cuda)
    xn = rng.uniform(1e-6, 1 - 1e-6, (n, D)).astype(np.float32)
    xn[:3 ** D] = _clamp_points(D)
    x = torch.from_numpy(xn).to(cuda)
    g = torch.from_numpy((rng.normal(size=(n, om.n_encoded_dims)) * 0.05).astype(np.float16)).to(cuda)
    gin = torch.from_numpy((rng.normal(size=(n, D)) * 0.01).astype(np.float32)).to(cuda)      # fp16 dL_d(dL_dy) stays finite at res 32030
    ref_fwd = lambda ref: ref.lod_fwd(rmeta(ref), x, p, None, None, None, None, True)
    y_o, d_o = ours.lod_fwd(om, x, p, None, None, None, None, True)
    G.equal(f"{gid}.y", y_o.view(torch.int16), lambda ref: ref_fwd(ref)[0].contiguous().view(torch.int16))
    d_r = G.value(f"{gid}.d_rows", lambda ref: _rows(ref_fwd(ref)[1].reshape(d_o.shape), D_ROWS))
    assert torch.allclose(d_r, _rows(d_o, D_ROWS), rtol=1e-6, atol=1e-7)
    cm = olotd.LoDMeta(D, **cfg)                                           # and the CPU oracle, on the same rows
    y_c, d_c = olotd.lod_fwd(cm, xn[:3000], p.cpu().numpy(), need_input_grad=True)
    G.equal(f"{gid}.y3000", torch.from_numpy(np.ascontiguousarray(y_c)).view(torch.int16),
            lambda ref: ref_fwd(ref)[0].contiguous()[:3000].view(torch.int16))
    assert np.allclose(d_c.reshape(3000, -1)[:D_ROWS], d_r.numpy(), rtol=1e-6, atol=1e-7)
    ml = om.n_levels - 2
    b, _ = ours.lod_fwd(om, x, p, None, None, None, ml, False)
    G.equal(f"{gid}.y_max_level{ml}", b.view(torch.int16), lambda ref: ref.lod_fwd(rmeta(ref), x, p, None, None, None, ml, False)[0].contiguous().view(torch.int16))
    ref_bwd = lambda ref: ref.lod_bwd(rmeta(ref), g, x, p, ref_fwd(ref)[1], None, None, None, None, True, True)
    gx_o, gp_o = ours.lod_bwd(om, g, x, p, d_o, None, None, None, None, True, True)
    gx_r = G.value(f"{gid}.gx_rows", lambda ref: _rows(ref_bwd(ref)[0], GX_ROWS))
    assert torch.allclose(gx_r, _rows(gx_o, GX_ROWS), rtol=1e-4, atol=1e-4)
    idx = G.value(f"{gid}.gp_idx", lambda ref: _support_sample(ref_bwd(ref)[1], N_SAMPLE, 1)).long()
    gp_r = G.value(f"{gid}.gp_sample", lambda ref: ref_bwd(ref)[1].reshape(-1)[idx.to(cuda)])
    gp_s = gp_o.reshape(-1)[idx.to(cuda)].float().cpu()
    err = float((gp_r.float() - gp_s).norm() / gp_s.norm())
    ref_bb = lambda ref: ref.lod_bwd_bwd_input(rmeta(ref), gin, g, x, p, ref_fwd(ref)[1].contiguous(), None, None, None, None, True, True, False)
    a_o, b_o, _ = ours.lod_bwd_bwd_input(om, gin, g, x, p, d_o, None, None, None, None, True, True, False)
    a_r = G.value(f"{gid}.a_rows", lambda ref: _rows(ref_bb(ref)[0], A_ROWS))
    a_err = float((a_r.float() - _rows(a_o, A_ROWS).float()).norm() / _rows(a_o, A_ROWS).float().norm())
    bidx = G.value(f"{gid}.b_idx", lambda ref: _support_sample(ref_bb(ref)[1], N_SAMPLE, 2)).long()
    b_r = G.value(f"{gid}.b_sample", lambda ref: ref_bb(ref)[1].reshape(-1)[bidx.to(cuda)])
    b_s = b_o.reshape(-1)[bidx.to(cuda)].float().cpu()
    b_err = float((b_r.float() - b_s).norm() / b_s.norm())
    print(f"METRIC lotd_ref {gid} gp={err:.2e} ddLdy={a_err:.2e} bwd_bwd={b_err:.2e}")
    assert err < 2e-2 and a_err < 5e-3 and b_err < 5e-2, (gid, err, a_err, b_err)
