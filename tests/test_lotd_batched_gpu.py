"""Batched LoTD tables (per-point `batch_inds`, per-batch `batch_offsets`, equal-size batches `batch_data_size`) through the five
kernels of csrc/lotd.cu, against the float64 oracle per table and per pseudo level, at the table geometries of
test_lotd_geometry_gpu.py.  The kernels are called through the C ABI (nsb_lotd_*_batched), so the table gradients are the kernels'
fp32 accumulators.

Each geometry holds three tables in `params` and runs three batch layouts:
  inds       batch_inds unsorted, ~10 % negative (skipped points), the third table referenced by no point
  offsets    batch_inds over four batches with non-uniform batch_offsets: batches 1 and 3 share table 0, batch 2's table starts
             half-way into table 0 (overlapping tables: gradients add up)
  data_size  [3, M, D] input, batch_data_size = M
G1 (17-level cfg3 table) runs enough points for every grid-stride loop of every kernel to make at least three trips; the oracle runs
on a sample of rows spanning every trip and the cotangents are non-zero only there.  Also here: a single table passed as a batch is
bit-equal to the unbatched call, the public `lotd_encoding*` functions against float64 autograd, and the reference project's own
kernels with batch arguments (tests/golden/ref__lotd_batched.npz, recorded from oracle/_ref/_lotd as tests/refgold.py describes).
Bounds are those of test_lotd_geometry_gpu.py (DESIGN.md §4)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import lotd as olotd
from oracle import lotd_batched as oblotd
from refgold import Golden
from test_lotd_geometry_gpu import (GEOMS, GRID_REL, GRID_REL_SMALL, INPUT_REL, SAMPLE, _boundary_points, _clamp_points, _rel, _rows,
                                    _stride, _support_sample)

pytestmark = pytest.mark.gpu

N_TABLES = 3
MODES = ["inds", "offsets", "data_size"]


def _L():
    from neuralsim_b200 import _lib as L
    return L


class BGeom:
    def __init__(self, gid):
        from neuralsim_b200.bindings import _lotd
        self.gid = gid
        D, make, n = GEOMS[gid]
        self.D, self.cfg = D, make()
        self.om = olotd.LoDMeta(D, **self.cfg)
        self.gm = _lotd.LoDMeta(D, self.cfg["lod_res"], self.cfg["lod_n_feats"], self.cfg["lod_types"], self.cfg["hashmap_size"])
        om = self.om
        self.P = P = om.n_params
        rng = np.random.default_rng(100 + sum(map(ord, gid)))
        self.p16 = rng.uniform(-0.5, 0.5, N_TABLES * P).astype(np.float16)
        big = n == 0
        if big:        # every thread of every launch loops at least three times (the forward's loop over points is the shortest)
            s = _stride(1 << 40)
            n = 3 * s + s // 3 + 78
        n -= n % N_TABLES
        self.n = n
        x = rng.uniform(1e-6, 1 - 1e-6, (n, D)).astype(np.float32)
        self.rows = np.unique(np.concatenate([rng.choice(n, SAMPLE, replace=False), [0, n - 1]])) if big else np.arange(n)
        S = len(self.rows)
        special = np.concatenate([_clamp_points(D), _boundary_points(rng, om, S // 5)])
        x[self.rows[rng.choice(S, len(special), replace=False)]] = special
        self.x, self.xr = x, x[self.rows]
        g = (rng.normal(size=(S, om.n_encoded_dims)) * 0.1).astype(np.float16)
        g[rng.random(S) < 0.3] = 0
        self.g, self.gin = g, rng.normal(size=(S, D)).astype(np.float32)
        self.ml_mid = om.n_levels // 2 - 1
        inds = rng.integers(0, N_TABLES - 1, n)                   # table N_TABLES-1: no point
        inds[rng.random(n) < 0.1] = -1
        half = (P // 2) & ~1
        self.modes = dict(
            inds=dict(inds=inds, offsets=None, ds=0),
            offsets=dict(inds=rng.integers(0, 4, n), offsets=np.array([2 * P, 0, half, 0]), ds=0),
            data_size=dict(inds=None, offsets=None, ds=n // N_TABLES))
        self.xg = torch.from_numpy(x).cuda()
        self.pg16 = torch.from_numpy(self.p16).cuda()

    def full(self, rows_val, dtype):
        out = torch.zeros((self.n,) + rows_val.shape[1:], dtype=dtype)
        out[torch.from_numpy(self.rows)] = torch.from_numpy(rows_val).to(dtype)
        return out.cuda()

    def batch(self, mode):
        """-> (nsb_lotd_batch, the device tensors it points to, the oracle's batch arguments on the sample rows)"""
        L, b = _L(), self.modes[mode]
        keep = [None if b["inds"] is None else torch.from_numpy(b["inds"]).cuda(),
                None if b["offsets"] is None else torch.from_numpy(b["offsets"]).cuda()]
        c = L.LotdBatchC(L.ptr(keep[0], allow_none=True), L.ptr(keep[1], allow_none=True), b["ds"])
        inds = b["inds"][self.rows] if b["inds"] is not None else (self.rows // b["ds"] if b["ds"] else None)
        return c, keep, dict(batch_inds=inds, batch_offsets=b["offsets"])

    def run(self, params, ml, c, dydx=True, grads=True):
        """fwd, bwd_grid, bwd_input, bwd_bwd (both outputs) of the batched entries; c: nsb_lotd_batch or None"""
        L = _L()
        lib, n, gm, D = L.lib(), self.n, self.gm, self.D
        bp = ctypes.byref(c) if c is not None else L._NULL
        F = gm.n_encoded_dims
        y = torch.empty((n, F), dtype=params.dtype, device="cuda")
        d = torch.empty((n, F * D), dtype=torch.float32, device="cuda") if dydx else None
        L.check(lib.nsb_lotd_fwd_batched(gm.c_ref, L.ptr(self.xg, "f32"), L.ptr(params), ctypes.c_int(params.dtype == torch.float16),
                                         L.c_i64(n), L.c_i32(ml), bp, L.ptr(y), L.ptr(d, "f32", allow_none=True), L.stream_ptr()), "fwd")
        if not grads:
            return y, d
        g = self.full(self.g, torch.float16)
        acc = torch.zeros(params.shape[0], dtype=torch.float32, device="cuda")
        dx = torch.empty((n, D), dtype=torch.float32, device="cuda")
        L.check(lib.nsb_lotd_bwd_grid_batched(gm.c_ref, L.ptr(g), 1, L.ptr(self.xg, "f32"), L.c_i64(n), L.c_i32(ml), bp, L.c_f32(1.0),
                                              L.ptr(acc), L.stream_ptr()), "bwd_grid")
        L.check(lib.nsb_lotd_bwd_input_batched(L.ptr(g), 1, L.ptr(d, "f32"), L.c_i64(n), L.c_i32(F), L.c_i32(D), bp, L.c_f32(1.0),
                                               L.ptr(dx), L.stream_ptr()), "bwd_input")
        gin = self.full(self.gin, torch.float32)
        ddy = torch.empty((n, F), dtype=torch.float32, device="cuda")
        acc2 = torch.zeros(params.shape[0], dtype=torch.float32, device="cuda")
        L.check(lib.nsb_lotd_bwd_bwd_input_batched(gm.c_ref, L.ptr(gin, "f32"), L.ptr(g), 1, L.ptr(self.xg, "f32"), L.ptr(d, "f32"),
                                                   L.c_i64(n), L.c_i32(ml), bp, L.c_f32(1.0), L.ptr(ddy), L.ptr(acc2), L.stream_ptr()),
                "bwd_bwd")
        return y, d, acc, dx, ddy, acc2

    def pseudo_slices(self):
        """(table, pseudo level) -> (level, index array of its table elements, output columns)"""
        om, F = self.om, self.om.n_feat_per_pseudo_lvl
        out = []
        for t in range(N_TABLES):
            for p in range(om.n_pseudo_levels):
                l = om.map_levels[p]
                base = t * self.P + om.level_offsets[l] + om.map_cnt[p] * F
                idx = (base + np.arange(om.level_sizes[l])[:, None] * om.level_n_feats[l] + np.arange(F)[None, :]).ravel()
                out.append((t, p, l, idx, slice(p * F, (p + 1) * F)))
        return out


_GEOMS = {}


@pytest.fixture(scope="module", params=list(GEOMS))
def geom(request):
    gid = request.param
    if gid not in _GEOMS:
        _GEOMS.clear()
        _GEOMS[gid] = BGeom(gid)
    return _GEOMS[gid]


def test_batched_loops(geom):
    """the layout the comparisons rely on: at G1 every kernel's grid-stride loop makes >= 3 trips and the sample rows hit each trip"""
    G = geom
    b = G.modes["inds"]["inds"]
    assert (b < 0).any() and not (b == N_TABLES - 1).any() and not np.all(np.diff(b) >= 0)
    if G.gid != "G1":
        return
    npl, nf = G.om.n_pseudo_levels, G.om.n_encoded_dims
    for items, per in ((G.n, 1), (G.n * npl, npl), (G.n * nf, nf)):
        s = _stride(items)
        iters = -(-items // s)
        assert iters >= 3, (items, s)
        assert np.array_equal(np.unique((G.rows[:, None] * per + np.arange(per)[None, :]) // s), np.arange(iters))


@pytest.mark.parametrize("mode", MODES)
def test_batched_against_oracle(geom, mode):
    """y bit-exact, dy_dx to 1e-6; table gradients per table and pseudo level; skipped rows zero, unreferenced tables exactly zero"""
    G, om = geom, geom.om
    c, keep, okw = G.batch(mode)
    rows = torch.from_numpy(G.rows).cuda()
    skipped_all = G.modes[mode]["inds"] < 0 if G.modes[mode]["inds"] is not None else np.zeros(G.n, bool)
    fails = []
    for ml in (om.n_levels, G.ml_mid):
        y, d, acc, dx, ddy, acc2 = G.run(G.pg16, ml, c)
        y_ref, J = oblotd.lod_fwd(om, G.xr, G.p16, ml, True, **okw)
        yr, dr = y[rows].cpu().numpy(), d[rows].view(len(G.rows), -1, G.D).cpu().numpy()
        if not np.array_equal(yr.view(np.uint16), y_ref.view(np.uint16)):
            fails.append((ml, "y", int((yr.view(np.uint16) != y_ref.view(np.uint16)).sum())))
        if not np.allclose(dr, J, rtol=1e-6, atol=1e-7):
            fails.append((ml, "dy_dx"))
        sk = torch.from_numpy(skipped_all).cuda()
        if sk.any() and (y[sk].abs().max() != 0 or d[sk].abs().max() != 0 or dx[sk].abs().max() != 0 or ddy[sk].abs().max() != 0):
            fails.append((ml, "non-zero row of a skipped point"))
        gp_ref = oblotd.lod_bwd_grid(om, G.g, G.xr, len(G.p16), ml, **okw)
        ddy_ref, gp2_ref, _ = oblotd.lod_bwd_bwd_input(om, G.gin, G.g, G.xr, G.p16, J, ml, **okw)
        dx_ref = olotd.lod_bwd_input(G.g, J)
        a, a2 = acc.double().cpu().numpy(), acc2.double().cpu().numpy()
        ddy_r, dx_r = ddy[rows].cpu().numpy(), dx[rows].cpu().numpy()
        errs = []
        for t, p, l, idx, cols in G.pseudo_slices():
            for k, got, want in (("grid", a[idx], gp_ref[idx]), ("bwd_bwd", a2[idx], gp2_ref[idx])):
                if not np.abs(want).max() > 0:                     # masked level, unreferenced table: exactly zero
                    if np.any(got != 0):
                        fails.append((ml, k, t, p, "non-zero gradient without a reference gradient"))
                    continue
                e = _rel(got, want)
                errs.append(e)
                if not e < GRID_REL.get(G.gid, GRID_REL_SMALL):
                    fails.append((ml, k, t, p, e))
        if mode == "inds" and (np.any(a[(N_TABLES - 1) * G.P:] != 0) or np.any(a2[(N_TABLES - 1) * G.P:] != 0)):
            fails.append((ml, "gradient in the unreferenced table"))
        e_ddy = _rel(ddy_r, ddy_ref)
        e_dx = [_rel(dx_r[:, k], dx_ref[:, k]) for k in range(G.D)]
        if not (e_ddy < INPUT_REL and max(e_dx) < INPUT_REL):
            fails.append((ml, "ddLdy / dL_dx", e_ddy, e_dx))
        print(f"METRIC lotd_batched {G.gid} {mode} ml={ml} grid max={max(errs):.2e} ddLdy={e_ddy:.2e} dL_dx={max(e_dx):.2e}")
    assert not fails, fails


def test_batched_fp32_forward(geom):
    G, om = geom, geom.om
    c, keep, okw = G.batch("offsets")
    p32 = (G.p16.astype(np.float32) + np.float32(1e-4) * np.sign(G.p16)).astype(np.float32)
    y, _ = G.run(torch.from_numpy(p32).cuda(), G.ml_mid, c, dydx=False, grads=False)
    y_ref, _ = oblotd.lod_fwd(om, G.xr, p32, G.ml_mid, **okw)
    assert y.dtype == torch.float32 and np.allclose(y[torch.from_numpy(G.rows).cuda()].cpu().numpy(), y_ref, rtol=1e-6, atol=1e-7)


def test_one_table_as_a_batch_is_the_unbatched_call(geom):
    """batch_inds all zero, batch_offsets [0] and batch_data_size = N on one table: fp16 y, dy_dx, dL_dx and dL_d(dL_dy) bit-equal to
    the unbatched call; the table gradients equal up to the order of the fp32 atomic sums"""
    G, L = geom, _L()
    one = G.pg16[:G.P].contiguous()
    ref = G.run(one, G.om.n_levels, None)
    g_abs = G.g
    G.g = np.abs(G.g)
    absum = G.run(one, G.om.n_levels, None)
    G.g = g_abs
    z = torch.zeros(G.n, dtype=torch.int64, device="cuda")
    o = torch.zeros(1, dtype=torch.int64, device="cuda")
    for c in (L.LotdBatchC(L.ptr(z), None, 0), L.LotdBatchC(None, L.ptr(o), 0), L.LotdBatchC(None, None, G.n)):
        got = G.run(one, G.om.n_levels, c)
        for k in (0, 1, 3, 4):
            assert torch.equal(got[k].view(torch.int32) if k else got[k].view(torch.int16),
                               ref[k].view(torch.int32) if k else ref[k].view(torch.int16)), k
        for k in (2, 5):          # the bwd-bwd terms carry signs that |dL_dy| does not remove: a floor of 2^-20 of the largest entry
            bound = 1e-5 * absum[k].abs().double() + 2.0 ** -20 * float(ref[k].abs().max())
            assert bool(((got[k].double() - ref[k].double()).abs() <= bound).all()), k


# ===================================================================================================================== public interface
def test_encoding_functions_batched_glue(cuda):
    """lotd_encoding_fwd_dydx -> lotd_encoding_bwd_dydx -> autograd with `bidx` (and with `input_batched`) at the 17-level cfg3 table,
    two tables: the loss scale 128, the division by it and the batch against float64 with the same factors written out"""
    from neuralsim_b200.fields import encoding
    cfg = GEOMS["G1"][1]()
    om = olotd.LoDMeta(3, **cfg)
    meta = encoding.generate_meta(3, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"])
    P, B, M = om.n_params, 2, 10000
    rng = np.random.default_rng(9)
    p16 = rng.uniform(-0.5, 0.5, B * P).astype(np.float16)
    x = rng.uniform(1e-6, 1 - 1e-6, (B, M, 3)).astype(np.float32)
    dLdy = (rng.normal(size=(B, M, om.n_encoded_dims)) * 1e-3).astype(np.float16)
    cot_y = rng.normal(size=(B, M, om.n_encoded_dims)).astype(np.float32)
    cot_n = (rng.normal(size=(B, M, 3)) * 0.1).astype(np.float32)
    bidx = rng.integers(0, B, B * M)
    s = 128.0
    for how in ("bidx", "input_batched"):
        master = torch.from_numpy(p16).cuda().float().requires_grad_(True)     # an fp32 master table, as LoTDEncoding keeps
        params = master.half()
        dg = torch.from_numpy(dLdy).cuda().reshape(B * M, -1) if how == "bidx" else torch.from_numpy(dLdy).cuda()
        dg.requires_grad_(True)
        xg = torch.from_numpy(x).cuda()
        kw = dict(bidx=torch.from_numpy(bidx).cuda()) if how == "bidx" else dict(input_batched=True)
        if how == "bidx":
            xg = xg.reshape(B * M, 3)
        y, dydx, _ = encoding.lotd_encoding_fwd_dydx(xg, params, meta=meta, **kw)
        nablas = encoding.lotd_encoding_bwd_dydx(meta, dg, dydx, xg, params, **kw)
        loss = (y.float() * torch.from_numpy(cot_y).cuda().reshape(y.shape)).sum() + (nablas * torch.from_numpy(cot_n).cuda().reshape(nablas.shape)).sum()
        g_table, g_dLdy = torch.autograd.grad(loss, [master, dg])

        okw = dict(batch_inds=bidx) if how == "bidx" else dict(batch_data_size=M)
        xs = x.reshape(-1, 3)
        cy, cn, dl = cot_y.reshape(B * M, -1), cot_n.reshape(B * M, 3), dLdy.reshape(B * M, -1)
        y_ref, J = oblotd.lod_fwd(om, xs, p16, None, True, **okw)
        assert np.array_equal(y.detach().reshape(B * M, -1).cpu().numpy().view(np.uint16), y_ref.view(np.uint16)), how
        scaled = (dl.astype(np.float32) * np.float32(s)).astype(np.float16)
        nab_ref = olotd.lod_bwd_input(scaled, J).astype(np.float64) / s
        nab_scale = np.einsum("nf,nfd->nd", np.abs(scaled.astype(np.float64)), np.abs(J.astype(np.float64))) / s
        a = oblotd.lod_bwd_grid(om, (cy.astype(np.float16).astype(np.float32) * np.float32(s)).astype(np.float16), xs, B * P, **okw) / s
        _, b, _ = oblotd.lod_bwd_bwd_input(om, cn, scaled, xs, p16, J, need_dLdy=False, **okw)
        b = b / s
        ddLdy_ref = np.einsum("nd,nfd->nf", cn.astype(np.float64), J.astype(np.float64))
        ddLdy_scale = np.einsum("nd,nfd->nf", np.abs(cn.astype(np.float64)), np.abs(J.astype(np.float64)))
        nab_err = np.abs(nablas.detach().reshape(B * M, 3).double().cpu().numpy() - nab_ref) / (nab_scale + 1e-30)
        got_t = g_table.double().cpu().numpy()
        tab_err = np.abs(got_t - (a + b)) / (2.0 ** -10 * (np.abs(a) + np.abs(b)) + 2.0 ** -23)
        got_y = g_dLdy.reshape(B * M, -1).double().cpu().numpy()
        y_err = np.abs(got_y - ddLdy_ref) / (2.0 ** -10 * np.abs(ddLdy_ref) + 2.0 ** -22 * ddLdy_scale + 2.0 ** -24)
        print(f"METRIC lotd_batched_glue {how} nablas max err / scale={nab_err.max():.2e} table max err / bound={tab_err.max():.2e} "
              f"dL_dy max err / bound={y_err.max():.2e}")
        assert nab_err.max() < 1e-5, how
        assert np.isfinite(got_t).all() and tab_err.max() <= 1.0 and np.abs(a[P:]).max() > 0 and np.abs(b[:P]).max() > 0, how
        assert y_err.max() <= 1.0, how


# ===================================================================================================================== reference kernels
def test_against_reference_kernels_batched(cuda):
    """the reference project's own _lotd kernels with batch_inds (negative entries included), batch_offsets and batch_data_size on
    three tables of the G5 geometry: y bit-exact, dy_dx rows, gradient samples (fp16 atomics there: tolerances of
    test_lotd_geometry_gpu.py)"""
    from neuralsim_b200.bindings import _lotd as ours
    G = Golden("_lotd_batched", "_lotd")
    D, make, _ = GEOMS["G5"]
    cfg = make()
    rmeta = lambda ref: ref.LoDMeta(D, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"], False)
    om = ours.LoDMeta(D, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"])
    P = om.n_params
    rng = np.random.default_rng(17)
    n = 60000
    p = torch.from_numpy(rng.uniform(-0.5, 0.5, N_TABLES * P).astype(np.float16)).to(cuda)
    xn = rng.uniform(1e-6, 1 - 1e-6, (n, D)).astype(np.float32)
    xn[:3 ** D] = _clamp_points(D)
    x = torch.from_numpy(xn).to(cuda)
    g = torch.from_numpy((rng.normal(size=(n, om.n_encoded_dims)) * 0.05).astype(np.float16)).to(cuda)
    gin = torch.from_numpy((rng.normal(size=(n, D)) * 0.01).astype(np.float32)).to(cuda)
    inds = rng.integers(0, N_TABLES, n)
    inds[rng.random(n) < 0.1] = -1
    inds[:50] = -1                                                       # skipped rows among the recorded rows
    cases = dict(inds=(torch.from_numpy(inds).to(cuda), None, None),
                 offsets=(torch.from_numpy(rng.integers(0, 3, n)).to(cuda), torch.tensor([2 * P, 0, 0], device=cuda), None),
                 data_size=(None, None, n // N_TABLES))
    for name, (bi, bo, ds) in cases.items():
        ref_fwd = lambda ref: ref.lod_fwd(rmeta(ref), x, p, bi, bo, ds, None, True)
        y_o, d_o = ours.lod_fwd(om, x, p, bi, bo, ds, None, True)
        G.equal(f"{name}.y", y_o.view(torch.int16), lambda ref: ref_fwd(ref)[0].contiguous().view(torch.int16))
        d_r = G.value(f"{name}.d_rows", lambda ref: _rows(ref_fwd(ref)[1].reshape(d_o.shape), 100))
        assert torch.allclose(d_r, _rows(d_o, 100), rtol=1e-6, atol=1e-7), name
        ref_bwd = lambda ref: ref.lod_bwd(rmeta(ref), g, x, p, ref_fwd(ref)[1], bi, bo, ds, None, True, True)
        gx_o, gp_o = ours.lod_bwd(om, g, x, p, d_o, bi, bo, ds, None, True, True)
        gx_r = G.value(f"{name}.gx_rows", lambda ref: _rows(ref_bwd(ref)[0], 1000))
        assert torch.allclose(gx_r, _rows(gx_o, 1000), rtol=1e-4, atol=1e-4), name
        idx = G.value(f"{name}.gp_idx", lambda ref: _support_sample(ref_bwd(ref)[1], 3000, 1)).long()
        gp_r = G.value(f"{name}.gp_sample", lambda ref: ref_bwd(ref)[1].reshape(-1)[idx.to(cuda)])
        gp_s = gp_o.reshape(-1)[idx.to(cuda)].float().cpu()
        err = float((gp_r.float() - gp_s).norm() / gp_s.norm())
        ref_bb = lambda ref: ref.lod_bwd_bwd_input(rmeta(ref), gin, g, x, p, ref_fwd(ref)[1].contiguous(), bi, bo, ds, None, True, True, False)
        a_o, b_o, _ = ours.lod_bwd_bwd_input(om, gin, g, x, p, d_o, bi, bo, ds, None, True, True, False)
        a_r = G.value(f"{name}.a_rows", lambda ref: _rows(ref_bb(ref)[0], 500))
        a_err = float((a_r.float() - _rows(a_o, 500).float()).norm() / _rows(a_o, 500).float().norm())
        bidx_ = G.value(f"{name}.b_idx", lambda ref: _support_sample(ref_bb(ref)[1], 3000, 2)).long()
        b_r = G.value(f"{name}.b_sample", lambda ref: ref_bb(ref)[1].reshape(-1)[bidx_.to(cuda)])
        b_s = b_o.reshape(-1)[bidx_.to(cuda)].float().cpu()
        b_err = float((b_r.float() - b_s).norm() / b_s.norm())
        if name == "inds":
            assert float(y_o[:50].abs().max()) == 0 and float(gx_o[:50].abs().max()) == 0 and float(a_o[:50].abs().max()) == 0
        print(f"METRIC lotd_ref_batched {name} gp={err:.2e} ddLdy={a_err:.2e} bwd_bwd={b_err:.2e}")
        assert err < 2e-2 and a_err < 5e-3 and b_err < 5e-2, (name, err, a_err, b_err)
    G.save()
