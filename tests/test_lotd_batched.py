"""Batched LoTD tables on the CPU: the batched oracle (oracle/lotd_batched.py) against per-batch calls of the unbatched one, its adjoint
identities, the autograd glue of fields/encoding.py with batches (on the oracle backend), and the argument checks of
bindings._lotd with the reference's messages (lotd_torch_api.cu:263-290)."""
import numpy as np
import pytest
import torch

from oracle import lotd as olotd
from oracle import lotd_batched as oblotd

CFG = dict(lod_res=[[5, 7, 4], [8, 12, 6], [13, 19, 9], [20, 30, 14]], lod_n_feats=[2, 4, 2, 2],
           lod_types=["Dense", "Dense", "Hash", "Hash"], hashmap_size=97)


def _meta():
    return olotd.LoDMeta(3, **CFG)


def _inputs(m, n, n_tables, seed, dtype=np.float16):
    rng = np.random.default_rng(seed)
    x = rng.uniform(1e-6, 1 - 1e-6, (n, 3)).astype(np.float32)
    p = rng.uniform(-0.5, 0.5, n_tables * m.n_params).astype(dtype)
    g = (rng.normal(size=(n, m.n_encoded_dims)) * 0.1).astype(np.float16)
    gin = rng.normal(size=(n, 3)).astype(np.float32)
    return rng, x, p, g, gin


def _per_batch(m, x, p, g, gin, b_of_point, start_of_batch, ml):
    """the batched contract spelled out: each batch's points through the unbatched oracle on that batch's table"""
    n, P = len(x), m.n_params
    y = np.zeros((n, m.n_encoded_dims), p.dtype)
    J = np.zeros((n, m.n_encoded_dims, 3), np.float32)
    gp = np.zeros(len(p))
    ddy = np.zeros((n, m.n_encoded_dims), np.float32)
    gp2 = np.zeros(len(p))
    for b, s in enumerate(start_of_batch):
        r = np.nonzero(b_of_point == b)[0]
        if r.size == 0:
            continue
        t = p[s:s + P]
        y[r], J[r] = olotd.lod_fwd(m, x[r], t, ml, True)
        gp[s:s + P] += olotd.lod_bwd_grid(m, g[r], x[r], P, ml)
        a, c, _ = olotd.lod_bwd_bwd_input(m, gin[r], g[r], x[r], t, J[r], ml)
        ddy[r] = a
        gp2[s:s + P] += c
    return y, J, gp, ddy, gp2


CASES = ["inds", "offsets_shared", "data_size", "inds_and_offsets"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("ml", [None, 1])
def test_batched_oracle_is_per_batch_calls(case, ml):
    m = _meta()
    P, n = m.n_params, 600
    rng, x, p, g, gin = _inputs(m, n, 3, CASES.index(case))
    kw = {}
    if case == "inds":                          # unsorted, some points skipped, batch 2 referenced by no point
        b = rng.integers(-1, 2, n)
        starts = [0, P, 2 * P]
        kw = dict(batch_inds=b)
    elif case == "offsets_shared":              # non-uniform offsets; batches 1 and 3 share a table, batch 2 overlaps table 0
        b = rng.integers(0, 4, n)
        starts = [2 * P, 0, (P // 2) & ~1, 0]
        kw = dict(batch_inds=b, batch_offsets=np.array(starts))
    elif case == "data_size":                   # [3, 200, 3] input: batch i // 200
        b = np.arange(n) // 200
        starts = [0, P, 2 * P]
        kw = dict(batch_data_size=200)
    else:                                       # offsets without inds: every point reads offsets[0]
        b = np.zeros(n, np.int64)
        starts = [P]
        kw = dict(batch_offsets=np.array(starts))
    y_w, J_w, gp_w, ddy_w, gp2_w = _per_batch(m, x, p, g, gin, b, starts, ml)
    y, J = oblotd.lod_fwd(m, x, p, ml, True, **kw)
    gp = oblotd.lod_bwd_grid(m, g, x, len(p), ml, **kw)
    ddy, gp2, _ = oblotd.lod_bwd_bwd_input(m, gin, g, x, p, J, ml, **kw)
    assert np.array_equal(y.view(np.uint16), y_w.view(np.uint16)) and np.array_equal(J, J_w)
    assert np.allclose(gp, gp_w, rtol=1e-12, atol=1e-15) and np.allclose(gp2, gp2_w, rtol=1e-12, atol=1e-12)
    assert np.array_equal(ddy, ddy_w)
    skipped = b < 0
    assert not (y[skipped].any() or J[skipped].any() or ddy[skipped].any())
    if case == "inds":
        assert skipped.any() and not gp[2 * P:].any() and not gp2[2 * P:].any() and np.abs(gp[:P]).max() > 0
    if case == "offsets_shared":
        assert np.abs(gp[P:2 * P]).max() == 0 or (b == 2).any()   # table 1 only through batch 2's overlapping window


def test_batched_adjoint_identities():
    """<dL_dy, fwd(p)> = <bwd_grid(dL_dy), p> and <gin, J(p)^T dL_dy> = <bwd_bwd_grid(gin, dL_dy), p> with batches, on an fp32 table"""
    m = _meta()
    P, n = m.n_params, 800
    rng, x, p, g, gin = _inputs(m, n, 3, 11, np.float32)
    kw = dict(batch_inds=rng.integers(-1, 4, n), batch_offsets=np.array([2 * P, 0, P, 0]))
    y, J = oblotd.lod_fwd(m, x, p, None, True, **kw)
    gp = oblotd.lod_bwd_grid(m, g, x, len(p), **kw)
    lhs, rhs = float(np.sum(g.astype(np.float64) * y)), float(gp @ p.astype(np.float64))
    assert abs(lhs - rhs) <= 1e-5 * abs(rhs)
    _, gp2, _ = oblotd.lod_bwd_bwd_input(m, gin, g, x, p, J, need_dLdy=False, **kw)
    dx = np.einsum("nf,nfd->nd", g.astype(np.float64), J.astype(np.float64))
    lhs, rhs = float(np.sum(gin * dx)), float(gp2 @ p.astype(np.float64))
    assert abs(lhs - rhs) <= 1e-5 * abs(rhs)


def test_encoding_glue_threads_the_batch(monkeypatch):
    """lotd_encoding* with `input_batched` and with `bidx` on the oracle backend equal per-batch unbatched calls, through the
    second-order chain (nablas -> table, dL_dy)"""
    from neuralsim_b200.fields import encoding
    monkeypatch.setattr(encoding, "_backend", oblotd.backend)
    m = _meta()
    P, B, M = m.n_params, 3, 50
    rng = np.random.default_rng(5)
    params = torch.from_numpy(rng.uniform(-0.5, 0.5, B * P).astype(np.float32))
    x = torch.from_numpy(rng.uniform(0.01, 0.99, (B, M, 3)).astype(np.float32))
    cot_y = torch.from_numpy(rng.normal(size=(B, M, m.n_encoded_dims)).astype(np.float32))
    cot_n = torch.from_numpy(rng.normal(size=(B, M, 3)).astype(np.float32))
    dLdy = torch.from_numpy(rng.normal(size=(B, M, m.n_encoded_dims)).astype(np.float32))

    def run(xx, pp, dd, cy, cn, **kw):
        pp = pp.clone().requires_grad_(True)
        dd = dd.clone().requires_grad_(True)
        y, dydx, _ = encoding.lotd_encoding_fwd_dydx(xx, pp, meta=m, **kw)
        nab = encoding.lotd_encoding_bwd_dydx(m, dd, dydx, xx, pp, **kw)
        y2 = encoding.lotd_encoding(xx, pp, meta=m, **kw)
        assert torch.equal(y, y2)
        loss = (y * cy.reshape(y.shape)).sum() + (nab * cn.reshape(nab.shape)).sum()
        return (y.detach(), nab.detach()) + torch.autograd.grad(loss, [pp, dd])

    batched = run(x, params, dLdy, cot_y, cot_n, input_batched=True)
    bidx = torch.arange(B).repeat_interleave(M)
    flat = run(x.reshape(-1, 3), params, dLdy.reshape(B * M, -1), cot_y, cot_n, bidx=bidx)
    per = [run(x[b], params[b * P:(b + 1) * P], dLdy[b], cot_y[b], cot_n[b]) for b in range(B)]
    for k in range(4):
        want = torch.cat([r[k] for r in per])
        assert torch.allclose(batched[k].reshape(want.shape), want, rtol=1e-6, atol=1e-7), k
        assert torch.allclose(flat[k].reshape(want.shape), want, rtol=1e-6, atol=1e-7), k


# ------------------------------------------------------------------------------------------------ argument checks of the shim
@pytest.fixture(scope="module")
def shim():
    from neuralsim_b200 import build
    build.build_library()
    from neuralsim_b200.bindings import _lotd
    return _lotd


def _shim_args(shim):
    meta = shim.LoDMeta(3, CFG["lod_res"], CFG["lod_n_feats"], CFG["lod_types"], CFG["hashmap_size"])
    n = 12
    return meta, torch.rand(n, 3), torch.zeros(2 * meta.n_params, dtype=torch.float16), torch.zeros(n, meta.n_encoded_dims, dtype=torch.float16)


@pytest.mark.parametrize("bad, match", [
    (dict(batch_inds=torch.zeros(12, dtype=torch.int32)), r"argument #\d 'batch_inds' to have scalar type Long"),
    (dict(batch_inds=torch.zeros(11, dtype=torch.int64)), r"Expected tensor of size \[12\], but got tensor of size \[11\]"),
    (dict(batch_inds=torch.zeros(12, 1, dtype=torch.int64)), r"Expected 1-dimensional tensor, but got 2-dimensional tensor for argument #\d 'batch_inds'"),
    (dict(batch_offsets=torch.zeros(2, 1, dtype=torch.int64)), r"Expected 1-dimensional tensor, but got 2-dimensional tensor for argument #\d 'batch_offset'"),
    (dict(batch_offsets=torch.zeros(2, dtype=torch.float32)), r"'batch_offset' to have scalar type Long"),
    (dict(batch_inds=torch.zeros(24, dtype=torch.int64)[::2]), r"Expected contiguous tensor, but got non-contiguous tensor for argument #\d 'batch_inds'"),
    (dict(batch_data_size=5), r"Expect nonzero `batch_data_size`=5 to be a divisor of `batch_size`=12"),
])
def test_shim_refuses_bad_batch_arguments(shim, bad, match):
    meta, x, p, g = _shim_args(shim)
    kw = dict(batch_inds=None, batch_offsets=None, batch_data_size=None)
    kw.update(bad)
    with pytest.raises(RuntimeError, match=match):
        shim.lod_fwd(meta, x, p, kw["batch_inds"], kw["batch_offsets"], kw["batch_data_size"], None, False)
    with pytest.raises(RuntimeError, match=match):
        shim.lod_bwd(meta, g, x, p, None, kw["batch_inds"], kw["batch_offsets"], kw["batch_data_size"], None, False, True)
    with pytest.raises(RuntimeError, match=match):
        shim.lod_bwd_bwd_input(meta, torch.zeros(12, 3), g, x, p, None, kw["batch_inds"], kw["batch_offsets"], kw["batch_data_size"],
                               None, False, True, False)


def test_shim_messages_name_the_reference_function(shim):
    meta, x, p, g = _shim_args(shim)
    with pytest.raises(RuntimeError, match=r"LoTDEncoding::fwd: Expect nonzero"):
        shim.lod_fwd(meta, x, p, None, None, 7, None, False)
    with pytest.raises(RuntimeError, match=r"LoTDEncoding::bwd: Expect nonzero"):
        shim.lod_bwd(meta, g, x, p, None, None, None, 7, None, False, True)
    with pytest.raises(RuntimeError, match=r"LoTDEncoding::bwd_bwd_input: Expect nonzero"):
        shim.lod_bwd_bwd_input(meta, torch.zeros(12, 3), g, x, p, None, None, None, 7, None, False, True, False)
    with pytest.raises(RuntimeError, match=r"while checking arguments for lod_bwd_common"):
        shim.lod_bwd(meta, g, x, p, None, torch.zeros(12, dtype=torch.int32), None, None, None, False, True)


@pytest.mark.parametrize("bad", [
    lambda P: dict(batch_inds=torch.full((12,), 2, dtype=torch.int64)),                             # 2 tables in params
    lambda P: dict(batch_inds=torch.zeros(12, dtype=torch.int64), batch_offsets=torch.tensor([1])),  # odd
    lambda P: dict(batch_offsets=torch.tensor([-2])),
    lambda P: dict(batch_offsets=torch.tensor([P + 2])),                                            # past the end
    lambda P: dict(batch_data_size=4),                                                              # 3 batches, 2 tables
])
def test_shim_refuses_tables_outside_params(shim, bad):
    meta, x, p, _ = _shim_args(shim)
    kw = dict(batch_inds=None, batch_offsets=None, batch_data_size=None)
    kw.update(bad(meta.n_params))
    with pytest.raises(RuntimeError, match=r"out of range|must be even and in"):
        shim.lod_fwd(meta, x, p, kw["batch_inds"], kw["batch_offsets"], kw["batch_data_size"], None, False)
