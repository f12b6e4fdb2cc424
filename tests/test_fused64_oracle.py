"""CPU: the float64 reference of the fused kernels (oracle/fused64.py) against (i) torch float64 double-backward of the same model
without rounding, where its hand-written backward passes must be exact, and (ii) the autocast restatement oracle/nets.py, which
rounds the forward at the same points."""
import numpy as np
import pytest
import torch

from oracle import fused64, lotd as olotd, nets as onets

CFG16 = olotd.gen_ngp_cfg(log2_hashmap_size=14)          # the 16 x 2 layout of the product, 2^14 entries per hashed level


def _weights(width, rw, n_appear, seed):
    g = torch.Generator().manual_seed(seed)
    meta = olotd.LoDMeta(3, **CFG16)
    table = (torch.rand(meta.n_params, generator=g) * 2 - 1) * 0.5
    lin = lambda o, i: onets.kaiming_linear(g, o, i)
    W1, b1 = lin(width, 32)
    W2, b2 = lin(1, width)
    R1, rb1 = lin(rw, 54 + n_appear)
    R2, rb2 = lin(rw, rw)
    R3, rb3 = lin(3, rw)
    return table, (W1, b1, W2, b2, R1, rb1, R2, rb2, R3, rb3)


def _inputs(n, n_appear, seed, lo=-0.95, hi=0.95):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g) * (hi - lo) + lo
    v = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ha = torch.randn(n, n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    return x, v, ha, cot


def _autograd_model(ref, ws, x, v, ha, cot):
    """The unrounded model as plain float64 torch: nablas = fac * d sdf / dx by double backward through the trilinear interpolation."""
    T = torch.tensor(ref.T, requires_grad=True)
    W = [torch.tensor(p.half().double().numpy(), requires_grad=True) for p in ws]
    W1, b1, W2, b2, R1, rb1, R2, rb2, R3, rb3 = W
    xs32 = ref.xs_of(x.numpy())
    x64 = x.double().requires_grad_(True)
    xs64 = x64 * 0.5 + 0.5
    cols = [torch.zeros(x.shape[0], dtype=torch.float64)] * 32
    for psl, lvl, loff, foff, ooff in olotd._level_iter(ref.meta, ref.max_level):
        res = np.array(ref.meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        cell, frac = olotd.pos_fract(xs32, scale)
        # the value is the fp32 fraction the kernels use, the derivative d frac / d xs = scale
        fr = torch.from_numpy(frac.astype(np.float64)) + (xs64 - xs64.detach()) * torch.from_numpy(scale.astype(np.float64))
        for c in range(8):
            off = np.array([(c >> d) & 1 for d in range(3)], dtype=np.uint32)
            idx = torch.from_numpy(olotd.grid_index(ref.meta, lvl, cell + off) * 2 + foff + loff)
            w = 1.0
            for d in range(3):
                w = w * (fr[:, d] if (c >> d) & 1 else 1.0 - fr[:, d])
            for f in range(2):
                cols[ooff + f] = cols[ooff + f] + w * T[idx + f]
    h = torch.stack(cols, -1)
    z = h @ W1.T + b1
    a = torch.nn.functional.softplus(z, beta=ref.beta, threshold=20.0)
    sdf = (a @ W2.T + b2)[:, 0]
    nab = torch.autograd.grad(sdf.sum(), x64, create_graph=True)[0] * torch.from_numpy(ref.fac)
    X = torch.cat([x.double(), onets.sh_encode(v.double(), 4), nab.detach().clamp(-1, 1), h, ha.double()], -1)
    Y1 = torch.relu(X @ R1.T + rb1)
    Y2 = torch.relu(Y1 @ R2.T + rb2)
    rgb = torch.sigmoid(Y2 @ R3.T + rb3)
    g_sdf, g_nab, g_rgb = (c.double() for c in cot)
    loss = (g_sdf * sdf).sum() + (g_nab * nab).sum() + (g_rgb * rgb).sum()
    grads = torch.autograd.grad(loss, [T, *W], retain_graph=True)
    sdf_only = torch.autograd.grad((g_sdf * sdf).sum(), [T, W1, b1, W2, b2])
    names = ["grid", "W1", "b1", "W2", "b2", "R1", "rb1", "R2", "rb2", "R3", "rb3"]
    return (dict(sdf=sdf, nablas=nab, rgb=rgb), {k: g.detach().numpy() for k, g in zip(names, grads)},
            {k: g.detach().numpy() for k, g in zip(names, sdf_only)}, dict(z=z, Y1=Y1, Y2=Y2))


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("width,rw,n_appear,max_level", [(64, 64, 4, None), (48, 40, 0, 7), (16, 64, 8, None)])
def test_unrounded_reference_equals_double_backward(width, rw, n_appear, max_level):
    table, ws = _weights(width, rw, n_appear, seed=width + rw)
    ref = fused64.Fused64(table, CFG16, *ws, fac=(1.0, 0.5, 2.0), max_level=max_level, rounding=False)
    x, v, ha, cot = _inputs(400, n_appear, seed=3)
    out, grads, sdf_grads, inter = _autograd_model(ref, ws, x, v, ha, cot)
    # the inputs reach both sides of every branch
    bz = ref.beta * inter["z"].detach().numpy()
    assert 0.01 < float((bz > 20).mean()) < 0.99
    for k in ("Y1", "Y2"):
        on = float((inter[k] > 0).double().mean())
        assert 0.1 < on < 0.9, (k, on)
    assert 0.02 < float((out["nablas"].abs() > 1).double().mean()) < 0.98
    fwd = ref.color_forward(x.numpy(), v.numpy(), ha.numpy())
    for k in ("sdf", "nablas", "rgb"):
        assert _rel(fwd[k], out[k].detach().numpy()) < 1e-12, k
    got = ref.color_backward(fwd, *(c.numpy() for c in cot))
    for k, g in grads.items():
        assert np.abs(g).max() > 0, k
        assert _rel(got[k], g) < 1e-10, (k, _rel(got[k], g))
    got = ref.sdf_backward(x.numpy(), cot[0].numpy())
    for k, g in sdf_grads.items():
        assert _rel(got[k], g) < 1e-10, (k, _rel(got[k], g))


def _ulps(a, b):
    """fraction of fp16 values that differ, and the largest difference in fp16 ulps of the reference value"""
    a16, b16 = np.asarray(a).astype(np.float16).astype(np.float64), np.asarray(b).astype(np.float16).astype(np.float64)
    ulp = np.maximum(np.abs(b16), 6.1e-5) * 2.0 ** -10
    d = np.abs(a16 - b16)
    return float((d > 0).mean()), float((d / ulp).max())


def test_rounded_reference_forward_matches_autocast_restatement():
    P = onets.LoTDNeuSParams(seed=5, lotd_cfg=CFG16, lotd_bound=0.5)
    x, v, ha, _ = _inputs(3000, P.n_appear, seed=4, lo=-1.0, hi=1.0)
    x[:8] = torch.tensor([[-1., -1, -1], [1, 1, 1], [1, 0, 0], [-1, 0.3, 0.2], [0.1, 1, -0.4], [0.2, -0.7, -1], [1, -1, 1], [0, 0, 0]])
    with torch.no_grad():
        want = onets.forward(P, x, v, ha, nablas_has_grad=False)
    ref = fused64.Fused64(P.grid, CFG16, P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3,
                          P.rad_b3, beta=100.0)
    got = ref.color_forward(x.numpy(), v.numpy(), ha.numpy())
    assert np.array_equal(ref.sdf(x.numpy()), got["sdf"])
    # same rounding points; the sums differ only between fp32 (nets) and float64 (here): rare one-ulp fp16 flips
    for k in ("sdf", "rgb"):
        frac, worst = _ulps(got[k], want[k].detach().numpy())
        assert frac < 1.5e-2 and worst <= 1.0, (k, frac, worst)
    err = np.abs(got["nablas"] - want["nablas"].detach().numpy()) / (got["nablas_scale"] + 1e-30)
    assert float(np.quantile(err, 0.99)) < 1e-5 and float(err.max()) < 2e-3, (np.quantile(err, 0.99), err.max())


def test_merge_census_matches_reference_addressing_and_counts_heads():
    """tests/util.py:merge_census, the model of the warp-merged table-gradient scatter that the GPU scatter tests use to assert which
    (warp, level) pairs merge: its cells address the table as Fused64 does, and it counts run heads by the kernel's rule"""
    from util import MERGE_MAX_HEADS, merge_census
    cfg = olotd.gen_ngp_cfg()
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(512, 3, generator=g) * 2 - 1).numpy()
    x[:40] = 0.0                                                    # the point an invalid lane loads
    for max_level in (None, 7):
        ref = fused64.Fused64(np.zeros(olotd.LoDMeta(3, **cfg).n_params, dtype=np.float32), cfg, np.zeros((64, 32)), np.zeros(64),
                              np.zeros((1, 64)), np.zeros(1), max_level=max_level)
        c = merge_census(x, cfg, max_level=max_level)
        levels = list(ref.levels(ref.xs_of(x)))
        assert len(levels) == len(c["levels"]) == (16 if max_level is None else 8)
        for (ooff, idx, w, dw), lvl, cell in zip(levels, c["levels"], c["cells"]):
            loff = ref.meta.level_offsets[lvl]
            assert np.array_equal(olotd.grid_index(ref.meta, lvl, cell) * 2 + loff, idx[0]), lvl
        assert c["mergeable"].tolist() == [r <= 1024 for r in np.array(cfg["lod_res"])[c["levels"]]]
    assert merge_census(x, cfg)["mergeable"].tolist() == [True] * 13 + [False] * 3      # levels 13..15 have more than 1024 cells per axis

    # hand-built warps; level 0 has 14 cells per axis, cell k holds table-space k / 14 at its centre
    cell0 = lambda kx, ky, kz, j=0: np.array([kx, ky, kz], dtype=np.float32) / 7.0 - 1.0 + np.float32(1e-5) * j
    A, B = (3, 4, 5), (3, 4, 6)
    pts = [cell0(*A, j) for j in range(10)] + [cell0(*B, j) for j in range(5)] + [cell0(*A, j) for j in range(9)]
    pts += [cell0(j % 14, j // 14, 1) for j in range(32)]           # warp 1: 32 cells
    pts += [cell0(*B, j) for j in range(32)]                        # warp 2: one cell
    x = np.stack(pts)
    order = np.concatenate([np.arange(24), np.full(8, -1), np.arange(24, 88)])
    active = np.ones(order.shape[0], dtype=bool)
    active[20] = False                                              # lane 20 (cell A): a zero cotangent in k_sdf_bwd_tc
    c = merge_census(x, cfg, order=order, active=active)
    # warp 0: A x10 | B x5 | A x5 | A (inactive) | A x3 | 8 invalid lanes -> 1 + 1 + 1 + 1 + 1 + 8 heads
    assert c["heads"][:, 0].tolist() == [13, 32, 1]
    assert c["heads"][0, 0] <= MERGE_MAX_HEADS < c["heads"][1, 0]
    c = merge_census(x, cfg, order=order)                           # every valid lane active: lanes 15..23 are one run
    assert c["heads"][:, 0].tolist() == [11, 32, 1]
    assert c["valid"].tolist() == [True] * 24 + [False] * 8 + [True] * 64
