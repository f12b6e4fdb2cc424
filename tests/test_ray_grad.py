"""CPU: the float64 ray gradient (tests/rays64.py on oracle/fused64.py) -- per sample and per ray -- against torch float64 autograd of a
float64 trilinear restatement of the query in which the depths are constants and the encoding's Jacobian is not differentiated."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fused64, lotd as olotd, nets as onets
from rays64 import color_rows, ray_grads, sdf_rows

CFG16 = olotd.gen_ngp_cfg(log2_hashmap_size=14)


def _ref(seed, n_appear=4):
    g = torch.Generator().manual_seed(seed)
    meta = olotd.LoDMeta(3, **CFG16)
    table = (torch.rand(meta.n_params, generator=g) * 2 - 1) * 0.5
    lin = lambda o, i: onets.kaiming_linear(g, o, i)
    ws = [*lin(64, 32), *lin(1, 64), *lin(64, 54 + n_appear), *lin(64, 64), *lin(3, 64)]
    return fused64.Fused64(table, CFG16, *ws, rounding=False, beta=20.0)


def _case(seed, n_rays=30, n_appear=4):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, 12, (n_rays,), generator=g)
    ridx = torch.repeat_interleave(torch.arange(n_rays), lens)
    o = (torch.rand(n_rays, 3, generator=g) * 1.2 - 0.6).double()
    d = F.normalize(torch.randn(n_rays, 3, generator=g), dim=-1).double()
    t = (torch.rand(ridx.shape[0], generator=g) * 0.3).double()
    v = F.normalize(torch.randn(n_rays, 3, generator=g), dim=-1).double()
    ha = (torch.randn(n_rays, n_appear, generator=g) * 0.5).double()
    n = ridx.shape[0]
    cot = (torch.randn(n, generator=g).double(), torch.randn(n, 3, generator=g).double() * 0.1, torch.randn(n, 3, generator=g).double())
    return ridx, o, d, t, v, ha, cot


def _torch_query(ref, x64, xs_np):
    """h(x) by trilinear interpolation with weights that are differentiable in x (their value at the fp32 point), and the Jacobian J
    held constant"""
    h = [None] * 32
    meta = ref.meta
    for psl, lvl, loff, foff, ooff in olotd._level_iter(meta, ref.max_level):
        res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        cell, frac = olotd.pos_fract(xs_np, scale)
        fr = torch.from_numpy(frac.astype(np.float64)) + (x64 - x64.detach()) * 0.5 * torch.from_numpy(scale.astype(np.float64))
        for f in range(2):
            acc = 0.0
            for c in range(8):
                off = np.array([(c >> k) & 1 for k in range(3)], dtype=np.uint32)
                idx = olotd.grid_index(meta, lvl, cell + off) * meta.level_n_feats[lvl] + foff + loff
                w = 1.0
                for k in range(3):
                    w = w * (fr[:, k] if (c >> k) & 1 else 1.0 - fr[:, k])
                acc = acc + torch.from_numpy(ref.T[idx + f]) * w
            h[ooff + f] = acc
    z0 = torch.zeros_like(x64[:, 0])
    return torch.stack([c if c is not None else z0 for c in h], -1)


def _torch_grads(ref, ridx, o, d, t, v, ha, cot, *, rgb=True, sdf_only=False):
    o, d, v = (a.clone().requires_grad_(True) for a in (o, d, v))
    x64 = o[ridx] + d[ridx] * t[:, None]
    x32 = x64.detach().float().numpy()
    xt = torch.from_numpy(x32.astype(np.float64)) + (x64 - x64.detach())      # the fp32 point the reference evaluates, gradient 1
    xs_np = ref.xs_of(x32)
    h = _torch_query(ref, xt, xs_np)
    tt = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    z = h @ tt(ref.W1).T + tt(ref.b1)
    a = F.softplus(z, beta=ref.beta, threshold=20.0)
    sdf = (a @ tt(ref.W2).T + tt(ref.b2))[:, 0]
    loss = (sdf * cot[0]).sum()
    if not sdf_only:
        g = torch.autograd.grad(sdf.sum(), h, create_graph=True)[0]
        _, J = ref.features(xs_np)
        nab = torch.einsum("nf,nfd->nd", g, tt(J)) * 0.5 * tt(ref.fac)
        loss = loss + (nab * cot[1]).sum()
        if rgb:
            X = torch.cat([xt, onets.sh_encode(v[ridx], 4), nab.detach().clamp(-1, 1), h, ha[ridx]], -1)
            Y1 = torch.relu(X @ tt(ref.R1).T + tt(ref.rb1))
            Y2 = torch.relu(Y1 @ tt(ref.R2).T + tt(ref.rb2))
            out = torch.sigmoid(Y2 @ tt(ref.R3).T + tt(ref.rb3))
            loss = loss + (out * cot[2]).sum()
    go, gd, gv = torch.autograd.grad(loss, (o, d, v), allow_unused=True)
    return x32, go.numpy(), gd.numpy(), (gv.numpy() if gv is not None else np.zeros_like(go.numpy()))


def _close(got, want):
    assert np.abs(want).max() > 0
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize("rgb", [True, False], ids=["colour", "geometry"])
def test_colour_ray_gradient_is_autograd_of_the_restated_query(rgb):
    ref = _ref(seed=5)
    ridx, o, d, t, v, ha, cot = _case(seed=6)
    x32, go, gd, gv = _torch_grads(ref, ridx, o, d, t, v, ha, cot, rgb=rgb)
    fwd = ref.color_forward(x32, v[ridx].numpy(), ha[ridx].numpy())
    g_x, g_v = color_rows(ref, fwd, v[ridx].numpy(), cot[0].numpy(), cot[1].numpy(), cot[2].numpy() if rgb else None)
    d_o, d_d, d_v = ray_grads(g_x, t.numpy(), ridx.numpy(), o.shape[0], g_v)
    _close(d_o, go)
    _close(d_d, gd)
    if rgb:
        _close(d_v, gv)
    else:
        assert (d_v == 0).all() and (gv == 0).all()
    empty = np.setdiff1d(np.arange(o.shape[0]), ridx.numpy())
    assert empty.size >= 1 and (d_o[empty] == 0).all()


def test_sdf_ray_gradient_is_autograd_of_the_restated_query():
    ref = _ref(seed=7)
    ridx, o, d, t, v, ha, cot = _case(seed=8)
    x32, go, gd, _ = _torch_grads(ref, ridx, o, d, t, v, ha, cot, sdf_only=True)
    d_o, d_d, _ = ray_grads(sdf_rows(ref, x32, cot[0].numpy()), t.numpy(), ridx.numpy(), o.shape[0])
    _close(d_o, go)
    _close(d_d, gd)
