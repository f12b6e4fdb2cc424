"""CPU self-test of oracle/neus64.py, the float64 statement of the per-ray NeuS stage kernels: its fp32 replay equals oracle/pack_ops.py
bit for bit, its hand-written backward passes equal torch float64 autograd of the masked forward (decisions fixed), and its float64
values agree with oracle/render.py to fp32 tolerance."""
import numpy as np
import pytest
import torch

from oracle import neus64 as o64, pack_ops as opk, render as orender

F32 = np.float32


def _pi(n):
    n = torch.as_tensor(n, dtype=torch.long)
    return torch.stack([n.cumsum(0) - n, n], 1)


def _alphas(rng, S, thre):
    a = (rng.random(S) ** 3 * 0.9).astype(F32)
    a[rng.random(S) < 0.2] = 0
    a[rng.random(S) < 0.05] = F32(thre)                  # ties with the threshold
    a[rng.random(S) < 0.02] = F32(1 - 2e-6)              # opaque samples
    return a


@pytest.mark.parametrize("thre", [0.0, 0.01])
def test_replay_equals_serial_pack_ops_bit_for_bit(thre):
    rng = np.random.default_rng(1)
    pi = _pi([0, 1, 2, 31, 32, 33, 64, 65, 0, 97, 300, 0])
    S = int(pi[:, 1].sum())
    a = _alphas(rng, S, thre)
    r = o64.replay(a, pi.numpy(), 1e-4, thre)
    w_ref = opk.packed_alpha_to_vw_forward(torch.from_numpy(a), pi, 1e-4, thre, False)[0].numpy()
    _, info, sel = opk.packed_alpha_to_vw_forward(torch.from_numpy(a), pi, 1e-4, thre, True)
    assert np.array_equal(r["w"].view(np.int32), w_ref.view(np.int32))
    assert np.array_equal(r["vis"], sel.numpy()) and np.array_equal(r["steps"], info[:, 1].numpy())
    assert (r["cross"] >= 0).sum() >= 3                                    # some packs stop
    # the backward's own replay (alpha >= thre) with float64 values reproduces the serial fp32 backward to fp32 rounding
    gw = rng.standard_normal(S).astype(F32)
    ga_ref = opk.packed_alpha_to_vw_backward(torch.from_numpy(w_ref), torch.from_numpy(gw), torch.from_numpy(a), pi, 1e-4, thre).numpy()
    rb = o64.replay(a, pi.numpy(), 1e-4, thre, backward=True)
    P = pi.shape[0]
    got = o64.composite_backward(a, np.zeros(S), pi.numpy(), r["w"], rb["T"], rb["vis"], np.zeros(P), np.zeros(P), g_vw=gw,
                                 normalize_depth=False)
    err = np.abs(got["d_alpha"] - ga_ref)
    assert (err <= 64 * o64.U32 * got["d_alpha_scale"] + 1e-30).all(), float((err / np.maximum(got["d_alpha_scale"], 1e-30)).max())
    if thre > 0:                                                           # the tie rule matters on these inputs
        tie = (a == F32(thre)) & rb["vis"]
        assert tie.any() and np.abs(ga_ref[tie]).max() > 0 and not r["vis"][tie].any()


def _no_tie_case(seed, thre):
    rng = np.random.default_rng(seed)
    pi = _pi([1, 5, 33, 70, 2, 40])
    S = int(pi[:, 1].sum())
    a = (rng.uniform(0.05, 0.4, S)).astype(F32)
    a[rng.random(S) < 0.2] = F32(thre / 2)                # skipped by both passes (strictly below thre)
    return rng, pi, a


@pytest.mark.parametrize("normalize_depth", [True, False])
def test_composite_backward_equals_float64_autograd(normalize_depth):
    rng, pi, a = _no_tie_case(2, 0.01)
    S, P = a.shape[0], pi.shape[0]
    r = o64.replay(a, pi.numpy(), 1e-4, 0.01)
    rb = o64.replay(a, pi.numpy(), 1e-4, 0.01, backward=True)
    assert np.array_equal(r["vis"], rb["vis"]) and (r["cross"] >= 0).any()
    t, rgb, nab = rng.uniform(0.5, 3, S), rng.random((S, 3)), rng.standard_normal((S, 3))
    g = dict(g_mask=rng.standard_normal(P), g_depth=rng.standard_normal(P), g_rgb=rng.standard_normal((P, 3)),
             g_nablas=rng.standard_normal((P, 3)), g_vw=rng.standard_normal(S))
    at, rt, nt = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (a.astype(np.float64), rgb, nab))
    vis = torch.from_numpy(r["vis"])
    ws = []
    for b, n in pi.tolist():                                             # the masked forward, decisions fixed
        T = torch.ones((), dtype=torch.float64)
        for j in range(b, b + n):
            if vis[j]:
                ws.append(at[j] * T)
                T = T * (1 - at[j])
            else:
                ws.append(at[j] * 0)
    w = torch.stack(ws)
    pk = torch.from_numpy(o64.pack_of(pi.numpy(), S))
    M = torch.zeros(P, dtype=torch.float64).index_add(0, pk, w)
    sd = torch.zeros(P, dtype=torch.float64).index_add(0, pk, w * torch.from_numpy(t))
    D = sd / (M + 1e-10) if normalize_depth else sd
    C = torch.zeros(P, 3, dtype=torch.float64).index_add(0, pk, w[:, None] * rt)
    Nn = torch.zeros(P, 3, dtype=torch.float64).index_add(0, pk, w[:, None] * nt)
    loss = ((M * torch.from_numpy(g["g_mask"])).sum() + (D * torch.from_numpy(g["g_depth"])).sum() + (C * torch.from_numpy(g["g_rgb"])).sum()
            + (Nn * torch.from_numpy(g["g_nablas"])).sum() + (w * torch.from_numpy(g["g_vw"])).sum())
    loss.backward()
    T64, w64 = o64.transmittance(a, r["vis"], pi.numpy())
    assert np.allclose(w64, w.detach().numpy(), rtol=1e-14, atol=0)
    fw = o64.composite_forward(w64, t, pi.numpy(), rgb, nab, normalize_depth)
    for k, v in (("mask", M), ("depth", D), ("rgb", C), ("nablas", Nn)):
        assert np.allclose(fw[k], v.detach().numpy(), rtol=1e-12, atol=1e-15), k
    got = o64.composite_backward(a, t, pi.numpy(), w64, T64, r["vis"], fw["mask"], fw["depth"], rgb=rgb, nablas=nab, normalize_depth=normalize_depth, **g)
    for k, ref in (("d_alpha", at.grad), ("d_rgb", rt.grad), ("d_nablas", nt.grad)):
        ref = ref.numpy()
        assert np.abs(got[k] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1), k


def test_alpha_backward_equals_float64_autograd():
    rng = np.random.default_rng(3)
    pi = _pi([1, 2, 40, 33, 7])
    S = int(pi[:, 1].sum())
    t = np.concatenate([np.sort(rng.uniform(0, 2, n)) for n in pi[:, 1].tolist()])
    sdf = (1.0 - t + 0.05 * rng.standard_normal(S)).astype(F32)          # crossing with noise: some intervals rise (clamp active)
    inv_s = 20.0
    g = rng.standard_normal(S)
    x = torch.tensor(o64.sigmoid_arg(sdf, inv_s).astype(np.float64), requires_grad=True)
    c = torch.sigmoid(x)
    last = torch.from_numpy(o64._last_mask(pi.numpy(), S))
    c1 = torch.where(last, torch.zeros_like(c), torch.roll(c, -1))
    raw = torch.where(last, torch.zeros_like(c), (c - c1) / (c + 1e-5))
    alpha = raw.clamp_min(0)
    assert (raw < 0).any() and (raw > 0).any()
    (alpha * torch.from_numpy(g)).sum().backward()
    # d/dsdf = dL/dx * inv_s, d/dinv_s = sum dL/dx * sdf (x = sdf * inv_s; the fp32 rounding of x is a decision point)
    got = o64.alpha_backward(sdf, pi.numpy(), inv_s, g)
    ref = x.grad.numpy()
    assert np.abs(got["d_sdf"] - ref * inv_s).max() <= 1e-12 * np.abs(ref * inv_s).max()
    assert abs(got["d_inv_s"] - float((ref * sdf.astype(np.float64)).sum())) <= 1e-12 * np.abs(ref * sdf).sum()
    a64, _ = o64.neus_alpha(sdf, pi.numpy(), inv_s)
    assert np.abs(a64 - alpha.detach().numpy()).max() <= 1e-15


@pytest.mark.parametrize("estimate", [False, True])
def test_values_agree_with_render_oracle(estimate):
    rng = np.random.default_rng(4)
    pi = _pi([3, 1, 64, 97, 33, 250])
    S = int(pi[:, 1].sum())
    t = np.concatenate([np.sort(rng.uniform(0.5, 2.5, n)) for n in pi[:, 1].tolist()]).astype(F32)
    sdf = ((1.4 - t) * 0.8 + 0.02 * rng.standard_normal(S)).astype(F32)
    inv_s = 64.0
    st, tt = torch.from_numpy(sdf), torch.from_numpy(t)
    if estimate:
        a_ref = orender.neus_packed_sdf_to_upsample_alpha(st, tt, inv_s, pi).numpy()
        a64 = o64.upsample_alpha(sdf, t, pi.numpy(), inv_s)
    else:
        a_ref = orender.neus_packed_sdf_to_alpha(st, inv_s, pi).numpy()
        a64, _ = o64.neus_alpha(sdf, pi.numpy(), inv_s)
    assert np.abs(a64 - a_ref).max() <= 2e-5, float(np.abs(a64 - a_ref).max())
    r = o64.replay(a_ref, pi.numpy(), 1e-4, 0.0)
    cdf64, _ = o64.upsample_cdf(r["w"], pi.numpy())
    vw = orender.packed_alpha_to_vw(torch.from_numpy(a_ref), pi)
    cdf = orender.packed_cumsum_exclusive(vw, pi)
    cdf = orender.packed_div(cdf, cdf[pi[:, 0] + pi[:, 1] - 1].clamp_min(1e-5), pi).numpy()
    assert np.abs(cdf64 - cdf).max() <= 1e-5
    u = np.linspace(0, 1, 35, dtype=F32)[1:-1]
    s64, _ = o64.invert_cdf(t, cdf.astype(F32), u, pi.numpy())
    s_ref = orender.packed_sample_cdf(tt, torch.from_numpy(cdf.astype(F32)), pi, 33)[0].numpy()
    assert np.abs(s64 - s_ref).max() <= 1e-6 * np.abs(t).max()
    # an empty pack has no bin: NaN
    s_e, _ = o64.invert_cdf(t, cdf.astype(F32), u, np.array([[S, 0]]))
    assert np.isnan(s_e).all()
