"""CPU: LoTD tables of fewer than 16 levels (L levels of 2 features, 2L decoder inputs) in the float64 reference of the fused kernels
(oracle/fused64.py through tests/fused64_levels.py) and in the radiance-input column map of the colour kernels (csrc/color_tc.cu: ref_col)."""
import numpy as np
import pytest
import torch

from fused64_levels import Fused64Levels, h_cols
from oracle import lotd as olotd, nets as onets

L12 = olotd.gen_ngp_cfg(log2_hashmap_size=14, num_levels=12)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _ulps(a, b):
    a16, b16 = np.asarray(a).astype(np.float16).astype(np.float64), np.asarray(b).astype(np.float16).astype(np.float64)
    d = np.abs(a16 - b16)
    return float((d > 0).mean()), float((d / (np.maximum(np.abs(b16), 6.1e-5) * 2.0 ** -10)).max())


def _setup(n=2000, seed=7):
    P = onets.LoTDNeuSParams(seed=seed, lotd_cfg=L12, lotd_bound=0.5)
    assert P.meta.n_pseudo_levels == 12 and P.meta.n_encoded_dims == 24 and tuple(P.dec_W1.shape) == (64, 24)
    assert tuple(P.rad_W1.shape) == (64, 22 + 24 + P.n_appear)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.rand(n, 3, generator=g) * 1.9 - 0.95
    v = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ha = torch.randn(n, P.n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    ref = Fused64Levels(P.grid, L12, P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3, P.rad_b3,
                          beta=100.0)
    assert ref.nh == 24 and ref.n_appear == P.n_appear
    return P, x, v, ha, cot, ref


def test_fused64_at_12_levels_matches_autocast_restatement_forward():
    P, x, v, ha, _cot, ref = _setup()
    with torch.no_grad():
        want = onets.forward(P, x, v, ha, nablas_has_grad=False)
    got = ref.color_forward(x.numpy(), v.numpy(), ha.numpy())
    assert not got["h"][:, 24:].any() and not got["J"][:, 24:].any() and got["h"][:, :24].any()
    assert np.array_equal(ref.sdf(x.numpy()), got["sdf"])
    for k in ("sdf", "rgb"):
        frac, worst = _ulps(got[k], want[k].detach().numpy())
        assert frac < 1.5e-2 and worst <= 1.0, (k, frac, worst)
    err = np.abs(got["nablas"] - want["nablas"].detach().numpy()) / (got["nablas_scale"] + 1e-30)
    assert float(np.quantile(err, 0.99)) < 1e-5 and float(err.max()) < 2e-3, (np.quantile(err, 0.99), err.max())


def test_fused64_at_12_levels_matches_autocast_restatement_gradients():
    """the hand-written backward passes against autograd through oracle/nets.py, which rounds every cotangent to fp16 (the fused kernels
    and fused64 keep them in fp32): agreement to the fp16 rounding of the cotangents"""
    P, x, v, ha, cot, ref = _setup(n=1500, seed=11)
    P.requires_grad_(True)
    names = dict(grid="grid", W1="dec_W1", b1="dec_b1", W2="dec_W2", b2="dec_b2", R1="rad_W1", rb1="rad_b1", R2="rad_W2", rb2="rad_b2",
                 R3="rad_W3", rb3="rad_b3")
    out = onets.forward(P, x, v, ha, nablas_has_grad=True)
    loss = (out["sdf"] * cot[0]).sum() + (out["nablas"] * cot[1]).sum() + (out["rgb"] * cot[2]).sum()
    want = dict(zip(names, torch.autograd.grad(loss, [getattr(P, n) for n in names.values()])))
    fwd = ref.color_forward(x.numpy(), v.numpy(), ha.numpy())
    got = ref.color_backward(fwd, *(c.numpy() for c in cot))
    for k in names:
        assert got[k].shape == tuple(want[k].reshape(got[k].shape).shape), k
        e = _rel(got[k], want[k].reshape(got[k].shape).numpy())
        assert e < 2e-2, (k, e)
    sdf = onets.forward_sdf(P, x)["sdf"]
    keys = ("grid", "W1", "b1", "W2", "b2")
    want = dict(zip(keys, torch.autograd.grad((sdf * cot[0]).sum(), [getattr(P, names[k]) for k in keys])))
    got = ref.sdf_backward(x.numpy(), cot[0].numpy())
    for k in keys:
        e = _rel(got[k], want[k].reshape(got[k].shape).numpy())
        assert e < 2e-2, (k, e)


def _ref_col(k, n_appear, nh):
    """csrc/color_tc.cu ref_col: internal radiance-input column k ([h(32, nh used) | x | SH | n | h_appear | 0]) -> reference column"""
    if k < 32:
        return 22 + k if k < nh else -1
    if k < 35:
        return k - 32
    if k < 51:
        return 3 + (k - 35)
    if k < 54:
        return 19 + (k - 51)
    if k < 54 + n_appear:
        return 22 + nh + (k - 54)
    return -1


@pytest.mark.parametrize("levels", [1, 11, 12, 16])
@pytest.mark.parametrize("n_appear", [0, 4, 8])
def test_radiance_column_map(levels, n_appear):
    nh = 2 * levels
    rin = 22 + nh + n_appear
    cols = [_ref_col(k, n_appear, nh) for k in range(64)]
    used = [c for c in cols if c >= 0]
    assert sorted(used) == list(range(rin))                    # every reference column exactly once, nothing past rad_in
    # the blocks land where the reference concatenates them: [x(3) | SH(16) | n(3) | h(2L) | h_appear]
    assert cols[32:35] == [0, 1, 2] and cols[35:51] == list(range(3, 19)) and cols[51:54] == [19, 20, 21]
    hc = h_cols(nh)
    assert cols[:nh] == list(range(hc.start, hc.stop)) and all(c == -1 for c in cols[nh:32])
    assert cols[54:54 + n_appear] == list(range(rin - n_appear, rin)) and all(c == -1 for c in cols[54 + n_appear:])
    if levels == 16:                                           # the 16-level map: h at 22..53, h_appear at 54..
        assert cols[:32] == list(range(22, 54)) and cols[54:54 + n_appear] == list(range(54, 54 + n_appear))
