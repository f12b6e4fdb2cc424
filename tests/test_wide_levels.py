"""CPU: LoTD tables of 17..24 levels in the 48-column layout of the fused kernels: the float64 reference (tests/fused64_wide.py) against the
autocast restatement, the wide radiance-input column map (csrc/color_tc.cu ref_col with a 48-column h tile), the max_fused_levels option
of the predicates, and the level counts auto_ngp_cfg gives the shipped StreetSurf camera models."""
import numpy as np
import pytest
import torch

from fused64_wide import H_WIDE, Fused64Wide, ref_col_wide
from oracle import lotd as olotd, nets as onets
from test_partial_levels import _ref_col, _rel, _ulps


def _setup(levels, n=1500, seed=7):
    cfg = olotd.gen_ngp_cfg(log2_hashmap_size=14, num_levels=levels)
    P = onets.LoTDNeuSParams(seed=seed, lotd_cfg=cfg, lotd_bound=0.5)
    nh = 2 * levels
    assert P.meta.n_pseudo_levels == levels and tuple(P.dec_W1.shape) == (64, nh) and tuple(P.rad_W1.shape) == (64, 22 + nh + P.n_appear)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.rand(n, 3, generator=g) * 1.9 - 0.95
    v = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ha = torch.randn(n, P.n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    ref = Fused64Wide(P.grid, cfg, P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3, P.rad_b3, beta=100.0)
    assert ref.nh == nh and ref.n_appear == P.n_appear
    return P, x, v, ha, cot, ref


@pytest.mark.parametrize("levels", [17, 19])
def test_fused64_wide_matches_autocast_restatement_forward(levels):
    P, x, v, ha, _cot, ref = _setup(levels)
    nh = 2 * levels
    with torch.no_grad():
        want = onets.forward(P, x, v, ha, nablas_has_grad=False)
    got = ref.color_forward(x.numpy(), v.numpy(), ha.numpy())
    assert got["h"].shape[1] == H_WIDE and not got["h"][:, nh:].any() and not got["J"][:, nh:].any() and got["h"][:, 32:nh].any()
    assert np.array_equal(ref.sdf(x.numpy()), got["sdf"])
    for k in ("sdf", "rgb"):
        frac, worst = _ulps(got[k], want[k].detach().numpy())
        # at most one fp16 step (_ulps measures it in units of |want| 2^-10, so a step just below a power of two reads as up to ~1.001)
        assert frac < 1.5e-2 and worst <= 1.002, (k, frac, worst)
    err = np.abs(got["nablas"] - want["nablas"].detach().numpy()) / (got["nablas_scale"] + 1e-30)
    assert float(np.quantile(err, 0.99)) < 1e-5 and float(err.max()) < 2e-3, (np.quantile(err, 0.99), err.max())


@pytest.mark.parametrize("levels", [17, 19])
def test_fused64_wide_matches_autocast_restatement_gradients(levels):
    P, x, v, ha, cot, ref = _setup(levels, n=1500, seed=11)
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


@pytest.mark.parametrize("levels", list(range(17, 25)))
@pytest.mark.parametrize("n_appear", list(range(0, 9)))
def test_wide_radiance_column_map(levels, n_appear):
    nh = 2 * levels
    rin = 22 + nh + n_appear
    cols = [ref_col_wide(k, n_appear, nh) for k in range(H_WIDE + 32)]
    assert sorted(c for c in cols if c >= 0) == list(range(rin))          # every reference column exactly once, nothing past rad_in
    assert cols[:nh] == list(range(22, 22 + nh)) and all(c == -1 for c in cols[nh:H_WIDE])
    assert cols[48:51] == [0, 1, 2] and cols[51:67] == list(range(3, 19)) and cols[67:70] == [19, 20, 21]
    assert cols[70:70 + n_appear] == list(range(rin - n_appear, rin)) and all(c == -1 for c in cols[70 + n_appear:])
    # the wide map is the 32-column one shifted by the 16 extra h columns
    assert [ref_col_wide(k, n_appear, 24, hc=32) for k in range(64)] == [_ref_col(k, n_appear, 24) for k in range(64)]


# ===================================================================================================================== predicates
def _model(levels, **kw):
    from neuralsim_b200.fields.neus import LoTDNeuS
    cfg = olotd.gen_ngp_cfg(log2_hashmap_size=12, num_levels=levels)
    return LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=cfg), **kw), radiance_cfg=dict(W=64, n_appear_embedding=0))


def _fusable_on_cuda(model):
    """the predicates with the table taken as a CUDA tensor (the only precondition a CPU build cannot meet)"""
    s = model.implicit_surface

    class _Cuda:
        is_cuda = True
    try:
        s.encoding.__dict__["flattened_params"] = _Cuda()                     # shadows the parameter (nn.Module looks there last)
        return s._fusable(), model._color_fusable(), model._geometry_fusable()
    finally:
        del s.encoding.__dict__["flattened_params"]


def test_default_bound_is_16_levels():
    from neuralsim_b200.fields.networks import LoTDSDF
    assert LoTDSDF().max_fused_levels == 16
    m = _model(17)
    assert m.implicit_surface.max_fused_levels == 16
    assert _fusable_on_cuda(m) == (False, False, False)
    assert _fusable_on_cuda(_model(16)) == (True, True, True)


@pytest.mark.parametrize("levels", [16, 17, 19, 23, 24, 25])
def test_bound_24_accepts_17_to_24_levels(levels):
    m = _model(levels, max_fused_levels=24)
    assert m.implicit_surface.max_fused_levels == 24
    want = levels <= 24
    assert _fusable_on_cuda(m) == (want, want, want)


@pytest.mark.parametrize("bad", [0, 15, 17, 20, 25, 32, None, True, "24", 24.5])
def test_bad_bound_raises(bad):
    from neuralsim_b200.fields.networks import LoTDSDF
    with pytest.raises(ValueError, match="max_fused_levels"):
        LoTDSDF(max_fused_levels=bad)
    with pytest.raises(ValueError, match="max_fused_levels"):
        _model(17, max_fused_levels=bad)


# ===================================================================================================================== auto_ngp_cfg
def test_auto_ngp_cfg_street_box_and_cube_fit_the_wide_kernels():
    """the shipped camera encoding (ngp, 32 Mi parameters, 2^20 hash map, no level cap): 2 dense + 15 hashed = 17 levels on the cfg3 street
    box, 4 dense + 15 hashed = 19 on a cube -- both within the 24 levels of the 48-column kernels"""
    from neuralsim_b200.fields.encoding import auto_ngp_cfg
    for box, want in (([40., 150., 15.], 17), ([50., 50., 50.], 19)):
        c = auto_ngp_cfg(box, 32 * 2 ** 20, dim=3, n_feats=2, log2_hashmap_size=20, min_res=16, max_num_levels=None)
        n = len(c["lod_res"])
        assert n == want and c["lod_types"].count("Dense") == want - 15, (box, n, c["lod_types"])
        assert 16 < n <= 24
