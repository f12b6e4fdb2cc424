"""The five wgmma kernels of the hot path against the float64 reference of their numerics contract (oracle/fused64.py):
k_fused_sdf_tc / k_sdf_bwd_tc (csrc/fused_tc.cu), k_color_fwd / k_color_rad_bwd / k_color_sdf_bwd (csrc/color_tc.cu).

The kernels run persistent grids, so the sizes are chosen from the SM count: every CTA loops over several tiles (the TMA prefetch
of the next tile, the mbarrier phases and the weight-gradient sums that accumulate over a CTA's tiles all run) and the last tile
is partial.  Forward outputs are compared per element (fraction of fp16 values that differ, largest difference in fp16 ulps),
so a wrong tile shows up as 128 wrong rows.  Backward passes are compared with every cotangent set, and with the cotangent
restricted to one tile at a time while the kernel still runs over all points.  Bounds are about 3x the errors measured on an
H100 80GB HBM3 (132 SMs, 400 W power limit); DESIGN.md §4 lists them."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import fused64, lotd as olotd

pytestmark = pytest.mark.gpu

TILE = 128
# CTAs per SM of the persistent grids: kSdfCtasPerSM and persistent_grid(tiles, 2) in nsb_fused_sdf_bwd (csrc/fused_tc.cu);
# persistent_grid(tiles, 2) for k_color_fwd and persistent_grid(tiles, 1) for both colour backward kernels (csrc/color_tc.cu)
CTAS_PER_SM = dict(sdf_fwd=4, sdf_bwd=2, color_fwd=2, color_bwd=1)

# (decoder width, radiance width, n_appear), max_level; the first is the production configuration
PRODUCTION = ((64, 64, 4), None)
CASES = [PRODUCTION, ((64, 64, 4), 7), ((48, 40, 0), None), ((48, 40, 0), 7), ((64, 64, 8), None), ((16, 64, 1), 7)]
CASE_IDS = [f"w{c[0]}-r{c[1]}-a{c[2]}-ml{m}" for c, m in CASES]

# Bounds.  Forwards: fraction of fp16 values that differ, largest difference in fp16 ulps (_fp16_metrics), nablas error relative
# to 0.5 fac sum |r16(g) J| (one fp16 flip of g moves it by <= 2^-11 of that).  Backward: rel-L2 of each gradient.  With every
# cotangent set and random in sign the hidden-layer gradients of the radiance net cancel down to ~1/sqrt(n) of their terms, and a
# rare ReLU mask that flips with a one-ulp change of its input changes one term by O(1): those four sit near 2e-3 (a tile's share
# is 1/sqrt(n_tiles) ~ 4e-2).  With one tile's cotangent everything agrees to ~5e-5.
SDF_FLIP_FRAC, SDF_MAX_ULP = 7e-3, 2.5              # measured <= 2.3e-3, 0.84
RGB_FLIP_FRAC, RGB_MAX_ULP = 3e-3, 3.0              # measured <= 8.9e-4, 1.0
NAB_MAX_REL, NAB_FRAC_1E5 = 2e-3, 1.5e-2            # measured <= 5.7e-4; fraction of elements above 1e-5 <= 4.2e-3
BWD_REL = dict(grid=1e-4, W1=6e-5, b1=1e-4, W2=8e-5, b2=5e-6, R1=6e-3, rb1=6e-3, R2=6e-3, rb2=6e-3, R3=2e-4, rb3=6e-5)
TILE_REL = {k: 1.5e-4 for k in BWD_REL}             # measured <= 4.6e-5


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid(kernel, n):
    return min(-(-n // TILE), _sms() * CTAS_PER_SM[kernel])


def _size(kernel, iters):
    """the smallest n at which every CTA of `kernel` runs at least `iters` tiles, with a partial last tile"""
    return (iters * _sms() * CTAS_PER_SM[kernel] + 1) * TILE - 51


def _assert_multi_tile(kernel, n, iters):
    n_tiles = -(-n // TILE)
    assert n % TILE != 0 and n_tiles // _grid(kernel, n) >= iters, (kernel, n, n_tiles, _grid(kernel, n))


def _fp16_metrics(got, want, scale):
    """fraction of fp16 values that differ, and the largest difference in fp16 ulps of max(|want|, scale): a value whose inputs
    cancel (an sdf near zero) moves by ulps of its inputs' scale, not of its own, when one of them flips across a rounding boundary"""
    a = np.asarray(got, dtype=np.float64).astype(np.float16).astype(np.float64)
    b = np.asarray(want, dtype=np.float64).astype(np.float16).astype(np.float64)
    d = np.abs(a - b)
    return float((d > 0).mean()), float((d / (np.maximum(np.maximum(np.abs(b), scale), 6.1e-5) * 2.0 ** -10)).max())


def _rel(got, want):
    got, want = np.asarray(got, dtype=np.float64).ravel(), np.asarray(want, dtype=np.float64).ravel()
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-300))


def _model(width, rw, n_appear, seed):
    from neuralsim_b200.fields.neus import LoTDNeuS
    gen = torch.Generator("cuda").manual_seed(seed)
    model = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg()), decoder_cfg=dict(W=width)),
                     radiance_cfg=dict(W=rw, n_appear_embedding=n_appear), device="cuda", generator=gen)
    with torch.no_grad():      # table values of order 0.1..1 (the weights keep their Kaiming-uniform init)
        model.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=gen)
    assert model._color_fusable()
    return model


def _inputs(n, n_appear, seed):
    """one ray per point: x = o + d t (t = 0 for the points put on the box faces and corners), view direction, h_appear"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g) * 2 - 1
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    t = torch.rand(n, generator=g) * 0.3
    special = torch.tensor([[-1., -1, -1], [1, 1, 1], [1, -1, 1], [1, 0.3, -0.2], [-1, 0.5, 0.5], [0.2, 1, -0.9], [0.7, -1, 0.1],
                            [-0.3, 0.4, 1], [0.5, 0.5, -1]])
    rows = (torch.arange(4 * len(special)) * 7919) % n
    x[rows] = special.repeat(4, 1)
    t[rows] = 0.0
    o = (x - d * t[:, None]).float()
    xe = (d.double() * t.double()[:, None] + o.double()).float()       # the kernels' fma(d, t, o)
    v = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ha = torch.randn(n, n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    return dict(x=xe, o=o, d=d, t=t, v=v, ha=ha, ridx=torch.arange(n), cot=cot)


def _cuda(inp, *keys):
    return [inp[k].cuda() for k in keys]


_CACHE = {}


@pytest.fixture(scope="module", params=CASES, ids=CASE_IDS)
def case(request):
    """module scope: pytest groups the tests of one configuration, so its model and reference are built once"""
    return request.param


def _case(case):
    """model, inputs, float64 reference and its colour forward for one configuration (built once per module)"""
    if case not in _CACHE:
        (width, rw, n_appear), max_level = case
        full = case == PRODUCTION
        n = _size("color_fwd", 3 if full else 2)
        model = _model(width, rw, n_appear, seed=width + 3 * rw + n_appear)
        model.max_level = max_level
        inp = _inputs(n, n_appear, seed=n_appear + 11)
        ref = fused64.Fused64.from_model(model, max_level=max_level)
        fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy())
        for k in [k for k in _CACHE if k != PRODUCTION]:
            del _CACHE[k]
        _CACHE[case] = (model, inp, ref, fwd)
    return _CACHE[case]


def _params(model):
    s, r = model.implicit_surface, model.radiance_net.blocks.layers
    d = s.decoder.layers
    return dict(grid=s.encoding.flattened_params, W1=d[0].weight, b1=d[0].bias, W2=d[1].weight, b2=d[1].bias, R1=r[0].weight,
                rb1=r[0].bias, R2=r[1].weight, rb2=r[1].bias, R3=r[2].weight, rb3=r[2].bias)


def _color_fwd(model, inp):
    ridx, t, o, d, v = _cuda(inp, "ridx", "t", "o", "d", "v")
    ha = inp["ha"].cuda() if model.use_h_appear else None
    return model.forward_on_rays(ridx, t, o, d, v, ha)


def _color_grads(model, out, cot, retain=False):
    c_sdf, c_nab, c_rgb = (c.cuda() for c in cot)
    loss = (out["sdf"] * c_sdf).sum() + (out["nablas"] * c_nab).sum() + (out["rgb"] * c_rgb).sum()
    p = _params(model)
    return dict(zip(p, torch.autograd.grad(loss, list(p.values()), retain_graph=retain)))


def _sdf_bwd_direct(model, x, d_sdf, max_level):
    """nsb_fused_sdf_bwd over all n points (the autograd op compacts the points with a zero cotangent away)"""
    from neuralsim_b200 import _lib as L
    s = model.implicit_surface
    grid16, dec = s._fused_state()
    p = _params(model)
    g = {k: torch.zeros(p[k].shape, dtype=torch.float32, device="cuda") for k in ("grid", "W1", "b1", "W2", "b2")}
    L.check(L.lib().nsb_fused_sdf_bwd(s.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), L.ptr(x, "f32"), None, None, None, None,
                                      L.ptr(d_sdf, "f32"), L.c_i64(x.shape[0]), L.c_i32(s._ml(max_level)), L.ptr(g["grid"]), L.ptr(g["W1"]),
                                      L.ptr(g["b1"]), L.ptr(g["W2"]), L.ptr(g["b2"]), L.stream_ptr()), "fused_sdf_bwd")
    return g


def _compare_grads(got, want, bounds, what):
    errs = {k: _rel(got[k].detach().double().cpu().numpy(), want[k]) for k in want}
    print(f"METRIC {what} " + " ".join(f"{k}={e:.2e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert np.abs(want[k]).max() > 0, (what, k)
        assert e < bounds[k], (what, k, e, bounds[k])


def _tile_rows(n):
    """8 rows of every tile, at positions that cycle through all 128 (13 is odd), plus the whole partial last tile"""
    n_tiles = -(-n // TILE)
    tiles = np.arange(n_tiles)[:, None]
    rows = (tiles * TILE + (tiles * 13 + np.arange(8)[None, :] * 16) % TILE).ravel()
    rows = np.union1d(rows[rows < n], np.arange((n_tiles - 1) * TILE, n))
    return rows


# ===================================================================================================================== forward
def test_sdf_forward_per_element(case):
    (width, rw, n_appear), max_level = case
    model, inp, ref, _ = _case(case)
    n = _size("sdf_fwd", 3 if case == PRODUCTION else 2)
    _assert_multi_tile("sdf_fwd", n, 3 if case == PRODUCTION else 2)
    big = _inputs(n, n_appear, seed=5)
    s = model.implicit_surface
    x, ridx, t, o, d = _cuda(big, "x", "ridx", "t", "o", "d")
    with torch.no_grad():
        got = dict(points=s.fused_sdf(x, max_level=max_level), rays=s.fused_sdf_rays(ridx, t, o, d, max_level=max_level))
    rows = _tile_rows(n)
    want, scale = ref.sdf(big["x"].numpy()[rows], with_scale=True)
    m = {k: _fp16_metrics(v.cpu().numpy()[rows], want, scale) for k, v in got.items()}
    print(f"METRIC sdf_fwd {case} rows={len(rows)} " + " ".join(f"{k}: flips={f:.2e} max_ulp={u:.2f}" for k, (f, u) in m.items()))
    for k, (frac, worst) in m.items():
        assert frac <= SDF_FLIP_FRAC and worst <= SDF_MAX_ULP, (k, frac, worst)


def test_color_forward_per_element(case):
    model, inp, ref, fwd = _case(case)
    n = inp["x"].shape[0]
    _assert_multi_tile("color_fwd", n, 3 if case == PRODUCTION else 2)
    # the inputs reach both sides of every branch
    assert 0.01 < float(fwd["lin"].mean()) < 0.99
    for k in ("Y1", "Y2"):
        assert 0.1 < float((fwd[k] > 0).mean()) < 0.9, k
    assert 0.01 < float((np.abs(fwd["nablas"]) < 1).mean()) < 0.99
    with torch.no_grad():
        got = _color_fwd(model, inp)
    assert torch.equal(got["x"].cpu(), inp["x"])
    sdf = _fp16_metrics(got["sdf"].cpu().numpy(), fwd["sdf"], fwd["sdf_scale"])
    rgb = _fp16_metrics(got["rgb"].cpu().numpy(), fwd["rgb"], 0.5)          # rgb in units of 2^-11, the fp16 ulp of [0.5, 1)
    nab = np.abs(got["nablas"].cpu().numpy() - fwd["nablas"]) / (fwd["nablas_scale"] + 1e-30)
    print(f"METRIC color_fwd {case} sdf: flips={sdf[0]:.2e} max_ulp={sdf[1]:.2f} rgb: flips={rgb[0]:.2e} max_ulp={rgb[1]:.2f} "
          f"nablas: max_rel={nab.max():.2e} frac>1e-5={(nab > 1e-5).mean():.2e}")
    assert sdf[0] <= SDF_FLIP_FRAC and sdf[1] <= SDF_MAX_ULP, sdf
    assert rgb[0] <= RGB_FLIP_FRAC and rgb[1] <= RGB_MAX_ULP, rgb
    assert float(nab.max()) <= NAB_MAX_REL and float((nab > 1e-5).mean()) <= NAB_FRAC_1E5


# ===================================================================================================================== backward
def test_color_backward_full(case):
    model, inp, ref, fwd = _case(case)
    _assert_multi_tile("color_bwd", inp["x"].shape[0], 3)
    got = _color_grads(model, _color_fwd(model, inp), inp["cot"])
    want = ref.color_backward(fwd, *(c.numpy() for c in inp["cot"]))
    _compare_grads(got, want, BWD_REL, f"color_bwd {case}")


def test_sdf_backward_full(case):
    model, inp, ref, _ = _case(case)
    n = inp["x"].shape[0]
    _assert_multi_tile("sdf_bwd", n, 2)
    x, c = inp["x"].cuda(), inp["cot"][0].cuda()
    p = _params(model)
    keys = ("grid", "W1", "b1", "W2", "b2")
    sdf = model.implicit_surface.fused_sdf_autograd(x, max_level=case[1])
    got = dict(zip(keys, torch.autograd.grad((sdf * c).sum(), [p[k] for k in keys])))
    _compare_grads(got, ref.sdf_backward(inp["x"].numpy(), inp["cot"][0].numpy()), BWD_REL, f"sdf_bwd {case}")


def _tiles_to_check(kernel, n):
    """tiles at a first, a second and a third iteration of a CTA (the latter two were prefetched while the CTA finished the tile
    before) and the partial last tile"""
    g = _grid(kernel, n)
    return dict(first=0, second=g + 1, third=2 * g + 2, last=-(-n // TILE) - 1)


@pytest.mark.parametrize("which", ["first", "second", "third", "last"])
def test_color_backward_one_tile(which):
    model, inp, ref, fwd = _case(PRODUCTION)
    n = inp["x"].shape[0]
    tile = _tiles_to_check("color_bwd", n)[which]
    rows = np.arange(tile * TILE, min(n, (tile + 1) * TILE))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[rows] = True
    cot = [c * mask.view(-1, *[1] * (c.dim() - 1)) for c in inp["cot"]]
    got = _color_grads(model, _color_fwd(model, inp), cot)
    sub = {k: (v[rows] if isinstance(v, np.ndarray) and v.ndim and v.shape[0] == n else v) for k, v in fwd.items()}
    want = ref.color_backward(sub, *(c.numpy()[rows] for c in inp["cot"]))
    _compare_grads(got, want, TILE_REL, f"color_bwd tile {which}={tile}")


@pytest.mark.parametrize("which", ["first", "second", "third", "last"])
def test_sdf_backward_one_tile(which):
    model, inp, ref, _ = _case(PRODUCTION)
    n = inp["x"].shape[0]
    tile = _tiles_to_check("sdf_bwd", n)[which]
    rows = np.arange(tile * TILE, min(n, (tile + 1) * TILE))
    c = torch.zeros(n)
    c[rows] = inp["cot"][0][rows]
    got = _sdf_bwd_direct(model, inp["x"].cuda(), c.cuda(), None)
    want = ref.sdf_backward(inp["x"].numpy()[rows], c.numpy()[rows])
    _compare_grads(got, want, TILE_REL, f"sdf_bwd tile {which}={tile}")

