"""The colour forward's one table gather (csrc/color_tc.cu: gather_row_and_jacobian) at the sizes and levels where it can go wrong.

k_color_fwd loads each level's 8 corners once and takes from them both the fp16 feature pair of the X tile and the level's Jacobian, which
stays in registers across the Z MMA, the decoder epilogue and the g MMA.  Both instantiations (<true>: the colour query; <false>: the
geometry-only query, selected by rgb == NULL) run the same gather.  For 1, 127, 128 and 129 points, a size at which every persistent CTA
loops over tiles, and a device count below the capacity; with every level and with max_level 5 and 13 (levels skipped in the middle of a
group of four gathered levels); on the table geometry of the cfg2 model (cubic, hashed and dense levels) and of the cfg3 street model
(cuboid levels, a different nablas scale per axis):
  - sdf and nablas against the float64 reference (oracle/fused64.py) with the bounds of tests/test_tc_kernels_gpu.py;
  - <true> and <false> bit for bit on sdf, nablas, x, the Z tile and the h half of the X tile."""
import numpy as np
import pytest
import torch

import test_tc_geometry_gpu as tg
import test_tc_kernels_gpu as tk
from oracle import fused64
from test_geometry_only_gpu import GEO_CTAS_PER_SM, _launch

pytestmark = pytest.mark.gpu

GEOMETRIES = ("cfg2", "cfg3")
MAX_LEVELS = (None, 5, 13)
SIZES = (1, 127, 128, 129, "loop")
BIT_KEYS = ("sdf", "nablas", "x", "Z", "Xh")


def _loop_size():
    """every CTA of both instantiations' grids (2 CTAs per SM) runs at least two tiles, and the last tile is partial"""
    assert GEO_CTAS_PER_SM == tk.CTAS_PER_SM["color_fwd"]
    return tk._size("color_fwd", 2)


def _twin(col, surface_cfg):
    """a geometry-only LoTDNeuS with the colour model's table geometry, table and decoder"""
    from neuralsim_b200.fields.neus import LoTDNeuS
    geo = LoTDNeuS(surface_cfg=surface_cfg, radiance_cfg=False, device="cuda")
    geo.implicit_surface.load_state_dict(col.implicit_surface.state_dict())
    assert geo.radiance_net is None and geo._geometry_fusable()
    return geo


_CACHE = {}


def _models(geometry):
    """the colour model, its geometry-only twin and the loop-size inputs of one table geometry"""
    if geometry not in _CACHE:
        from oracle import lotd as olotd
        if geometry == "cfg2":            # gen_ngp_cfg() is bench.py's table: 16 levels, dense up to 80^3 cells, then hashed into 2^19
            col = tk._model(64, 64, 4, seed=71)
            surface_cfg = dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg()), decoder_cfg=dict(W=64))
        else:
            cfg = tg._cfg()
            col = tg._model(cfg, seed=73)
            surface_cfg = dict(aabb=tg.AABB, sdf_scale=tg.SDF_SCALE, encoding_cfg=dict(lotd_cfg=cfg))
        types = {t.lower() for t in olotd.LoDMeta(3, **surface_cfg["encoding_cfg"]["lotd_cfg"]).level_types_str}
        assert {"dense", "hash"} <= types, types
        _CACHE[geometry] = dict(col=col, geo=_twin(col, surface_cfg), inp=tk._inputs(_loop_size(), 4, seed=79), ref={})
    return _CACHE[geometry]


def _reference(c, max_level):
    """float64 sdf, nablas and their scales of all loop-size inputs (the smaller sizes take their first rows)"""
    if max_level not in c["ref"]:
        ref = fused64.Fused64.from_model(c["col"], max_level=max_level)
        inp = c["inp"]
        c["ref"][max_level] = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy())
    return c["ref"][max_level]


def _first(inp, n):
    return {k: (v[:n] if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}


def _check_against_float64(got, fwd, n, what):
    sdf = tk._fp16_metrics(got["sdf"].cpu().numpy()[:n], fwd["sdf"][:n], fwd["sdf_scale"][:n])
    nab = np.abs(got["nablas"].cpu().numpy()[:n] - fwd["nablas"][:n]) / (fwd["nablas_scale"][:n] + 1e-30)
    print(f"METRIC one_gather {what} sdf: flips={sdf[0]:.2e} max_ulp={sdf[1]:.2f} nablas: max_rel={nab.max():.2e} "
          f"frac>1e-5={(nab > 1e-5).mean():.2e}")
    assert sdf[1] <= tk.SDF_MAX_ULP and float(nab.max()) <= tk.NAB_MAX_REL, (what, sdf, float(nab.max()))
    if n >= 1024:                          # the fractions are statistics of a population: single points are held to the per-element bounds
        assert sdf[0] <= tk.SDF_FLIP_FRAC and float((nab > 1e-5).mean()) <= tk.NAB_FRAC_1E5, (what, sdf, float((nab > 1e-5).mean()))


def _check_twins(a, b, what, live=None):
    for k in BIT_KEYS:
        if live is not None and k in ("sdf", "nablas", "x"):
            assert torch.equal(a[k][:live], b[k][:live]), (what, k)
        else:
            assert torch.equal(a[k], b[k]), (what, k)


@pytest.mark.parametrize("max_level", MAX_LEVELS, ids=lambda m: f"ml{m}")
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("geometry", GEOMETRIES)
def test_one_gather_forward(geometry, n, max_level):
    c = _models(geometry)
    if n == "loop":
        n = _loop_size()
        n_tiles = -(-n // tk.TILE)
        assert n % tk.TILE and n_tiles // min(n_tiles, tk._sms() * GEO_CTAS_PER_SM) >= 2
    inp = _first(c["inp"], n)
    a = _launch(c["col"], inp, True, max_level=max_level)
    b = _launch(c["geo"], inp, False, max_level=max_level)
    what = f"{geometry} n={n} ml={max_level}"
    _check_twins(a, b, what)
    assert bool(torch.isfinite(a["sdf"]).all()) and bool(torch.isfinite(a["nablas"]).all()), what
    _check_against_float64(a, _reference(c, max_level), n, what)


@pytest.mark.parametrize("max_level", (None, 5), ids=lambda m: f"ml{m}")
@pytest.mark.parametrize("geometry", GEOMETRIES)
def test_one_gather_device_count_below_capacity(geometry, max_level):
    c = _models(geometry)
    n = _loop_size()
    live = n - tk._sms() * tk.TILE - 37              # a partial last tile; on the capacity's grid some CTAs run two tiles and some one
    assert live % tk.TILE and -(-live // tk.TILE) > tk._sms() * GEO_CTAS_PER_SM
    a = _launch(c["col"], c["inp"], True, max_level=max_level, count=live)
    b = _launch(c["geo"], c["inp"], False, max_level=max_level, count=live)
    what = f"{geometry} live={live}/{n} ml={max_level}"
    _check_twins(a, b, what, live=live)
    for k in ("sdf", "nablas", "x"):
        assert bool(torch.isnan(a[k][live:]).all()) and bool(torch.isnan(b[k][live:]).all()), (what, k)   # nothing written past the count
    _check_against_float64(a, _reference(c, max_level), live, what)
