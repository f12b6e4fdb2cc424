"""The three backward wgmma kernels at their persistent grids, against the float64 reference of their numerics contract
(oracle/fused64.py): k_color_rad_bwd and k_color_sdf_bwd at kColorBwdCtasPerSM = 2 CTAs per SM (csrc/color_tc.cu), k_sdf_bwd_tc at
kSdfBwdCtasPerSM = 4 (csrc/fused_tc.cu).

These kernels keep their weight-gradient sums in wgmma register fragments across all tiles of a persistent CTA, run the element-wise
epilogues on the fragments and stage only what the table scatter needs.  The sizes make every CTA of these grids loop over at least
three tiles with a partial last tile; the one-tile checks put the cotangent on a tile of a CTA's first, second and third iteration
(the latter two were prefetched while the CTA finished the tile before, and their sums add to registers that already hold the earlier
tiles' zeros) and on the partial last tile.  Bounds are those of test_tc_kernels_gpu.py (BWD_REL, TILE_REL)."""
import numpy as np
import pytest
import torch

import test_tc_kernels_gpu as tk
from oracle import fused64

pytestmark = pytest.mark.gpu

TILE = tk.TILE
CTAS_PER_SM = dict(color_bwd=2, sdf_bwd=4)
# the production configuration, a narrow decoder with a level cap, and a narrow radiance net without appearance channels
CASES = [tk.PRODUCTION, ((16, 64, 1), 7), ((48, 40, 0), None)]
CASE_IDS = [f"w{c[0]}-r{c[1]}-a{c[2]}-ml{m}" for c, m in CASES]


def _grid(kernel, n):
    return min(-(-n // TILE), tk._sms() * CTAS_PER_SM[kernel])


def _size(kernel, iters):
    """the smallest n at which every CTA of `kernel` runs at least `iters` tiles, with a partial last tile"""
    return (iters * tk._sms() * CTAS_PER_SM[kernel] + 1) * TILE - 51


def _assert_multi_tile(kernel, n, iters):
    n_tiles = -(-n // TILE)
    assert n % TILE != 0 and n_tiles // _grid(kernel, n) >= iters, (kernel, n, n_tiles, _grid(kernel, n))


def _tiles_to_check(kernel, n):
    g = _grid(kernel, n)
    return dict(first=0, second=g + 1, third=2 * g + 2, last=-(-n // TILE) - 1)


_CACHE = {}


def _setup(case, kernel):
    """model, inputs and float64 reference at the size `kernel` needs (one entry kept at a time)"""
    key = (case, kernel)
    if key not in _CACHE:
        _CACHE.clear()
        (width, rw, n_appear), max_level = case
        model = tk._model(width, rw, n_appear, seed=width + 3 * rw + n_appear)
        model.max_level = max_level
        inp = tk._inputs(_size(kernel, 3), n_appear, seed=n_appear + 11)
        ref = fused64.Fused64.from_model(model, max_level=max_level)
        fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy()) if kernel == "color_bwd" else None
        _CACHE[key] = (model, inp, ref, fwd)
    return _CACHE[key]


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_color_backward_full_new_grid(case):
    model, inp, ref, fwd = _setup(case, "color_bwd")
    _assert_multi_tile("color_bwd", inp["x"].shape[0], 3)
    got = tk._color_grads(model, tk._color_fwd(model, inp), inp["cot"])
    want = ref.color_backward(fwd, *(c.numpy() for c in inp["cot"]))
    tk._compare_grads(got, want, tk.BWD_REL, f"color_bwd(2/SM) {case}")


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_sdf_backward_full_new_grid(case):
    model, inp, ref, _ = _setup(case, "sdf_bwd")
    n = inp["x"].shape[0]
    _assert_multi_tile("sdf_bwd", n, 3)
    # db2 = sum of the cotangent.  Over these ~200k random-sign values it cancels to ~1e-4 of sum |d| (the fp32 sum is then only good
    # to ~1e-5 relative, whatever the kernel); an offset keeps db2 a sum that measures the kernel, not the cancellation.
    cot = inp["cot"][0] + 0.25
    x, c = inp["x"].cuda(), cot.cuda()
    p = tk._params(model)
    keys = ("grid", "W1", "b1", "W2", "b2")
    sdf = model.implicit_surface.fused_sdf_autograd(x, max_level=case[1])
    got = dict(zip(keys, torch.autograd.grad((sdf * c).sum(), [p[k] for k in keys])))
    tk._compare_grads(got, ref.sdf_backward(inp["x"].numpy(), cot.numpy()), tk.BWD_REL, f"sdf_bwd(4/SM) {case}")


@pytest.mark.parametrize("which", ["first", "second", "third", "last"])
def test_color_backward_one_tile_new_grid(which):
    model, inp, ref, fwd = _setup(tk.PRODUCTION, "color_bwd")
    n = inp["x"].shape[0]
    tile = _tiles_to_check("color_bwd", n)[which]
    rows = np.arange(tile * TILE, min(n, (tile + 1) * TILE))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[rows] = True
    cot = [c * mask.view(-1, *[1] * (c.dim() - 1)) for c in inp["cot"]]
    got = tk._color_grads(model, tk._color_fwd(model, inp), cot)
    sub = {k: (v[rows] if isinstance(v, np.ndarray) and v.ndim and v.shape[0] == n else v) for k, v in fwd.items()}
    want = ref.color_backward(sub, *(c.numpy()[rows] for c in inp["cot"]))
    tk._compare_grads(got, want, tk.TILE_REL, f"color_bwd(2/SM) tile {which}={tile}")


@pytest.mark.parametrize("which", ["first", "second", "third", "last"])
def test_sdf_backward_one_tile_new_grid(which):
    model, inp, ref, _ = _setup(tk.PRODUCTION, "sdf_bwd")
    n = inp["x"].shape[0]
    tile = _tiles_to_check("sdf_bwd", n)[which]
    rows = np.arange(tile * TILE, min(n, (tile + 1) * TILE))
    c = torch.zeros(n)
    c[rows] = inp["cot"][0][rows]
    got = tk._sdf_bwd_direct(model, inp["x"].cuda(), c.cuda(), None)
    want = ref.sdf_backward(inp["x"].numpy()[rows], c.numpy()[rows])
    tk._compare_grads(got, want, tk.TILE_REL, f"sdf_bwd(4/SM) tile {which}={tile}")
