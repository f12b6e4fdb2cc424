"""The hard-mask LoTD level schedule (LoTDEncoding's `anneal_cfg`, fields/encoding.py:MultiresAnnealer) against the reference's own
MultiresAnnealer (tests/golden/ref_anneal.npz, made by tests/golden/make_golden_anneal.py from multires_annealer.py), the training hooks that
apply it, the shipped StreetSurf encoding configurations, and the refusals.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from neuralsim_b200.fields import LoTDNeuSModel
from neuralsim_b200.fields.encoding import LoTDEncoding, MultiresAnnealer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_anneal.npz")


def _cases():
    z = np.load(GOLDEN)
    n = len([k for k in z.files if k.endswith(".cfg")])
    return [(z[f"case{k}.cfg"].tolist(), z[f"case{k}.max_level"].astype(np.int64), int(z[f"case{k}.stop_state"])) for k in range(n)]


def _encoding(levels, anneal_cfg):
    cfg = dict(lod_res=[4 + l for l in range(levels)], lod_n_feats=[2] * levels, lod_types=["Dense"] * levels)
    return LoTDEncoding(3, lotd_cfg=cfg, anneal_cfg=anneal_cfg)


def test_schedule_equals_the_reference_annealer():
    cases = _cases()
    assert {c[0][0] for c in cases} == {12, 16, 17} and {c[0][2] for c in cases} == {1, 7}
    assert {c[0][1] for c in cases} >= {-3, -1, 0, 2, 11, 15, 16, 14, 18, 19}
    for (L, sl, ue, s0, s1), want, stop in cases:
        its = np.arange(s0 - 20, s1 + 21)
        an = MultiresAnnealer([2] * L, "hardmask", stop_it=s1, start_it=s0, update_every=ue, start_level=sl)
        got = np.array([an(int(i))[0] for i in its])
        assert np.array_equal(got, want), (L, sl, ue, s0, s1, np.flatnonzero(got != want)[:5])
        assert an()[0] == stop == L - 1 and an(s0 + 3)[1] is None
        assert int(want[0]) == max(min(sl, L - 1), -1)                # before start_it: the clamped start level
        assert np.unique(np.diff(want)).tolist() in ([0], [0, 1], [1])  # one level at a time
    # through the encoding, on a 16-level table
    (L, sl, ue, s0, s1), want, _ = next(c for c in cases if c[0] == [16, 2, 1, 0, 4000])
    enc = _encoding(16, dict(type="hardmask", start_it=0, start_level=2, stop_it=4000))
    for it in (-1, 0, 307, 308, 615, 616, 3999, 4000, 4020):
        enc.set_anneal_iter(it)
        assert enc.max_level == want[it + 20] and enc.window is None, it
    enc.set_anneal_iter(307)
    assert enc.max_level == 2
    enc.set_anneal_iter(308)
    assert enc.max_level == 3


def test_stop_state_before_the_first_iteration():
    enc = _encoding(12, dict(type="hardmask", start_it=0, start_level=2, stop_it=3000))
    assert enc.max_level is None and enc.annealer.it == 3000 and enc.annealer()[0] == 11
    assert _encoding(12, None).annealer is None


def test_refusals():
    with pytest.raises(RuntimeError, match="cosine"):
        _encoding(12, dict(type="cosine", start_it=0, start_level=2, stop_it=3000))
    with pytest.raises(RuntimeError, match="anneal_type"):
        _encoding(12, dict(type="linear", start_it=0, stop_it=3000))
    with pytest.raises(RuntimeError, match="stop_it"):
        _encoding(12, dict(type="hardmask", start_it=500, stop_it=500))
    with pytest.raises(RuntimeError, match="stop_it"):
        _encoding(12, dict(type="hardmask", start_it=0, stop_it=5, update_every=7))


def _street(anneal_cfg, stop_it=4000):
    """the shipped StreetSurf surface configuration (withmask_withlidar_withnormal and the other annealed colour configs), with a small
    hash table: lotd_use_cuboid, the `ngp` auto config, and the hard-mask schedule from level 2"""
    enc = dict(lotd_use_cuboid=True, lotd_auto_compute_cfg=dict(type="ngp", target_num_params=18 * 2 ** 14, min_res=16, n_feats=2,
                                                                log2_hashmap_size=14, max_num_levels=None),
               param_init_cfg=dict(type="uniform_to_type", bound=1.0e-4))
    if anneal_cfg:
        enc["anneal_cfg"] = dict(type="hardmask", start_it=0, start_level=2, stop_it=stop_it)
    torch.manual_seed(0)
    return LoTDNeuSModel(surface_cfg=dict(aabb=[[-20., -75., -7.5], [20., 75., 7.5]], encoding_cfg=enc,
                                          decoder_cfg=dict(type="mlp", D=1, W=64, activation=dict(type="softplus", beta=100.0))),
                         radiance_cfg=dict(n_appear_embedding=4, D=2, W=64), var_ctrl_cfg=dict(ln_inv_s_init=0.3),
                         accel_cfg=dict(resolution=[8, 8, 8], update_from_samples_cfg=None))


@pytest.mark.parametrize("stop_it", [3000, 4000])
def test_shipped_encoding_cfg_constructs_and_anneals(stop_it):
    m = _street(True, stop_it).eval()                 # eval: no occupancy update (it queries the field on the GPU)
    enc = m.implicit_surface.encoding
    L = enc.meta.n_levels
    assert enc.annealer is not None and enc.max_level is None and m.max_level is None
    m.training_before_per_step(0)
    assert enc.max_level == 2 and m.implicit_surface._ml(m.max_level) == 2
    m.training_before_per_step(stop_it)
    assert enc.max_level == L - 1


def test_state_dict_keys_unchanged():
    a, b = _street(True).state_dict(), _street(False).state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape for k in a)


def test_level_resolution_keeps_the_reference_quirk():
    """`max_level or encoding.max_level` (lotd_encoding.py:162): an explicit 0 falls through to the encoding's level"""
    m = _street(True)
    s = m.implicit_surface
    s.encoding.max_level = 5
    assert s._ml(None) == 5 and s._ml(0) == 5 and s._ml(3) == 3 and s._ml(-1) == -1
    s.encoding.max_level = None
    assert s._ml(None) == s.encoding.meta.n_levels and s._ml(0) == s.encoding.meta.n_levels


def test_training_hook_anneals_before_the_accel_step(monkeypatch):
    """LoTDNeuSModel.training_before_per_step: the variance schedule, then the level schedule, then the occupancy update, which queries
    the field at the new level (lotd_neus.py:116-121, renderer_mixin.py:176-182)"""
    m = _street(True).train()
    seen = []
    monkeypatch.setattr(m.accel, "step", lambda it, query, logger=None: seen.append((it, m.implicit_surface.encoding.max_level, m.ctrl_var.it)))
    m.training_before_per_step(308)
    assert seen == [(308, 2 + int(308 / 4000 * (m.implicit_surface.encoding.meta.n_levels - 3)), 308)] and m.it == 308
