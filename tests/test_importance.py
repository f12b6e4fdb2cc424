"""Error-map importance sampling (neuralsim_b200/importance.py) against the reference's own ErrorMap / ImpSampler, executed on the CPU
(tests/golden/ref_errmap.npz, made by tests/golden/make_golden_errmap.py with recorded draws): the package's torch restatement of the
update, the cdf construction and the batch draw bit for bit; the host schedule per camera; the state-dict keys; the refusals.  No GPU."""
import os

import numpy as np
import pytest
import torch

from neuralsim_b200 import importance as I

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_errmap.npz"))


def _eq(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a, b), f"{what}: not bit-equal, max |diff| {np.abs(a.astype(np.float64) - b).max():.3e}"


@pytest.fixture
def deterministic():
    """CPU index_put_ splits a large batch over threads unless deterministic algorithms are on (then the last ray of a cell writes)"""
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was)


@pytest.mark.parametrize("k", range(3))
def test_update_equals_reference(k, deterministic):
    n_images, ry, rx, nb = (int(v) for v in GOLD[f"update{k}.meta"])
    em = torch.zeros(n_images, ry, rx)
    for b in range(nb):
        p = f"update{k}.b{b}."
        I.recipe_update_error_map(em, torch.from_numpy(GOLD[p + "fidx"]), torch.from_numpy(GOLD[p + "xy"]), torch.from_numpy(GOLD[p + "val"]))
        _eq(em.numpy(), GOLD[p + "error_map"], p)


def test_update_batches_collide():
    """the cases hold cells hit by several rays in one corner statement (the last-writer rule is exercised)"""
    for k in range(3):
        n_images, ry, rx, _ = (int(v) for v in GOLD[f"update{k}.meta"])
        xy, fi = GOLD[f"update{k}.b0.xy"], GOLD[f"update{k}.b0.fidx"]
        w = np.clip((xy[:, 0] * np.float32(rx)).astype(np.int64), 0, rx - 2)
        h = np.clip((xy[:, 1] * np.float32(ry)).astype(np.int64), 0, ry - 2)
        cells = (fi * ry + h) * rx + w
        assert len(np.unique(cells)) < len(cells) // 2


@pytest.mark.parametrize("k", range(4))
def test_construct_cdf_equals_reference(k):
    n_images, ry, rx, mp = (int(v) for v in GOLD[f"cdf{k}.meta"])
    m = I.ErrorMap(n_images, (ry, rx), max_pdf=None if mp < 0 else 1.0, device="cpu")
    m.error_map.copy_(torch.from_numpy(GOLD[f"cdf{k}.error_map_in"]))
    ptrs = [t.data_ptr() for t in (m.cdf_x_cond_y, m.cdf_y, m.cdf_img)]
    m.construct_cdf()
    assert [t.data_ptr() for t in (m.cdf_x_cond_y, m.cdf_y, m.cdf_img)] == ptrs          # rebuilt in place
    for name in ("cdf_x_cond_y", "cdf_y", "cdf_img"):
        _eq(getattr(m, name).numpy(), GOLD[f"cdf{k}.{name}"], f"cdf{k}.{name}")
    _eq(m.error_map.numpy(), GOLD[f"cdf{k}.error_map_out"], f"cdf{k}.error_map")


class _Replay:
    def __init__(self, draws):
        self.draws = list(draws)

    def rand(self, *size, dtype=None, device=None, generator=None, **kw):
        v = self.draws.pop(0)
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple)) else tuple(size)
        assert v.dtype == np.float32 and v.shape == shape
        return torch.from_numpy(v.copy())

    def randint(self, high, size, dtype=None, device=None, generator=None, **kw):
        v = self.draws.pop(0)
        assert v.dtype == np.int64 and v.shape == tuple(size) and v.max() < high
        return torch.from_numpy(v.copy())


@pytest.mark.parametrize("k", range(5))
def test_sample_img_pixel_recipe_equals_reference(k, monkeypatch):
    n_images, ry, rx, n, nd = (int(v) for v in GOLD[f"sample{k}.meta"])
    frac = float(GOLD[f"sample{k}.frac"])
    r = _Replay(GOLD[f"sample{k}.draw{j}"] for j in range(nd))
    monkeypatch.setattr(torch, "rand", r.rand)
    monkeypatch.setattr(torch, "randint", r.randint)
    cdfs = tuple(torch.from_numpy(GOLD[f"sample{k}.{c}"]) for c in ("cdf_x_cond_y", "cdf_y", "cdf_img"))
    i, xy = I.recipe_sample_img_pixel(cdfs, n_images, n, frac)
    assert not r.draws
    _eq(i.numpy(), GOLD[f"sample{k}.i"], "i")
    _eq(xy.numpy(), GOLD[f"sample{k}.xy"], "xy")
    n_u, n_e = I.split(n, frac)
    assert n_u == int(n * frac) and n_u + n_e == n


def test_sample_cases_cover_edges():
    fracs = {float(GOLD[f"sample{k}.frac"]) for k in range(5)}
    assert fracs == {0.0, 0.5, 1.0}
    assert any(int(GOLD[f"sample{k}.meta"][3]) % 2 for k in range(5))
    xy = np.concatenate([GOLD[f"sample{k}.xy"] for k in range(5)])
    assert xy.min() > 0 and xy.max() < 1
    assert any(np.float32(1e-6) in GOLD[f"sample{k}.xy"] for k in range(5))           # a clamped uniform draw reaches the output


def test_schedule_equals_reference():
    m = I.ErrorMap(2, (4, 8), n_steps_max=500, device="cpu")
    rebuilt = []
    for it in range(2000):
        before = m.n_steps_between_update
        if m.count_step():
            rebuilt.append((it, before))
    _eq(np.array(rebuilt, np.int64), GOLD["sched.rebuilt"], "rebuild steps")
    assert [m.n_steps_since_update, m.n_steps_between_update] == GOLD["sched.state"].tolist()
    assert [b for _, b in rebuilt][:4] == [128, 192, 288, 432] and rebuilt[-1][1] == 500


def test_schedule_is_per_camera():
    """each camera counts the steps it was drawn in: two maps stepped alternately rebuild at their own 128th step"""
    a, b = I.ErrorMap(2, (4, 8), device="cpu"), I.ErrorMap(3, (4, 8), device="cpu")
    hits = {"a": [], "b": []}
    for it in range(300):
        m, name = (a, "a") if it % 3 else (b, "b")
        if m.count_step():
            hits[name].append(it)
    assert hits["a"] == [[i for i in range(300) if i % 3][127]] and hits["b"] == []


def test_state_dict_keys():
    m = I.ErrorMap(3, (4, 8), device="cpu")
    assert sorted(m.state_dict().keys()) == GOLD["state.keys"].tolist() == ["error_map"]
    sd = {"error_map": torch.rand(3, 4, 8)}
    m.load_state_dict(sd)
    assert torch.equal(m.error_map, sd["error_map"])
    s = I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=0.5)
    assert sorted(s.state_dict().keys()) == ["error_maps.rgb.error_map"]


def test_refusals():
    base = dict(error_map_hw=[32, 64], frac_uniform=0.5, frac_mask_err=0, n_steps_max=500)
    I.check_error_map_cfg(base, joint=True)
    for bad, match in ((dict(frac_mask_err=0.1), "frac_mask_err"), (dict(frac_on_classnames=0.2, on_classnames=["Vehicle"]), "focus_on"),
                       (dict(enable_after=100), "enable_after")):
        with pytest.raises(RuntimeError, match=match):
            I.check_error_map_cfg({**base, **bad})
    with pytest.raises(RuntimeError, match="non-joint"):
        I.check_error_map_cfg(base, joint=False)
    m, m2 = I.ErrorMap(2, (4, 8), device="cpu"), I.ErrorMap(2, (4, 8), device="cpu")
    with pytest.raises(RuntimeError, match="exactly one error map"):
        I.ImpSampler({"rgb": (m, 0.5), "mask": (m2, 0.1)})
    with pytest.raises(RuntimeError, match="frac_uniform"):
        I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=1.5)
    for args, match in (((0, (4, 8)), "n_images"), ((2, (1, 8)), "error_map_hw"), ((2, (4, 8, 2)), "error_map_hw")):
        with pytest.raises(RuntimeError, match=match):
            I.ErrorMap(*args, device="cpu")
    with pytest.raises(RuntimeError, match="dtype"):
        I.ErrorMap(2, (4, 8), dtype=torch.float64, device="cpu")
    with pytest.raises(RuntimeError, match="xy"):
        m.update_error_map(0, torch.rand(5, 3), torch.rand(5))
    with pytest.raises(RuntimeError, match="val"):
        m.update_error_map(0, torch.rand(5, 2), torch.rand(4))
    with pytest.raises(RuntimeError, match="out of"):
        m.update_error_map(torch.tensor([0, 2]), torch.rand(2, 2), torch.rand(2))
    with pytest.raises(RuntimeError, match="negative"):
        m.update_error_map(0, torch.rand(2, 2), torch.tensor([0.5, -1.0]))
    with pytest.raises(RuntimeError, match="construct_cdf"):
        I.ErrorMap(2, (4, 8), device="cpu").sample_img(4)


def test_offsets_of_a_draw():
    """the generator offsets a batch advances: the four draws' increments, torch's policy (torch_rng.py:uniform_inc)"""
    from neuralsim_b200.torch_rng import uniform_inc
    cap = 132 * 8
    for n, f in ((8192, 0.5), (4097, 0.5), (7, 0.0), (7, 1.0), (1, 0.5)):
        n_u, n_e = I.split(n, f)
        assert I.sampler_inc(n, f, cap) == uniform_inc(n_u, cap) + uniform_inc(2 * n_u, cap) + uniform_inc(n_e, cap) + uniform_inc(2 * n_e, cap)
    assert I.sampler_inc(8192, 0.5, cap) == 4 * 4                     # four draws below one grid's worth of values: 4 offsets each
