"""CPU: the occupancy grid's update from the network as a graph replay (fields/occ_update.py) -- the sampler it restates pinned to the
reference's own sample_pts_in_voxels, executed (tests/golden/ref_occ_sample.npz), the generator reservation against every draw sequence the
host-sized update can make (tests/torch_uniform.py's launch policy), the host-side schedule, and the refusals."""
import functools
import os

import numpy as np
import pytest
import torch

import torch_uniform as TU
from neuralsim_b200.fields import LoTDNeuSModel
from neuralsim_b200.fields import occ_update as U
from neuralsim_b200.fields.accel import OccGridEma, OccGridEmaBatched, sample_pts_in_voxels

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_occ_sample.npz")


def _gold():
    z = np.load(GOLD)
    n = len({k.split(".")[0] for k in z.files if k.startswith("case")})
    return z["res"], [{k.split(".", 1)[1]: z[k] for k in z.files if k.startswith(f"case{i}.")} for i in range(n)]


def test_golden_cases_cover_both_branches_and_their_edge():
    _, cs = _gold()
    nv_n = [(len(c["gidx"]), int(c["num_pts"])) for c in cs]
    assert (1, 1) in nv_n and (1, 2) in nv_n                           # one voxel, on both sides of the branch
    assert any(n == 2 * nv and nv > 1 for nv, n in nv_n)                # the n_per_vox branch at its edge
    assert any(n == 2 * nv - 1 and nv > 1 for nv, n in nv_n)            # the randint branch at its edge
    assert any(nv > n for nv, n in nv_n)


@pytest.mark.parametrize("case", range(9))
def test_sampler_matches_executed_reference(case):
    res, cs = _gold()
    c = cs[case]
    gen = torch.Generator().manual_seed(int(c["seed"]))
    pts, vidx = sample_pts_in_voxels(torch.from_numpy(c["gidx"]), int(c["num_pts"]), torch.from_numpy(res), torch.float, gen)
    assert pts.dtype == torch.float32 and np.array_equal(pts.numpy(), c["pts"])
    assert np.array_equal(vidx.numpy(), c["vidx"])


# ------------------------------------------------------------------------------------------------------------ the generator reservation
H100 = (132, 2048)           # SMs, threads per SM: torch's grid cap of a draw is SMs * (threads / 256)


@functools.lru_cache(maxsize=None)
def _inc(numel, sms, tps):
    return 0 if numel <= 0 else TU.calc_execution_policy(numel, sms, tps)[0]


def _part(n, nv, dev):
    """the offsets sample_pts_in_voxels(gidx of nv voxels, n) advances the generator by, and the points it returns"""
    if n < 2 * nv:
        return _inc(n, *dev) + _inc(3 * n, *dev), n
    per = n // nv + 1
    return _inc(3 * nv * per, *dev), nv * per


def _host_update(cells, n_occ, num_steps, num_pts, warmup, dev):
    """(offsets, points) of OccGridEma.step's host-sized update on a grid with n_occ occupied cells"""
    if warmup:
        parts = [_part(num_pts, cells, dev)]
    else:
        n_empty = cells - n_occ
        parts = [_part(num_pts // 2, cells, dev)] + ([_part(num_pts // 4, n_empty, dev)] if n_empty > 0 else []) + [_part(num_pts // 4, n_occ, dev)]
    return num_steps * sum(p[0] for p in parts), num_steps * sum(p[1] for p in parts)


GRIDS = {"64^3": (64, 64, 64), "cfg3": (40, 150, 15), "8^3": (8, 8, 8)}


@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("num_steps,num_pts", [(4, 2 ** 20), (2, 2 ** 15), (3, 1001)])
@pytest.mark.parametrize("dev", [H100, (16, 1536)], ids=["h100", "small"])
def test_reservation_and_capacity_bound_every_draw_sequence(grid, num_steps, num_pts, dev):
    cells = int(np.prod(GRIDS[grid]))
    cap = dev[0] * (dev[1] // 256)
    reserve, arena = U.reservation(cells, num_steps, num_pts, cap), U.capacity(cells, num_steps, num_pts)
    worst_off, worst_pts = _host_update(cells, 0, num_steps, num_pts, True, dev)            # the warm-up phase
    for n_occ in range(1, cells + 1):                                                         # n_occ = cells: the empty list is skipped
        off, pts = _host_update(cells, n_occ, num_steps, num_pts, False, dev)
        worst_off, worst_pts = max(worst_off, off), max(worst_pts, pts)
    assert worst_off <= reserve and worst_pts <= arena
    assert arena <= int(1.5 * num_steps * num_pts) + 3 * num_steps


def test_reservation_refuses_draws_torch_would_split():
    with pytest.raises(RuntimeError, match="2\\^31"):
        U.reservation(64 ** 3, 4, 2 ** 30, 1056)


# ------------------------------------------------------------------------------------------------------------ the host-side schedule
class _Gen:
    def __init__(self):
        self.off = 40

    def initial_seed(self):
        return 7

    def get_offset(self):
        return self.off

    def set_offset(self, v):
        self.off = v


class _Graph:
    def __init__(self):
        self.replays = []

    def replay(self):
        self.replays.append(None)


def _stub_update():
    """an OccGridUpdate around a CPU grid, with a stand-in graph: the host logic of step() without a device"""
    class _Model:
        max_level = None

        def query_sdf(self, x):
            return x

        class implicit_surface:
            @staticmethod
            def _ml(ml):
                return 5
    occ = OccGridEma(resolution=[4, 4, 4], update_from_samples_cfg=None)
    u = object.__new__(U.OccGridUpdate)
    u.model, u.occ, u.gen, u.graph, u.reservation = _Model(), occ, _Gen(), _Graph(), 11
    u.warmup, u.max_level, u.rng = torch.zeros((), dtype=torch.int32), torch.zeros((), dtype=torch.int32), torch.zeros(2, dtype=torch.int64)
    u._captured = [t.data_ptr() if t is not None else None for t in u._targets()]
    occ.net_update = u
    return u, occ


def test_schedule_replays_on_update_iterations_only():
    u, occ = _stub_update()
    phases = []
    for it in range(0, 300):
        before = len(u.graph.replays)
        updated = occ.step(it, u.model.query_sdf)
        assert updated == (len(u.graph.replays) == before + 1)
        if updated:
            phases.append((it, int(u.warmup), int(u.max_level), u.rng.tolist()))
    assert [p[0] for p in phases] == list(range(16, 300, 16))                  # not at 0, not off the multiples of 16
    assert all(w == (1 if it < 256 else 0) for it, w, _, _ in phases)
    assert all(ml == 5 for _, _, ml, _ in phases)
    assert [p[3] for p in phases] == [[7, 40 + 11 * k] for k in range(len(phases))]      # (seed, offset) of each update, then the reservation
    assert u.gen.off == 40 + 11 * len(phases)


def test_step_refuses_another_query_and_a_generator():
    u, occ = _stub_update()
    with pytest.raises(RuntimeError, match="query_sdf"):
        occ.step(16, lambda x: x)
    with pytest.raises(RuntimeError, match="generator"):
        occ.step(16, u.model.query_sdf, generator=torch.Generator())
    assert u.graph.replays == []


def test_a_reassigned_grid_is_captured_again():
    u, occ = _stub_update()
    occ.occ_val_grid = occ.occ_val_grid.clone()
    captured = []
    u.capture = lambda: (captured.append(1), setattr(u, "graph", _Graph()), setattr(u, "_captured", [t.data_ptr() if t is not None else None
                                                                                                      for t in u._targets()]))
    assert occ.step(16, u.model.query_sdf) and captured == [1] and len(u.graph.replays) == 1
    assert occ.step(32, u.model.query_sdf) and captured == [1] and len(u.graph.replays) == 2


# ------------------------------------------------------------------------------------------------------------ refusals
def test_refuses_batched_grids():
    class _M:
        class accel:
            occ = OccGridEmaBatched(2, resolution=[4, 4, 4], update_from_samples_cfg=None)
    with pytest.raises(RuntimeError, match="OccGridEmaBatched"):
        U.OccGridUpdate(_M())


def test_refuses_a_model_without_a_single_grid():
    class _M:
        accel = None
    with pytest.raises(RuntimeError, match="no single occupancy grid"):
        U.OccGridUpdate(_M())


def test_refuses_an_sdf_off_the_fused_kernels():
    torch.manual_seed(0)
    m = LoTDNeuSModel(surface_cfg=dict(bounding_size=2.0), radiance_cfg=False, accel_cfg=dict(resolution=[8, 8, 8], update_from_samples_cfg=None))
    assert not m.implicit_surface._fusable()
    with pytest.raises(RuntimeError, match="fused kernels"):
        U.OccGridUpdate(m)
    assert m.accel.occ.net_update is None


def test_refuses_other_occupancy_values():
    with pytest.raises(RuntimeError, match="'sdf'"):
        OccGridEma(resolution=[4, 4, 4], occ_val_fn_cfg=dict(type="raw"))
