"""The occupancy grid's update from the network as one graph replay (fields/occ_update.py, csrc/occ_update.cu) against the host-sized
OccGridEma.step it replaces, from the same generator state: the voxel lists against nonzero(), the drawn points against
sample_pts_in_voxels on CUDA, one whole update against the host-sized one (grids and collected evidence bit for bit), a StaticFrame training
loop with the update attached against the same loop on the host path, and no synchronisation on an update iteration."""
import copy
import gc
import os
import sys

import pytest
import torch

import bench_cfg3 as C
from neuralsim_b200.fields import OccGridUpdate
from neuralsim_b200.fields import occ_update as U
from neuralsim_b200.fields.accel import OccGridEma, sample_pts_in_voxels
from neuralsim_b200 import torch_rng as TR
from util import rel_l2

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def _street_occ(res=(40, 150, 15)):
    """bench_cfg3's road-plane grid"""
    half_z, zc = 7.5, 0.0
    cz = ((torch.arange(res[2], dtype=torch.float64) + 0.5) / res[2] * 2 - 1) * half_z + zc
    return ((cz - C.ROAD_Z).abs() < 1.0).view(1, 1, -1).expand(*res).contiguous().cuda()


def _grids():
    g = torch.Generator().manual_seed(3)
    single = torch.zeros(8, 8, 8, dtype=torch.bool)
    single[5, 2, 7] = True
    return {"empty": torch.zeros(8, 8, 8, dtype=torch.bool).cuda(), "single": single.cuda(), "full": torch.ones(8, 8, 8, dtype=torch.bool).cuda(),
            "random": (torch.rand(16, 12, 20, generator=g) < 0.3).cuda(), "street": _street_occ()}


def _lists(occ_grid):
    cells, dev = occ_grid.numel(), occ_grid.device
    occupied, empty = torch.full((2, cells), -1, dtype=torch.int64, device=dev).unbind(0)
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    flags, first = torch.zeros(2, cells, dtype=torch.int32, device=dev).unbind(0)
    from neuralsim_b200.graphics.neus_fused import _scan_ws_bytes
    ws = torch.full((_scan_ws_bytes(),), 7, dtype=torch.uint8, device=dev)       # the entry point zeroes its workspace
    U.voxel_lists(occ_grid, occupied, empty, counts, flags, first, ws)
    return occupied, empty, counts


def _unravel(flat, shape):
    return torch.stack([flat // (shape[1] * shape[2]), (flat // shape[2]) % shape[1], flat % shape[2]], -1)


@pytest.mark.parametrize("name", ["empty", "single", "full", "random", "street"])
def test_voxel_lists_equal_nonzero(cuda, name):
    grid = _grids()[name]
    occupied, empty, counts = _lists(grid)
    ref_o, ref_e = grid.nonzero(), grid.logical_not().nonzero()
    assert counts.tolist() == [ref_o.shape[0], ref_e.shape[0]]
    assert torch.equal(_unravel(occupied[:ref_o.shape[0]], grid.shape), ref_o)
    assert torch.equal(_unravel(empty[:ref_e.shape[0]], grid.shape), ref_e)


# ------------------------------------------------------------------------------------------------------------ the draws
def _host_pts(occ, warmup, num_steps, num_pts, gen):
    """the points OccGridEma.step's host-sized update queries, in its order"""
    occupied, empty = occ.occ_grid.nonzero().long(), occ.occ_grid.logical_not().nonzero().long()
    out = []
    for _ in range(num_steps):
        if warmup:
            out.append(sample_pts_in_voxels(occ.gidx_full, num_pts, occ.resolution, torch.float, gen)[0])
            continue
        out.append(sample_pts_in_voxels(occ.gidx_full, num_pts // 2, occ.resolution, torch.float, gen)[0])
        if empty.numel() > 0:
            out.append(sample_pts_in_voxels(empty, num_pts // 4, occ.resolution, torch.float, gen)[0])
        out.append(sample_pts_in_voxels(occupied, num_pts // 4, occ.resolution, torch.float, gen)[0])
    return torch.cat(out, 0)


def _draw(occ, warmup, num_steps, num_pts, seed):
    """(graph-path points, host-path points, offsets the host path used, the reservation) from one generator state"""
    dev = occ.occ_grid.device
    cells = occ.occ_grid.numel()
    gen = torch.Generator(dev).manual_seed(seed)
    gen.set_offset(4 * seed)
    rng = TR.take(gen, 0)
    occupied, empty, counts = _lists(occ.occ_grid)
    cap = U.capacity(cells, num_steps, num_pts)
    pts = torch.full((cap, 3), float("nan"), device=dev)
    out = torch.zeros(2, dtype=torch.int64, device=dev)
    U.draw_pts(rng, torch.tensor(1 if warmup else 0, dtype=torch.int32, device=dev), counts, occupied, empty, occ.occ_grid.shape, num_steps, num_pts, pts, out)
    off0 = gen.get_offset()
    host = _host_pts(occ, warmup, num_steps, num_pts, gen)
    assert int(out[1]) == 0 and int(out[0]) == host.shape[0] <= cap
    return pts[:host.shape[0]], host, gen.get_offset() - off0, U.reservation(cells, num_steps, num_pts, TR.grid_cap(dev))


def _occ_with(res, occupied_cells):
    occ = OccGridEma(resolution=list(res), update_from_samples_cfg=None, device="cuda")
    g = torch.zeros(res, dtype=torch.bool, device="cuda")
    g.view(-1)[occupied_cells] = True
    occ.set_occ_grid(g)
    return occ


DRAW_CASES = {
    # (resolution, occupied flat cells, num_steps, num_pts): what the occupied part (num_pts // 4 points) meets
    "nv1": ((8, 8, 8), [77], 2, 8),                                      # one voxel, n = 2 nv: the n_per_vox branch; empty part: randint
    "n_eq_2nv": ((8, 8, 8), list(range(3, 400, 40)), 1, 80),             # 10 voxels, n = 20
    "n_eq_2nv_minus_1": ((8, 8, 8), list(range(3, 400, 40)), 2, 79),     # 10 voxels, n = 19: randint
    "nv_gt_n": ((8, 8, 8), list(range(0, 512, 2)), 3, 400),              # 256 voxels, n = 100
    "shipped_64": ((64, 64, 64), list(range(5, 262144, 37)), 4, 2 ** 20),
    "street": ((40, 150, 15), None, 2, 2 ** 18),
}


@pytest.mark.parametrize("warmup", [False, True], ids=["steady", "warmup"])
@pytest.mark.parametrize("case", list(DRAW_CASES))
def test_draws_equal_sample_pts_in_voxels(cuda, case, warmup):
    res, cells, num_steps, num_pts = DRAW_CASES[case]
    occ = _occ_with(res, cells) if cells is not None else _occ_with(res, _street_occ(res).view(-1).nonzero()[:, 0].tolist())
    pts, host, used, reserve = _draw(occ, warmup, num_steps, num_pts, seed=len(case))
    assert torch.equal(pts, host)
    assert used <= reserve


def test_draws_without_empty_voxels_and_without_occupied_ones(cuda):
    full = _occ_with((8, 8, 8), list(range(512)))
    pts, host, used, reserve = _draw(full, False, 2, 64, seed=9)                # the empty part is skipped
    assert torch.equal(pts, host) and used <= reserve
    none = _occ_with((8, 8, 8), [])
    occupied, empty, counts = _lists(none.occ_grid)
    out = torch.full((2,), -5, dtype=torch.int64, device=cuda)
    pts = torch.zeros(U.capacity(512, 2, 64), 3, device=cuda)
    U.draw_pts(TR.take(torch.Generator(cuda).manual_seed(1), 0), torch.tensor(0, dtype=torch.int32, device=cuda), counts, occupied, empty, (8, 8, 8),
               2, 64, pts, out)
    assert out.tolist() == [0, 1]


# ------------------------------------------------------------------------------------------------------------ one update
def _cfg_model(collect):
    torch.manual_seed(0)
    return bench.build_model(torch.device("cuda"), collect_samples=collect).train()


def _street_model(levels):
    if levels == 17:
        model = C.build_model(torch.device("cuda"), max_num_levels=17, log2_hashmap_size=16, target_num_params=19 * 2 ** 17).train()
        model.implicit_surface.max_fused_levels = 24
    else:
        model = C.build_model(torch.device("cuda")).train()
    assert model.implicit_surface._fusable()
    return model


def _state(occ):
    return [t.clone() for t in (occ.occ_val_grid, occ.occ_grid) + ((occ._occ_val_grid_pcl,) if occ.should_collect_samples else ())]


def _seed_pcl(occ, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    p = occ._occ_val_grid_pcl
    p.copy_(torch.where(torch.rand(p.shape, device="cuda", generator=g) < 0.05, torch.rand(p.shape, device="cuda", generator=g), 0.))


def _one_update(model, it, pcl_seed=None):
    """(host-sized state after step(it), graph state after step(it)) from the same grids and generator state"""
    occ = model.accel.occ
    occ.update_from_net_cfg = dict(num_steps=2, num_pts=2 ** 18)
    if pcl_seed is not None:
        _seed_pcl(occ, pcl_seed)
    before = _state(occ)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    off = gen.get_offset()
    assert occ.step(it, model.query_sdf)
    host = _state(occ)
    for t, s in zip((occ.occ_val_grid, occ.occ_grid) + ((occ._occ_val_grid_pcl,) if occ.should_collect_samples else ()), before):
        t.copy_(s)
    upd = OccGridUpdate(model)
    gen.set_offset(off)
    assert occ.step(it, model.query_sdf)
    upd.check()
    return host, _state(occ), before


@pytest.mark.parametrize("it,collect", [(16, False), (16, True), (512, False), (512, True)], ids=["warmup", "warmup-pcl", "steady", "steady-pcl"])
def test_one_update_equals_host_sized_cfg(cuda, it, collect):
    model = _cfg_model(collect)
    host, graph, before = _one_update(model, it, pcl_seed=it if collect else None)
    assert not torch.equal(host[0], before[0])
    for h, g in zip(host, graph):
        assert torch.equal(h, g)
    if collect:
        assert float(graph[2].abs().sum()) == 0.0


@pytest.mark.parametrize("levels", [16, 17])
def test_one_update_equals_host_sized_street(cuda, levels):
    model = _street_model(levels)
    host, graph, _ = _one_update(model, 512)
    for h, g in zip(host, graph):
        assert torch.equal(h, g)


def test_one_update_at_an_annealed_level(cuda):
    model = _cfg_model(False)
    model.max_level = 9
    host, graph, _ = _one_update(model, 512)
    for h, g in zip(host, graph):
        assert torch.equal(h, g)


def test_one_update_on_a_grid_without_empty_voxels(cuda):
    model = _cfg_model(False)
    model.accel.occ.set_occ_grid(torch.ones(64, 64, 64, dtype=torch.bool, device=cuda))
    host, graph, _ = _one_update(model, 512)
    for h, g in zip(host, graph):
        assert torch.equal(h, g)


def test_a_grid_without_occupied_voxels_changes_nothing_and_check_raises(cuda):
    model = _cfg_model(True)
    occ = model.accel.occ
    occ.set_occ_grid(torch.zeros(64, 64, 64, dtype=torch.bool, device=cuda))
    _seed_pcl(occ, 4)
    with pytest.raises(AssertionError, match="becomes empty"):
        occ.step(512, model.query_sdf)                                    # the host-sized update asserts
    before = _state(occ)
    upd = OccGridUpdate(model)
    assert occ.step(512, model.query_sdf)
    for b, a in zip(before, _state(occ)):
        assert torch.equal(b, a)
    with pytest.raises(RuntimeError, match="becomes empty during training"):
        upd.check()


# ------------------------------------------------------------------------------------------------------------ a training loop
N_RAYS = 4096


def _batch(it):
    o, d = bench.pinhole_rays(120, 160, bench.orbit(it % 8, 8))
    sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(it))[:N_RAYS]
    return o[sel].cuda(), d[sel].cuda()


def test_training_loop_with_the_update_equals_the_host_path(cuda):
    """48 StaticFrame steps with an update every 16 (warm-up at 16, steady at 32 and 48), SGD on arm a, arm b's parameters copied from a
    after every step: both arms see the same parameters, so their grids, losses and rendered images must agree bit for bit; the gradients
    agree to the order of the fp32 atomics (the spread of two runs of one arm)"""
    from neuralsim_b200.graphics.neus_static import StaticFrame
    a = _cfg_model(True)
    b = copy.deepcopy(a)
    for m in (a, b):
        m.accel.occ.n_steps_warmup = 32
        m.accel.occ.update_from_net_cfg = dict(num_steps=2, num_pts=2 ** 17)
    upd = OccGridUpdate(a)
    frames = [StaticFrame(m, N_RAYS, loss_fn=bench.loss_of, near=0.01, zero_grads=True) for m in (a, b)]
    opt = torch.optim.SGD(a.parameters(), lr=1e-3)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    changed = 0
    for it in range(1, 49):
        off = gen.get_offset()
        a.training_before_per_step(it)
        gen.set_offset(off)                               # both arms' updates draw from the same state
        b.training_before_per_step(it)
        gen.set_offset(off)
        o, d = _batch(it)
        loss_a, loss_b = frames[0].step(o, d), frames[1].step(o, d)
        assert torch.equal(loss_a, loss_b), it
        for k, v in frames[1].rendered.items():
            assert torch.equal(frames[0].rendered[k], v), (it, k)
        for s_a, s_b in zip(_state(a.accel.occ), _state(b.accel.occ)):
            assert torch.equal(s_a, s_b), it
        for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
            if pa.grad is not None:
                assert rel_l2(pa.grad, pb.grad) < 1e-4, (it, n)
        if it % 16 == 0:
            upd.check()
            changed += 1
        opt.step()
        with torch.no_grad():
            for pa, pb in zip(a.parameters(), b.parameters()):
                pb.copy_(pa)
    assert changed == 3 and upd.graph is not None


def test_an_update_iteration_does_not_synchronise(cuda):
    model = _cfg_model(True)
    upd = OccGridUpdate(model)
    occ = model.accel.occ
    assert occ.step(16, model.query_sdf)                  # the first update captures
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        assert occ.step(32, model.query_sdf)
        assert occ.step(512, model.query_sdf)
        assert not occ.step(513, model.query_sdf)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    upd.check()
