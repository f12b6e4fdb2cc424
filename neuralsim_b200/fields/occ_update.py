"""The occupancy grid's update from the network as one CUDA graph (csrc/occ_update.cu, csrc/occ_ema.cu): OccGridEma.step without a host read.

The host-sized step (fields/accel.py:OccGridEma.step, the reference's ema_single.py:133-190) reads the occupied and the empty voxel lists
back with nonzero() -- a synchronisation that drains every graph step queued before it -- and sizes its draws and queries from them.  Here
one replay builds both lists on the device, draws the num_steps iterations' points from torch's CUDA generator (the values
sample_pts_in_voxels draws from the same state), queries the SDF with the fused kernel at the model's device level bound and runs the EMA
over the device count of points, with torch_rng.py's generator contract: `reservation(...)` bounds what an update can draw."""
from __future__ import annotations

import torch

from .. import _lib as L
from .. import torch_rng as TR
from .accel import OccGridEma, OccGridEmaBatched
from .networks import sdf_fwd

__all__ = ["OccGridUpdate", "part_points", "capacity", "reservation", "voxel_lists", "draw_pts", "EMPTY_GRID_MSG"]

EMPTY_GRID_MSG = ("Occupancy grid becomes empty during training. Your model/algorithm/training settings might be incorrect. "
                  "Please check configs and tensorboard.")


def part_points(n: int, cells: int) -> int:
    """the most points sample_pts_in_voxels(gidx, n) returns for any nv <= cells: n (n < 2 nv), else nv (n // nv + 1) <= n + nv with nv <= n / 2"""
    return int(n) + min(int(cells), int(n) // 2)


def _phases(num_pts):
    """the parts' point counts of one iteration, per phase: warm-up, steady (all cells, empty, occupied)"""
    return [num_pts], [num_pts // 2, num_pts // 4, num_pts // 4]


def capacity(cells: int, num_steps: int, num_pts: int) -> int:
    """points one update may draw (the arena; csrc/occ_update.cu checks the same bound)"""
    return int(num_steps) * max(sum(part_points(n, cells) for n in ph) for ph in _phases(int(num_pts)))


def reservation(cells: int, num_steps: int, num_pts: int, cap: int) -> int:
    """generator offsets one update reserves.  A part of n points draws randint([n]) + rand([n, 3]) or rand([nv, per, 3]) with nv per <=
    part_points(n, cells); inc() is monotone in N, so the larger of the two branches' bounds bounds the part whatever nv is.  Refuses a draw
    of 2^31 or more values."""
    def part(n):
        return max(TR.uniform_inc(n, cap) + TR.uniform_inc(3 * n, cap), TR.uniform_inc(3 * part_points(n, cells), cap))
    TR.check_draw(3 * part_points(int(num_pts), cells), "the occupancy update")
    return int(num_steps) * max(sum(part(n) for n in ph) for ph in _phases(int(num_pts)))


def voxel_lists(occ_grid, occupied, empty, counts, flags, first, ws):
    """occupied / empty [cells] int64 := the flat indices of occ_grid's occupied / empty cells in nonzero() order; counts[0], counts[1] := their
    numbers (nsb_occ_voxel_lists; flags / first: int32 [cells] scratch, ws: the scan workspace)"""
    P = L.ptr
    g = occ_grid.view(torch.uint8)
    L.check(L.lib().nsb_occ_voxel_lists(P(g, "u8", "occ_grid"), g.numel(), P(flags, "i32"), P(first, "i32"), P(occupied, "i64"), P(empty, "i64"),
                                        P(counts, "i64"), P(ws), L.stream_ptr()), "occ_voxel_lists")


def draw_pts(rng, warmup, counts, occupied, empty, res, num_steps, num_pts, pts, out):
    """pts [capacity, 3] := the points of one update's num_steps iterations, drawn at (rng[0], rng[1]); out[0] := their number, out[1] := 1
    when the steady phase (warmup == 0) found no occupied voxel (nsb_occ_draw_pts)"""
    P = L.ptr
    L.check(L.lib().nsb_occ_draw_pts(P(rng, "i64", "rng"), P(warmup, "i32", "warmup"), P(counts, "i64"), P(occupied, "i64"), P(empty, "i64"),
                                     int(res[0]), int(res[1]), int(res[2]), int(num_steps), int(num_pts), pts.shape[0], P(pts, "f32"), P(out, "i64"),
                                     L.stream_ptr()), "occ_draw_pts")


class OccGridUpdate:
    """`OccGridEma.step`'s update from the network, captured once as a CUDA graph and attached to `model.accel.occ`: from then on
    `model.training_before_per_step(it)` (-> OccGridEma.step(it, model.query_sdf)) decides on the host whether `it` is an update
    iteration (it > 0 and it % n_steps_between_update == 0) and replays the graph -- no host read, no synchronisation.  The graph:

        fp16 images of the SDF masters -> voxel lists (one scan) -> the points of all num_steps iterations (one kernel) -> the fused SDF query
        at the level bound of this iteration (a device scalar) -> the EMA over the device count (decay, max, threshold; merges and zeroes
        the collected evidence)

    Both phases (warm-up: it < n_steps_warmup; steady) come from the one capture: a device scalar holds the phase.  `occ_grid` and
    `occ_val_grid` are updated in place, so a captured StaticFrame step sees the new grid.

    Random state: torch_rng.take before each replay, with `self.reservation`; from the same generator state the replay draws exactly the
    host-sized update's points, so it leaves the same grids (runs of the two drift apart: torch_rng.py).

    If the steady phase finds no occupied voxel the update changes nothing and records it; `check()` (one device-to-host read) then raises the
    reference's error.  The update's size (`update_from_net_cfg`, the grid's resolution) is read when the object is made.  Memory: an arena
    of `capacity(...)` points (at most 1.5 num_steps num_pts) plus a few int64 arrays of the grid size."""

    def __init__(self, model, generator=None):
        accel = getattr(model, "accel", None)
        occ = getattr(accel, "occ", None)
        if isinstance(occ, OccGridEmaBatched):
            raise RuntimeError("OccGridUpdate: batched occupancy grids (OccGridEmaBatched) are not built; their update stays host-sized")
        if not isinstance(occ, OccGridEma):
            raise RuntimeError(f"OccGridUpdate: the model has no single occupancy grid (model.accel.occ is {type(occ).__name__})")
        if not model.implicit_surface._fusable():
            raise RuntimeError("OccGridUpdate: the model's SDF does not run on the fused kernels (LoTDSDF._fusable(): e.g. more levels than "
                               f"max_fused_levels={model.implicit_surface.max_fused_levels}); its update stays host-sized")
        g, v = occ.occ_grid, occ.occ_val_grid
        if g.dim() != 3 or not g.is_cuda or not g.is_contiguous() or v.dtype != torch.float32 or not v.is_contiguous() or v.shape != g.shape:
            raise RuntimeError("OccGridUpdate: the grid must be a contiguous 3-D CUDA grid with a float32 occ_val_grid")
        self.model, self.occ = model, occ
        dev = g.device
        self.gen = TR.cuda_generator(generator, dev)
        cfg = occ.update_from_net_cfg
        self.num_steps, self.num_pts = int(cfg.get("num_steps", 4)), int(cfg.get("num_pts", 2 ** 18))       # OccGridEma.step's defaults
        self.res = [int(r) for r in g.shape]
        cells = g.numel()
        self.reservation = reservation(cells, self.num_steps, self.num_pts, TR.grid_cap(dev))
        self.capacity = capacity(cells, self.num_steps, self.num_pts)
        i64 = dict(dtype=torch.int64, device=dev)
        self.rng = torch.zeros(2, **i64)
        self.warmup = torch.zeros((), dtype=torch.int32, device=dev)
        self.max_level = torch.zeros((), dtype=torch.int32, device=dev)
        self.counts = torch.zeros(2, **i64)                 # occupied, empty voxels
        self.out = torch.zeros(2, **i64)                    # points drawn, no-occupied-voxel flag
        self.occupied, self.empty = torch.zeros(2, cells, **i64).unbind(0)
        self._flags, self._first = torch.zeros(2, cells, dtype=torch.int32, device=dev).unbind(0)
        from ..graphics.neus_fused import _scan_ws_bytes
        self._ws = torch.zeros(_scan_ws_bytes(), dtype=torch.uint8, device=dev)
        self.pts = torch.zeros(self.capacity, 3, device=dev)
        self.sdf = torch.zeros(self.capacity, device=dev)
        self._scratch = torch.zeros(cells, device=dev)
        self.graph, self._captured, self._held = None, None, None
        occ.net_update = self

    def _targets(self):
        o = self.occ
        return (o.occ_grid, o.occ_val_grid, o._occ_val_grid_pcl if o.should_collect_samples else None)

    @torch.no_grad()
    def _run(self):
        from ..graphics.neus_static import _fp16_images
        m, o = self.model, self.occ
        t16, dec, _net, _ = _fp16_images(m, radiance=False)          # re-cast inside the graph: it follows the optimizer's updates
        self._held = (t16, dec)
        grid, val, pcl = self._targets()
        voxel_lists(grid, self.occupied, self.empty, self.counts, self._flags, self._first, self._ws)
        draw_pts(self.rng, self.warmup, self.counts, self.occupied, self.empty, self.res, self.num_steps, self.num_pts, self.pts, self.out)
        sdf_fwd(m.implicit_surface.encoding.meta, t16[0], dec, self.sdf, self.max_level, x=self.pts, count=(self.out, 0))
        P = L.ptr
        L.check(L.lib().nsb_occ_ema_update_count(P(self.pts, "f32"), P(self.sdf, "f32"), L.slot(self.out, 0), self.capacity, 1, o.occ_inv_s,
                                                 *self.res, P(pcl, "f32", allow_none=True), P(val, "f32"), P(grid.view(torch.uint8), "u8"), None,
                                                 o.ema_decay, o.occ_thre, P(self._scratch), L.slot(self.out, 1), L.stream_ptr()), "occ_ema_update_count")

    def capture(self):
        """one eager run on copies of the grids' state (module loads, the allocator), then the capture"""
        if not bool(self.occ.is_initialized):
            raise RuntimeError("OccGridUpdate: init() the occupancy grid first")
        self.model._nablas_fac()             # _fp16_images reads it; its first call reads the device, which a capture must not do
        saved = [t.clone() if t is not None else None for t in self._targets()]
        TR.take(self.gen, 0, self.rng)
        self._run()
        for t, s in zip(self._targets(), saved):
            if t is not None:
                t.copy_(s)
        torch.cuda.synchronize(self.rng.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._run()
        self.graph = g
        self._captured = [t.data_ptr() if t is not None else None for t in self._targets()]
        return self

    def step(self, cur_it, val_query_fn=None):
        """OccGridEma.step's schedule; on an update iteration, refresh the phase, the level bound and the random state, and replay.
        -> True if it updated"""
        if val_query_fn is not None and val_query_fn != self.model.query_sdf:
            raise RuntimeError("OccGridUpdate: the captured update queries the model's own query_sdf; another val_query_fn needs the host-sized "
                               "update (detach it: model.accel.occ.net_update = None)")
        o = self.occ
        if cur_it <= 0 or cur_it % o.n_steps_between_update != 0:
            return False
        self.warmup.fill_(1 if cur_it < o.n_steps_warmup else 0)
        self.max_level.fill_(self.model.implicit_surface._ml(self.model.max_level))
        if self.graph is not None and self._captured != [t.data_ptr() if t is not None else None for t in self._targets()]:
            self.graph = None                                        # a grid buffer was re-assigned (set_occ_grid): capture again
        if self.graph is None:
            self.capture()
        TR.take(self.gen, self.reservation, self.rng)
        self.graph.replay()
        return True

    def check(self):
        """one device-to-host read: raises the reference's error if the last update found no occupied voxel (and so changed nothing)"""
        if int(self.out[1]) != 0:
            raise RuntimeError(EMPTY_GRID_MSG)
