"""Occupancy-grid acceleration -- API of `nr3d_lib.models.accelerations.OccGridEma / OccGridAccel`
(reference: models/accelerations/occgrid/ema_single.py:21-260, occgrid/utils.py:17-109, occgrid_accel/single.py:36-135).
torch_scatter's `scatter_max(out=decay*grid)` is `Tensor.scatter_reduce_('amax', include_self=True)` here."""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn

from ..graphics.raymarch import occgrid_raymarch


# True: the EMA update of a CUDA grid runs as the kernels of csrc/occ_ema.cu; False: as the torch restatement of the reference's chain
# (scatter_reduce_('amax') for torch_scatter's scatter_max) -- tests/test_occ_ema_gpu.py compares both with the oracle.
DEVICE_EMA = True


def sample_pts_in_voxels(gidx, num_pts, resolution, dtype=torch.float, generator=None):
    """Uniform points in [-1,1]^3 inside the listed voxels (+ the voxel each one fell in)  (utils.py:17-41)."""
    device, nv = gidx.device, gidx.shape[0]
    if num_pts / nv < 2.0:
        vidx = torch.randint(nv, [num_pts], device=device, generator=generator)
        off = torch.rand([num_pts, 3], device=device, dtype=dtype, generator=generator)
        return ((gidx[vidx] + off) / resolution.float()) * 2 - 1, vidx
    per = int(num_pts // nv) + 1
    off = torch.rand([nv, per, 3], device=device, dtype=dtype, generator=generator)
    pts = ((gidx[:, None, :] + off) / resolution.float()).view(-1, 3) * 2 - 1
    return pts, torch.arange(nv, device=device).unsqueeze(-1).expand(nv, per).reshape(-1)


def sdf_to_occ_val(sdf, inv_s):
    """normalised logistic density with peak 1, as the reference writes it: (1 / cosh(clamp(inv_s x / 2, -20, 20)))^2
    (nr3d_lib/maths/common.py:122-133), evaluated in the dtype of `sdf` (the reference's sdf is a half tensor)."""
    return (1. / torch.cosh((inv_s * sdf / 2.).clamp_(-20, 20))) ** 2


class OccGridEma(nn.Module):
    def __init__(self, resolution=(64, 64, 64), occ_val_fn_cfg=dict(type="sdf", inv_s=256.0), occ_thre=0.3, ema_decay=0.95,
                 init_cfg=dict(mode="from_net", num_steps=4, num_pts=2 ** 20), update_from_net_cfg=dict(num_steps=4, num_pts=2 ** 20),
                 update_from_samples_cfg=dict(), n_steps_between_update=16, n_steps_warmup=256, dtype=torch.float, device=None):
        super().__init__()
        res = torch.tensor([resolution] * 3 if isinstance(resolution, int) else list(resolution), dtype=torch.int32, device=device)
        self.register_buffer("is_initialized", torch.tensor([False], dtype=torch.bool, device=device), persistent=True)
        self.register_buffer("resolution", res, persistent=False)
        self.register_buffer("occ_grid", torch.zeros(res.tolist(), dtype=torch.bool, device=device), persistent=True)
        self.register_buffer("occ_val_grid", torch.zeros(res.tolist(), dtype=dtype, device=device), persistent=True)
        g = torch.stack(torch.meshgrid([torch.arange(r, device=device) for r in res.tolist()], indexing="ij"), -1).view(-1, 3)
        self.register_buffer("gidx_full", g, persistent=False)
        if occ_val_fn_cfg.get("type", "sdf") != "sdf":
            raise RuntimeError("only occ_val_fn type 'sdf' is built")
        self.occ_inv_s = float(occ_val_fn_cfg["inv_s"])
        self.occ_thre, self.ema_decay = occ_thre, ema_decay
        self.init_cfg, self.update_from_net_cfg = dict(init_cfg), dict(update_from_net_cfg)
        self.should_collect_samples = update_from_samples_cfg is not None
        self.n_steps_between_update, self.n_steps_warmup = n_steps_between_update, n_steps_warmup
        if self.should_collect_samples:
            self.register_buffer("_occ_val_grid_pcl", torch.zeros(res.tolist(), dtype=dtype, device=device), persistent=False)
        self.net_update = None          # an attached fields/occ_update.py:OccGridUpdate runs step()'s update as one graph replay

    def occ_val_fn(self, sdf):
        # the model's sdf is fp16-valued (autocast decoder): evaluate like the reference does on its half tensor, then widen
        return sdf_to_occ_val(sdf.half(), self.occ_inv_s).float()

    def _set_grid(self, new):
        """the reference re-assigns `self.occ_grid = binarize(...)` (ema_single.py:190); here the buffer is updated IN PLACE when the shape is
        unchanged, so that raw pointers captured by a CUDA graph (graphics/neus_static.py) keep seeing the current grid"""
        if new.shape == self.occ_grid.shape and new.device == self.occ_grid.device:
            self.occ_grid.copy_(new)
        else:
            self.occ_grid = new

    def collect_struct(self):
        """nsb_occ_collect for the fused query kernels (None when samples are not collected): they max-accumulate the occupancy evidence
        of every point they evaluate into `_occ_val_grid_pcl`, which is what `collect_samples(x, sdf)` does after the query."""
        if not (self.training and self.should_collect_samples):
            return None
        from .. import _lib as L
        g = self._occ_val_grid_pcl
        c = L.OccCollectC(g.data_ptr(), (ctypes.c_int32 * 3)(*g.shape), float(self.occ_inv_s))
        c._keep = g
        return c

    def _ravel(self, gidx):
        r = self.occ_val_grid.shape
        return (gidx * gidx.new_tensor([r[1] * r[2], r[2], 1])).sum(-1)

    def _gidx_of(self, pts):
        return ((pts / 2. + 0.5) * self.resolution).long().clamp(self.resolution.new_tensor([0]), self.resolution - 1)

    @torch.no_grad()
    def _update(self, gidx, occ_val, ema_decay):
        """EMA-decay every voxel, take the max with the new evidence, write back only the touched voxels (utils.py:89-101)."""
        flat = self._ravel(gidx)
        new = (ema_decay * self.occ_val_grid.flatten()).scatter_reduce_(0, flat, occ_val.flatten().to(self.occ_val_grid), "amax", include_self=True)
        self.occ_val_grid.view(-1)[flat] = new[flat]
        self._set_grid(self.occ_val_grid > self.occ_thre)

    @torch.no_grad()
    def _step_update_device(self, pts, sdf):
        """`_step_update_occ` (ema_single.py:176-190) as the three launches of csrc/occ_ema.cu: evidence of the points (from their sdf) and the
        evidence collected while rendering -> decay + max on the touched voxels -> threshold (+ the bit-packed grid the marcher reads).
        No nonzero(), no host read."""
        from .. import _lib as L
        r = [int(v) for v in self.occ_val_grid.shape]
        pts = pts.detach().reshape(-1, 3).contiguous().float()
        sdf = sdf.detach().reshape(-1).contiguous().float()
        pcl = self._occ_val_grid_pcl if self.should_collect_samples else None
        scratch = torch.empty(self.occ_val_grid.numel(), dtype=torch.float32, device=pts.device)
        occ = torch.empty(r, dtype=torch.bool, device=pts.device)
        grid = self.occ_val_grid if (self.occ_val_grid.is_contiguous() and self.occ_val_grid.dtype == torch.float32) else self.occ_val_grid.contiguous().float()
        L.check(L.lib().nsb_occ_ema_update(L.ptr(pts, "f32"), L.ptr(sdf, "f32"), L.c_i64(pts.shape[0]), L.c_i32(1), L.c_f32(self.occ_inv_s), L.c_i32(r[0]),
                                           L.c_i32(r[1]), L.c_i32(r[2]), L.ptr(pcl, "f32", allow_none=True), L.ptr(grid, "f32"), L.ptr(occ.view(torch.uint8), "u8"),
                                           None, L.c_f32(self.ema_decay), L.c_f32(self.occ_thre), L.ptr(scratch), L.stream_ptr()), "occ_ema_update")
        if grid is not self.occ_val_grid:
            self.occ_val_grid.copy_(grid)
        self._set_grid(occ)

    @torch.no_grad()
    def set_occ_grid(self, occ_grid):
        self._set_grid(occ_grid.to(self.occ_grid.device).bool().contiguous())
        self.occ_val_grid = self.occ_grid.to(self.occ_val_grid.dtype)
        self.is_initialized.fill_(True)

    @torch.no_grad()
    def init(self, val_query_fn=None, logger=None, generator=None):
        if bool(self.is_initialized):
            return False
        cfg = dict(self.init_cfg)
        mode = cfg.pop("mode")
        if mode == "constant":
            self.occ_val_grid.fill_(cfg["constant_value"])
            self._set_grid(self.occ_val_grid > self.occ_thre)
        elif mode == "from_net":
            for _ in range(cfg.get("num_steps", 4)):
                empty = self.occ_grid.logical_not().nonzero().long()
                if empty.shape[0] > 0:
                    pts = sample_pts_in_voxels(empty, cfg.get("num_pts", 2 ** 18), self.resolution, self.occ_val_grid.dtype, generator)[0]
                    self._update(self._gidx_of(pts), self.occ_val_fn(val_query_fn(pts)), 1.0)
        else:
            raise RuntimeError(f"Invalid init_mode={mode}")
        self.is_initialized.fill_(True)
        return True

    @torch.no_grad()
    def step(self, cur_it, val_query_fn, logger=None, generator=None):
        if self.net_update is not None:
            if generator is not None:
                raise RuntimeError("OccGridEma.step: the attached OccGridUpdate draws from its own generator; pass it to OccGridUpdate(generator=...)")
            return self.net_update.step(cur_it, val_query_fn)
        assert bool(self.is_initialized), "init() first"
        if cur_it <= 0 or cur_it % self.n_steps_between_update != 0:
            return False
        num_steps, num_pts = self.update_from_net_cfg.get("num_steps", 4), self.update_from_net_cfg.get("num_pts", 2 ** 18)
        dt = self.occ_val_grid.dtype
        pts_all, val_all = [], []
        occupied, empty = self.occ_grid.nonzero().long(), self.occ_grid.logical_not().nonzero().long()
        for _ in range(num_steps):
            if cur_it < self.n_steps_warmup:
                pts = sample_pts_in_voxels(self.gidx_full, num_pts, self.resolution, dt, generator)[0]
            else:
                assert occupied.numel() > 0, "Occupancy grid becomes empty during training."
                parts = [sample_pts_in_voxels(self.gidx_full, num_pts // 2, self.resolution, dt, generator)[0]]
                if empty.numel() > 0:
                    parts.append(sample_pts_in_voxels(empty, num_pts // 4, self.resolution, dt, generator)[0])
                parts.append(sample_pts_in_voxels(occupied, num_pts // 4, self.resolution, dt, generator)[0])
                pts = torch.cat(parts, 0)
            pts_all.append(pts)
            val_all.append(val_query_fn(pts))
        if DEVICE_EMA and self.occ_val_grid.is_cuda and self.occ_val_grid.dim() == 3:
            self._step_update_device(torch.cat(pts_all, 0), torch.cat(val_all, 0))
            return True
        pts, occ_val = torch.cat(pts_all, 0), self.occ_val_fn(torch.cat(val_all, 0).flatten())
        gidx = self._gidx_of(pts)
        if self.should_collect_samples:
            idx = self._occ_val_grid_pcl.nonzero().long()
            if idx.numel() > 0:
                gidx = torch.cat([gidx, idx], 0)
                occ_val = torch.cat([occ_val, self._occ_val_grid_pcl[tuple(idx.t())]], 0)
            self._occ_val_grid_pcl.zero_()
        self._update(gidx, occ_val, self.ema_decay)
        return True

    @torch.no_grad()
    def collect_samples(self, pts, val=None):
        """Max-accumulate the occupancy evidence of points seen during rendering (ema_single.py:213-240)."""
        if self.training and self.should_collect_samples and val is not None:
            flat = self._ravel(self._gidx_of(pts.flatten(0, -2)))
            self._occ_val_grid_pcl.view(-1).scatter_reduce_(0, flat, self.occ_val_fn(val.flatten()).to(self._occ_val_grid_pcl), "amax", include_self=True)

    @torch.no_grad()
    def sample_pts_in_occupied(self, num_pts, generator=None):
        return sample_pts_in_voxels(self.occ_grid.nonzero().long(), num_pts, self.resolution, self.occ_val_grid.dtype, generator)[0]


class OccGridAccel(nn.Module):
    """Single-block occupancy-grid accelerator: `occ` (the EMA grid) + `ray_march` (occgrid_accel/single.py:36-135)."""

    def __init__(self, space=None, device=None, **occ_cfg):
        super().__init__()
        occ_cfg.pop("type", None)
        vox_size = occ_cfg.pop("vox_size", None)
        if vox_size is not None and "resolution" not in occ_cfg:
            # occgrid_accel/single.py:51-55: a voxel edge in world units -> per-axis resolution of the cuboid space
            occ_cfg["resolution"] = [max(int(float(e) / float(vox_size)), 1) for e in (space.radius3d * 2).tolist()]      # `.long()`: truncation
        self.space = space
        self.occ = OccGridEma(**occ_cfg, device=device)
        self.training_granularity = 0.0

    def init(self, query_fn, logger=None):
        return self.occ.init(query_fn, logger)

    def step(self, cur_it, query_fn, logger=None):
        return self.occ.step(cur_it, query_fn, logger)

    def collect_samples(self, pts, val=None):
        self.occ.collect_samples(pts, val)

    def sample_pts_in_occupied(self, num_pts):
        return self.occ.sample_pts_in_occupied(num_pts)

    def ray_march(self, rays_o, rays_d, near=None, far=None, perturb=False, **march_cfg):
        return occgrid_raymarch(self.occ.occ_grid, rays_o, rays_d, near, far, perturb=perturb, **march_cfg)


# ---------------------------------------------------------------------------------------------------------------- batched (multi-object)
class OccGridEmaBatched(nn.Module):
    """`num_batches` occupancy grids of one resolution, one per object instance of a shared model (occgrid/ema_batched.py:17-309):
    `occ_val_grid` [B,X,Y,Z] with the EMA / per-voxel-maximum update of `update_batched_occ_val_grid_idx_` (occgrid/utils.py:111-124)."""

    def __init__(self, num_batches, resolution=(32, 32, 32), occ_val_fn_cfg=dict(type="sdf", inv_s=256.0), occ_thre=0.3, ema_decay=0.95,
                 update_from_samples_cfg=dict(), dtype=torch.float, device=None):
        super().__init__()
        res = torch.tensor([resolution] * 3 if isinstance(resolution, int) else list(resolution), dtype=torch.int32, device=device)
        self.num_batches = int(num_batches)
        self.register_buffer("resolution", res, persistent=False)
        shape = [self.num_batches] + res.tolist()
        self.register_buffer("occ_grid", torch.zeros(shape, dtype=torch.bool, device=device), persistent=True)
        self.register_buffer("occ_val_grid", torch.zeros(shape, dtype=dtype, device=device), persistent=True)
        if occ_val_fn_cfg.get("type", "sdf") != "sdf":
            raise RuntimeError("only occ_val_fn type 'sdf' is built")
        self.occ_inv_s, self.occ_thre, self.ema_decay = float(occ_val_fn_cfg["inv_s"]), occ_thre, ema_decay
        self.should_collect_samples = update_from_samples_cfg is not None
        if self.should_collect_samples:
            self.register_buffer("_occ_val_grid_pcl", torch.zeros(shape, dtype=dtype, device=device), persistent=False)

    def occ_val_fn(self, sdf):
        return sdf_to_occ_val(sdf.half(), self.occ_inv_s).float()

    def _gidx_of(self, pts):
        return ((pts / 2. + 0.5) * self.resolution).long().clamp(self.resolution.new_tensor([0]), self.resolution - 1)

    def _ravel(self, bidx, gidx):
        r = self.occ_val_grid.shape[1:]
        return bidx * (r[0] * r[1] * r[2]) + (gidx * gidx.new_tensor([r[1] * r[2], r[2], 1])).sum(-1)

    @torch.no_grad()
    def update(self, pts, bidx, val):
        """`_step_update_occ` with per-point batch indices (ema_batched.py:226-261): evidence of the points + the collected evidence -> decay and
        per-voxel maximum on the touched voxels of the touched grids -> threshold"""
        bidx, occ_val = bidx.flatten().long(), self.occ_val_fn(val.flatten())
        gidx = self._gidx_of(pts.flatten(0, -2))
        if self.should_collect_samples:
            idx = self._occ_val_grid_pcl.nonzero().long()
            if idx.numel() > 0:
                bidx = torch.cat([bidx, idx[:, 0]], 0)
                gidx = torch.cat([gidx, idx[:, 1:]], 0)
                occ_val = torch.cat([occ_val, self._occ_val_grid_pcl[tuple(idx.t())]], 0)
            self._occ_val_grid_pcl.zero_()
        flat = self._ravel(bidx, gidx)
        new = (self.ema_decay * self.occ_val_grid.flatten()).scatter_reduce_(0, flat, occ_val.to(self.occ_val_grid), "amax", include_self=True)
        self.occ_val_grid.view(-1)[flat] = new[flat]
        self.occ_grid = self.occ_val_grid > self.occ_thre

    @torch.no_grad()
    def collect_samples(self, pts, bidx, val):
        if self.training and self.should_collect_samples:
            flat = self._ravel(bidx.flatten().long(), self._gidx_of(pts.flatten(0, -2)))
            self._occ_val_grid_pcl.view(-1).scatter_reduce_(0, flat, self.occ_val_fn(val.flatten()).to(self._occ_val_grid_pcl), "amax", include_self=True)


class OccGridAccelBatched(nn.Module):
    """The accel of a shared (batched) model: the grids of the instances of the CURRENT batch are selected with `set_condition`, rays carry the
    batch index of their object and are marched by the batched kernel (occgrid_accel/batched.py:31-170; csrc/march.cu with `batch_inds`)."""

    def __init__(self, num_batches, device=None, **occ_cfg):
        super().__init__()
        occ_cfg.pop("type", None)
        self.occ = OccGridEmaBatched(num_batches, **occ_cfg, device=device)
        self.training_granularity = 0.0
        self.clean_condition()

    def set_condition(self, batch_size, *, ins_inds_per_batch):
        self.batch_size, self.ins_inds_per_batch = int(batch_size), ins_inds_per_batch
        self.occ_grid_per_batch = self.occ.occ_grid[ins_inds_per_batch].contiguous()

    def clean_condition(self):
        self.batch_size = self.ins_inds_per_batch = self.occ_grid_per_batch = None

    def _need(self):
        if self.occ_grid_per_batch is None:
            raise RuntimeError("OccGridAccelBatched: call set_condition() first")

    @torch.no_grad()
    def cur_batch__query_occupancy(self, pts, bidx):
        self._need()
        g = self.occ._gidx_of(pts)
        return self.occ_grid_per_batch[(bidx,) + tuple(g.movedim(-1, 0))]

    @torch.no_grad()
    def cur_batch__sample_pts_in_occupied(self, num_pts):
        self._need()
        idx = self.occ_grid_per_batch.nonzero().long()
        assert idx.numel() > 0, "Occupancy grid becomes empty during training."
        pts, vidx = sample_pts_in_voxels(idx[:, 1:], num_pts, self.occ.resolution, self.occ.occ_val_grid.dtype)
        return pts, idx[:, 0][vidx]

    def cur_batch__ray_march(self, rays_o, rays_d, rays_bidx=None, *, near=None, far=None, perturb=False, step_size=1e-3, max_step_size=1e10,
                             dt_gamma=0.0, max_steps=512):
        from ..graphics.raymarch import occgrid_raymarch_batched
        self._need()
        return occgrid_raymarch_batched(self.occ_grid_per_batch, rays_o, rays_d, near, far, rays_bidx, perturb=perturb, step_size=step_size,
                                        max_step_size=max_step_size, dt_gamma=dt_gamma, max_steps=max_steps)

    def cur_batch__collect_samples(self, pts, bidx, val):
        self.occ.collect_samples(pts, self.ins_inds_per_batch[bidx], val)

    def cur_batch__step(self, pts, bidx, val):
        """EMA update with points of the current batch (bidx = batch-local instance index)"""
        self.occ.update(pts, self.ins_inds_per_batch[bidx], val)
