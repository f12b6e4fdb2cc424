"""The LiDAR batch source of the one-launch step (csrc/lidar_sample.cu): LidarDataset.sample_merged (dataio/data_loader/lidar_loader.py:
119-204) in the merged_weighted / merged_equal modes of every shipped StreetSurf LiDAR config (`lidar_dataset: {equal_mode: ray_batch,
lidar_sample_mode: merged_weighted}`), with the beams moved to world as the trainer does (MultiRaysLidarBundle.get_selected_rays,
app/resources/observers/lidars.py:80-175).

The reference reads the frame's per-lidar beam counts back to the host on every step (unique_consecutive + .cpu()), splits num_rays in
float64 numpy and draws one torch.randint per lidar.  The counts of a frame are fixed once the data are preloaded (filter_when_preload runs
at load time), so `LidarSampler` splits every frame once, with the reference's arithmetic (`lidar_split`), into a device table; the kernel
then draws the per-lidar randints of torch's CUDA generator in-kernel (torch_uniform.cuh), gathers the beams and applies each (lidar,
frame)'s 3 x 4 transform.  `recipe_sample_merged` keeps the reference's torch ops as the reference the kernel is compared against.

One difference by construction: the reference zeroes the weights of empty lidars IN `self.multi_lidar_weight` (lidar_loader.py:167-168
assign into the stored array), so with merged_weighted a frame with an empty lidar changes the split of every frame drawn after it; here
each frame is split from the configured weights, as a freshly built LidarDataset splits it.

Not built (RuntimeError): lidar_sample_mode other than merged_weighted / merged_equal, equal_mode point_batch, a frame without beams, more
than NSB_LIDAR_MAX lidars, a lidar with 2^32 or more beams in a frame."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib as L
from . import torch_rng as TR

__all__ = ["LidarSampler", "lidar_split", "recipe_sample_merged", "LIDAR_MAX", "TABLE_WIDTH"]

LIDAR_MAX, TABLE_WIDTH = 8, 32           # include/neuralsim_b200.h NSB_LIDAR_MAX, NSB_LIDAR_TABLE_WIDTH
_DATA_OFF, _POSE_BASE, _INC, _N_LIDARS, _RAY_START = 0, 1, 2, 3, 4
_CUMU = _RAY_START + LIDAR_MAX + 1
_DRAW_OFF = _CUMU + LIDAR_MAX + 1
_MODES = ("merged_weighted", "merged_equal")


def _normalized_weight(multi_lidar_weight, lidar_sample_mode):
    """LidarDataset.__init__'s weight (lidar_loader.py:63-68): the given weights normalised for the weighted modes, None otherwise"""
    if lidar_sample_mode not in _MODES:
        raise RuntimeError(f"LidarSampler: lidar_sample_mode={lidar_sample_mode!r} is not built (built: {', '.join(_MODES)})")
    if "weighted" not in lidar_sample_mode:
        return None
    if multi_lidar_weight is None:
        raise RuntimeError("LidarSampler: lidar_sample_mode='merged_weighted' needs multi_lidar_weight")
    w = np.array(multi_lidar_weight)
    return w / w.sum()


def lidar_split(cnt, num_rays, weight):
    """the reference's split of num_rays over the lidars (lidar_loader.py:166-176) for beam counts cnt [L] and the normalised weight
    (None: equal): -> list of L ray counts"""
    cnt = np.asarray(cnt)
    weight = np.full([len(cnt), ], 1 / len(cnt)) if weight is None else np.array(weight, copy=True)
    weight[cnt == 0] = 0
    weight = weight / weight.sum()
    num_rays_each_lidar = np.array(num_rays * weight, dtype=int).tolist()
    if sum(num_rays_each_lidar) != num_rays:
        for i, n in enumerate(num_rays_each_lidar):
            if n != 0:
                break
        num_rays_each_lidar[i] += (num_rays - sum(num_rays_each_lidar))
    return num_rays_each_lidar


@torch.no_grad()
def recipe_sample_merged(rays_o, rays_d, ranges, li, n_lidars, num_rays, weight, generator=None):
    """LidarDataset.sample_merged (lidar_loader.py:160-196) on one frame's merged beams (li [N] non-decreasing, the lidar of each beam)
    with the normalised weight (None: merged_equal), drawing from `generator` (else torch's default one of the data's device).
    -> dict(split, inds, li, rays_o, rays_d, ranges): the beams in lidar-local coordinates"""
    dev = rays_o.device
    cnt = torch.zeros([n_lidars, ], dtype=torch.long, device=dev)
    unique_i, unique_cnt = torch.unique_consecutive(li, return_counts=True)
    cnt[unique_i] = unique_cnt
    cnt = cnt.data.cpu().numpy()
    num_rays_each_lidar = lidar_split(cnt, num_rays, weight)
    cumu_cnt = [0, *np.cumsum(cnt).tolist()]
    inds = torch.cat([torch.randint(cumu_cnt[i], cumu_cnt[i + 1], [num, ], device=dev, dtype=torch.long, generator=generator)
                      for i, num in enumerate(num_rays_each_lidar) if num > 0])
    return dict(split=num_rays_each_lidar, inds=inds, li=li[inds], rays_o=rays_o[inds], rays_d=rays_d[inds], ranges=ranges[inds])


class LidarSampler:
    """The batch source of StaticFrame(sampler=LidarSampler(...)).

        rays_o, rays_d  [N, 3] float32: every frame's merged beams in lidar-local coordinates, frame after frame, each frame's beams
                        ordered by lidar (the merged data's `li` is non-decreasing)
        ranges          [N] float32
        counts          [F, L] integer (tensor or array): the beams of lidar li in frame f; N = counts.sum()
        l2w             [F, L, 3, 4] float32: the lidar-to-world transform of lidar li at frame f, as the trainer evaluates its scene graph
        num_rays        the batch (`lidar_dataset.num_rays`)
        multi_lidar_weight, lidar_sample_mode, equal_mode: the `lidar_dataset` settings

    The split of every frame is computed here, once (`split[f]`).  `sample(frame_ind, generator)` draws one batch on the kernel outside
    a graph; `frame.step(frame_ind=f)` draws frame f's batch inside the graph.  With LidarLoss the ranges reach the loss inside the
    replay: `loss_fn = lambda ret, gt: sum(lidar_loss(None, ret, ground_truth=gt).values())`, its weights set by
    `lidar_loss.set_step(None, it)` before `step()`."""

    def __init__(self, rays_o, rays_d, ranges, counts, l2w, num_rays, multi_lidar_weight=None, *, lidar_sample_mode="merged_weighted",
                 equal_mode="ray_batch"):
        if equal_mode != "ray_batch":
            raise RuntimeError(f"LidarSampler: equal_mode={equal_mode!r} is not built (only 'ray_batch'; the reference's point_batch is WIP)")
        self.weight = _normalized_weight(multi_lidar_weight, lidar_sample_mode)
        self.lidar_sample_mode = lidar_sample_mode
        counts = np.asarray(counts.cpu() if isinstance(counts, torch.Tensor) else counts).astype(np.int64)
        if counts.ndim != 2 or counts.shape[0] < 1 or counts.shape[1] < 1 or (counts < 0).any():
            raise RuntimeError(f"LidarSampler: counts must be a non-negative [n_frames, n_lidars] array, got shape {counts.shape}")
        F, Ln = counts.shape
        if Ln > LIDAR_MAX:
            raise RuntimeError(f"LidarSampler: {Ln} lidars, at most NSB_LIDAR_MAX = {LIDAR_MAX} are built")
        if self.weight is not None and len(self.weight) != Ln:
            raise RuntimeError(f"LidarSampler: multi_lidar_weight has {len(self.weight)} entries for {Ln} lidars")
        if (counts >= 2 ** 32).any():
            f, li = (int(v) for v in np.argwhere(counts >= 2 ** 32)[0])
            raise RuntimeError(f"LidarSampler: frame {f} lidar {li} has {counts[f, li]} beams; a segment of 2^32 or more beams is not built")
        num_rays = int(num_rays)
        if not 1 <= num_rays < 2 ** 31:
            raise RuntimeError(f"LidarSampler: num_rays must lie in [1, 2^31), got {num_rays}")
        N = int(counts.sum())
        dev = rays_o.device
        for name, t, shape in (("rays_o", rays_o, (N, 3)), ("rays_d", rays_d, (N, 3)), ("ranges", ranges, (N,)), ("l2w", l2w, (F, Ln, 3, 4))):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous() or t.device != dev:
                raise RuntimeError(f"LidarSampler: {name} must be a contiguous float32 tensor {list(shape)} on {dev}, "
                                   f"got {getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
        self.rays_o, self.rays_d, self.ranges, self.l2w = rays_o, rays_d, ranges, l2w
        self.counts, self.num_rays, self.n_frames, self.n_lidars, self.device = counts, num_rays, F, Ln, dev
        self._cap = None
        self.split, self._rows = [], []
        data_off = 0
        for f in range(F):
            if counts[f].sum() == 0:
                raise RuntimeError(f"LidarSampler: frame {f} has no beams")
            with np.errstate(invalid="ignore", divide="ignore"):
                split = lidar_split(counts[f], num_rays, self.weight)
            if any(n < 0 for n in split) or sum(split) != num_rays or any(n > 0 and c == 0 for n, c in zip(split, counts[f])):
                raise RuntimeError(f"LidarSampler: frame {f}: the weights give no rays to its lidars with beams (split {split}, counts "
                                   f"{counts[f].tolist()})")
            self.split.append(split)
            row = [0] * TABLE_WIDTH
            row[_DATA_OFF], row[_POSE_BASE], row[_N_LIDARS] = data_off, f * Ln, Ln
            rs, cu = np.concatenate([[0], np.cumsum(split)]), np.concatenate([[0], np.cumsum(counts[f])])
            row[_RAY_START:_RAY_START + Ln + 1] = [int(v) for v in rs]
            row[_CUMU:_CUMU + Ln + 1] = [int(v) for v in cu]
            self._rows.append(row)
            data_off += int(counts[f].sum())
        self.frame = torch.zeros((), dtype=torch.int64, device=dev)
        self.table = None

    def rows(self, cap):
        """the table rows (host lists, include/neuralsim_b200.h nsb_lidar_sample) for torch's grid cap `cap`, which the draw offsets
        depend on"""
        for row, split in zip(self._rows, self.split):
            o = 0
            for li, num in enumerate(split):
                row[_DRAW_OFF + li] = o
                o += TR.uniform_inc(num, cap)
            row[_INC] = o
        return [list(r) for r in self._rows]

    def _table(self, cap):
        if self._cap != cap:
            self.table = torch.tensor(self.rows(cap), dtype=torch.int64).to(self.device)
            self._cap = cap
        return self.table

    def frame_inc(self, f, cap):
        """the generator offsets frame f's draws advance: sum over its lidars of inc(num_li)"""
        return sum(TR.uniform_inc(num, cap) for num in self.split[f])

    def inc(self, n, cap):
        """the reservation of one draw of n (= num_rays) rays: the largest frame_inc over the frames (bounds every frame's draws)"""
        if int(n) != self.num_rays:
            raise RuntimeError(f"LidarSampler: the frame draws {n} rays, the sampler was split for num_rays = {self.num_rays}")
        return max(self.frame_inc(f, cap) for f in range(self.n_frames))

    def check_frame(self, frame_ind):
        if isinstance(frame_ind, bool) or not isinstance(frame_ind, (int, np.integer)) or not 0 <= int(frame_ind) < self.n_frames:
            raise RuntimeError(f"LidarSampler: frame_ind must be an int in [0, {self.n_frames}), got {frame_ind!r}")
        return int(frame_ind)

    def launch(self, frame, rng, rays_o, rays_d, ranges, li, rays_fidx, rng_next=None):
        """nsb_lidar_sample: frame *frame's batch (frame: device int64 scalar) from rng = device int64 {seed, offset} into the buffers"""
        P = L.ptr
        table = self._table(TR.grid_cap(self.device))
        L.check(L.lib().nsb_lidar_sample(P(table, "i64", "table"), P(frame, "i64", "frame"), P(rng, "i64", "rng"), L.c_i64(self.num_rays),
                                         P(self.rays_o, "f32", "rays_o"), P(self.rays_d, "f32", "rays_d"), P(self.ranges, "f32", "ranges"),
                                         P(self.l2w, "f32", "l2w"), P(rays_o, "f32", "out rays_o"), P(rays_d, "f32", "out rays_d"),
                                         P(ranges, "f32", "out ranges"), P(li, "i64", "li"), P(rays_fidx, "i64", "rays_fidx"),
                                         P(rng_next, "i64", "rng_next", allow_none=True), L.stream_ptr()), "lidar_sample")

    @torch.no_grad()
    def sample(self, frame_ind, generator=None):
        """frame frame_ind's batch on the kernel from torch's CUDA generator (`generator`, else the default one), which then moves past
        the draws as the reference's randints move it.  -> dict(rays_o, rays_d (world), ranges, li, rays_fidx)"""
        f = self.check_frame(frame_ind)
        n, dev = self.num_rays, self.device
        self.frame.fill_(f)
        rng = TR.take(TR.cuda_generator(generator, dev), self.frame_inc(f, TR.grid_cap(dev)))
        out = dict(rays_o=torch.empty(n, 3, device=dev), rays_d=torch.empty(n, 3, device=dev), ranges=torch.empty(n, device=dev),
                   li=torch.empty(n, dtype=torch.int64, device=dev), rays_fidx=torch.empty(n, dtype=torch.int64, device=dev))
        self.launch(self.frame, rng, out["rays_o"], out["rays_d"], out["ranges"], out["li"], out["rays_fidx"])
        return out

    def frame_data(self, frame_ind):
        """frame frame_ind's merged beams (views) and their lidar indices: -> (rays_o, rays_d, ranges, li)"""
        f = self.check_frame(frame_ind)
        a = int(self.counts[:f].sum())
        b = a + int(self.counts[f].sum())
        li = torch.repeat_interleave(torch.arange(self.n_lidars), torch.from_numpy(self.counts[f])).to(self.device)
        return self.rays_o[a:b], self.rays_d[a:b], self.ranges[a:b], li

    def recipe(self, frame_ind, generator=None):
        """recipe_sample_merged on frame frame_ind's data"""
        o, d, r, li = self.frame_data(frame_ind)
        return recipe_sample_merged(o, d, r, li, self.n_lidars, self.num_rays, self.weight, generator)

    # -- the batch source of a StaticFrame: every per-frame buffer lives on the frame, so one sampler serves several frames
    def attach(self, frame):
        """check the frame, give it `frame_ind` (a device index), `rays_li`, `rays_fidx`, `ground_truth` = {"ranges"}.  -> the draw's reservation"""
        if frame.pose is not None or frame.with_rgb:
            raise RuntimeError("StaticFrame(sampler=LidarSampler): needs with_rgb=False, and takes no pose= (the sampler writes the world rays)")
        dev, n = frame.device, frame.n_rays
        frame.frame_ind = torch.zeros((), dtype=torch.int64, device=dev)
        frame.rays_li = torch.zeros(n, dtype=torch.int64, device=dev)
        frame.rays_fidx = torch.zeros(n, dtype=torch.int64, device=dev)
        frame.ground_truth = dict(ranges=torch.zeros(n, device=dev))
        return self.inc(n, TR.grid_cap(dev))

    def select(self, frame, cam, frame_ind, rays):
        """frame.step(frame_ind=f), which takes no cam or rays: f into frame.frame_ind.  -> None: nothing runs on the host after the step"""
        if cam is not None or any(v is not None for v in rays):
            raise RuntimeError("StaticFrame.step: a frame with sampler=LidarSampler draws its own batch; pass frame_ind= only")
        frame.frame_ind.fill_(self.check_frame(frame_ind))

    def draw(self, frame, rng):
        """frame frame.frame_ind's batch, drawn at the device block rng: world rays, `rays_li` (the reference's rays_sel), `rays_fidx`, ranges"""
        self.launch(frame.frame_ind, rng, frame.rays_o, frame.rays_d, frame.ground_truth["ranges"], frame.rays_li, frame.rays_fidx, frame.rng)

    def loss(self, frame, arg):
        """-> (frame.loss_fn(arg, frame.ground_truth), None: nothing runs after the backward)"""
        return frame.loss_fn(arg, frame.ground_truth), None

    def check(self, frame):
        """nothing to check: a LiDAR draw records no error"""
