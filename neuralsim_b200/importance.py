"""Error-map importance sampling of training pixels on the project's kernels (csrc/importance.cu): the drop-in of
nr3d_lib.models.importance (`ErrorMap`, `ImpSampler`, importance.py:14-336) and the per-camera batch source of the one-launch step
(`CameraSampler`, graphics/neus_static.py StaticFrame(sampler=...)).

The shipped camera configs set `training.error_map` and draw every batch with ImpSampler.sample_img_pixel over one 'rgb' map; the trainer
then feeds the per-ray rgb error back with ErrorMap.step_error_map, which rebuilds the cdfs every n_steps_between_update of that camera's
steps (128, x1.5, up to n_steps_max).  Here `sample_img_pixel` is one kernel (nsb_imp_sample: the reference's four draws of torch's CUDA
generator, searchsorted and 2-D inverse cdf in its fp32 operation order), `update_error_map` two (nsb_error_map_update: the four corner
statements with the last ray of a cell winning, as index_put_ does), and `construct_cdf` stays the reference's torch code, written in place
into buffers allocated once, so a captured step keeps reading them.  `recipe_*` are the reference's own torch ops, kept as the reference the
kernels are compared against.

Not built (RuntimeError): more than one error map (`frac_mask_err > 0`, the `focus_on` maps), `enable_after > 0` (the single-frame uniform
warm-up) and the non-joint PixelDataset's frame weights (check_error_map_cfg)."""
from __future__ import annotations

import ctypes
from numbers import Number

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from . import torch_rng as TR

__all__ = ["ErrorMap", "ImpSampler", "CameraSampler", "check_error_map_cfg", "split", "sampler_inc", "recipe_update_error_map",
           "recipe_sample_img_pixel", "recipe_pixels", "TABLE_WIDTH", "MAX_GT"]

TABLE_WIDTH, MAX_GT = 16, 5           # include/neuralsim_b200.h NSB_IMP_TABLE_WIDTH, NSB_IMP_MAX_GT
_GT_SLOT = 11


def check_error_map_cfg(error_map_cfg, *, joint=True, enable_after=None):
    """Refuse the error-map options this module does not build.  error_map_cfg: the trainer's `training.error_map` dict; joint: the
    pixel dataset's `joint` (JointFramePixelDataset); enable_after: the trainer's, when given apart from the dict."""
    cfg = dict(error_map_cfg or {})
    if not joint:
        raise RuntimeError("error map: the non-joint PixelDataset (per-frame weights from get_pdf_image) is not built; use pixel_dataset.joint: true")
    if float(cfg.get("frac_mask_err", 0) or 0) > 0:
        raise RuntimeError("error map: frac_mask_err > 0 (the 'mask' error map) is not built")
    if float(cfg.get("frac_on_classnames", 0) or 0) > 0 and cfg.get("on_classnames"):
        raise RuntimeError("error map: the 'focus_on' error maps (frac_on_classnames, on_classnames) are not built")
    ea = cfg.get("enable_after", 0) if enable_after is None else enable_after
    if int(ea or 0) > 0:
        raise RuntimeError("error map: enable_after > 0 (the single-frame uniform warm-up) is not built")
    if "error_map_hw" not in cfg:
        raise RuntimeError("error map: error_map_hw is required")


def split(n, frac_uniform):
    """(n_uniform, n_error_map) of a batch of n rays, as ImpSampler.sample_img_pixel splits it over one map"""
    n_u = int(n * frac_uniform)
    return n_u, n - n_u


def sampler_inc(n, frac_uniform, cap):
    """the generator offsets one draw of n rays advances: randint and rand of the uniform rays, rand of the frames and rand of the pixels"""
    n_u, n_e = split(n, frac_uniform)
    return TR.uniform_inc(n_u, cap) + TR.uniform_inc(2 * n_u, cap) + TR.uniform_inc(n_e, cap) + TR.uniform_inc(2 * n_e, cap)


# ---------------------------------------------------------------------------------------------------------------- the reference's torch ops
@torch.no_grad()
def recipe_update_error_map(error_map, i, xy, val):
    """ErrorMap.update_error_map (importance.py:87-109) on the tensor error_map [N, res_y, res_x], in place (its assert left to the caller)"""
    res_y, res_x = error_map.shape[1], error_map.shape[2]
    x_img, y_img = xy.movedim(-1, 0)
    wf, hf = x_img * res_x, y_img * res_y
    w, h = wf.long(), hf.long()
    w_w, w_h = (wf - w), (hf - h)
    w.clamp_(0, res_x - 2)
    h.clamp_(0, res_y - 2)
    error_map[i, h, w] += (1 - w_h) * (1 - w_w) * val
    error_map[i, h + 1, w] += w_h * (1 - w_w) * val
    error_map[i, h, w + 1] += (1 - w_h) * w_w * val
    error_map[i, h + 1, w + 1] += w_h * w_w * val
    return error_map


@torch.no_grad()
def recipe_construct_cdf(error_map, min_pdf, max_pdf, min_cdfs):
    """ErrorMap.construct_cdf (importance.py:120-142): -> (cdf_x_cond_y, cdf_y, cdf_img); clamps error_map in place when max_pdf is set"""
    min_cdf_x_cond_y, min_cdf_y, min_cdf_img = min_cdfs
    if max_pdf is not None:
        error_map.clamp_max_(max_pdf)
    cdf_x_cond_y = (error_map + 1e-10).cumsum(dim=2)
    cumu = pdf_y = cdf_x_cond_y[:, :, -1]
    cdf_x = (1 - min_pdf) * cdf_x_cond_y / cumu.unsqueeze(-1) + min_pdf * min_cdf_x_cond_y
    cdf_y = pdf_y.cumsum(dim=1)
    cumu = pdf_img = cdf_y[:, -1]
    cdf_y = (1 - min_pdf) * cdf_y / cumu.unsqueeze(-1) + min_pdf * min_cdf_y
    cdf_img = pdf_img.cumsum(dim=0)
    cdf_img = (1 - min_pdf) * cdf_img / cdf_img[-1:] + min_pdf * min_cdf_img
    return cdf_x, cdf_y, cdf_img


@torch.no_grad()
def recipe_sample_pixel(cdf_x_cond_y, cdf_y, num_samples, frame_ind, generator=None):
    """ErrorMap.sample_pixel (importance.py:174-201)"""
    res_y, res_x = cdf_x_cond_y.shape[1], cdf_x_cond_y.shape[2]
    x, y = torch.rand([2, num_samples], dtype=cdf_y.dtype, device=cdf_y.device, generator=generator).clamp_(1e-6, 1 - 1e-6)
    h = torch.searchsorted(cdf_y[frame_ind], y.unsqueeze(-1), right=False).squeeze(-1)
    prev = torch.where(h > 0, cdf_y[frame_ind, h - 1], cdf_y.new_zeros([]))
    y = ((y - prev) / (cdf_y[frame_ind, h] - prev) + h) / res_y
    w = torch.searchsorted(cdf_x_cond_y[frame_ind, h], x.unsqueeze(-1), right=False).squeeze(-1)
    prev = torch.where(w > 0, cdf_x_cond_y[frame_ind, h, w - 1], cdf_x_cond_y.new_zeros([]))
    x = ((x - prev) / (cdf_x_cond_y[frame_ind, h, w] - prev) + w) / res_x
    return torch.stack([x, y], dim=-1)


@torch.no_grad()
def recipe_sample_img(cdf_img, num_samples, generator=None):
    """ErrorMap.sample_img (importance.py:204-216)"""
    i = torch.rand([num_samples], device=cdf_img.device, dtype=cdf_img.dtype, generator=generator).clamp_(1e-6, 1 - 1e-6)
    return torch.searchsorted(cdf_img, i, right=False)


@torch.no_grad()
def recipe_sample_img_pixel(cdfs, n_images, num_samples, frac_uniform, generator=None):
    """ImpSampler.sample_img_pixel (importance.py:317-336) over one error map with cdfs = (cdf_x_cond_y, cdf_y, cdf_img): -> (i, xy)"""
    cdf_x, cdf_y, cdf_img = cdfs
    dev, dt = cdf_img.device, cdf_img.dtype
    n_u, n_e = split(num_samples, frac_uniform)
    i, xy = [], []
    if n_u > 0:
        i.append(torch.randint(n_images, [n_u], dtype=torch.long, device=dev, generator=generator))
        xy.append(torch.rand([n_u, 2], dtype=dt, device=dev, generator=generator).clamp_(1e-6, 1 - 1e-6))
    if n_e > 0:
        fi = recipe_sample_img(cdf_img, n_e, generator)
        i.append(fi)
        xy.append(recipe_sample_pixel(cdf_x, cdf_y, n_e, fi, generator))
    return torch.cat(i, dim=0), torch.cat(xy, dim=0)


@torch.no_grad()
def recipe_pixels(xy, fidx, wh, intr):
    """the pixel (w, h) of each ray and its camera-space direction: (xy * WH).long().clamp_(0, WH - 1) (pixel_loader.py:316,
    cameras.py:301-306), pinhole_lift(w + 0.5, h + 0.5, 1)[..., :3] (pinhole.py:62-74) with intrinsics intr [F, 3, 3].  -> (w, h, dirs)"""
    WH = wh.long().view(1, 2)
    w, h = (WH * xy).long().clamp_(WH.new_zeros([]), WH - 1).movedim(-1, 0)
    u, v = w + 0.5, h + 0.5
    K = intr[fidx]
    fx, fy, cx, cy, sk = K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2], K[..., 0, 1]
    d = torch.ones_like(u)
    x_lift = (u - cx + cy * sk / fy - sk * v / fy) / fx * d
    y_lift = (v - cy) / fy * d
    return w, h, torch.stack((x_lift, y_lift, d), dim=-1)


# ---------------------------------------------------------------------------------------------------------------- kernels
def _gt_arrays(gts):
    n = len(gts)
    rb = (ctypes.c_int64 * max(n, 1))(*[int(t[0].element_size() * t[0][0].numel()) for t in gts])
    outs = (ctypes.c_void_p * max(n, 1))(*[L.ptr(t[0], None, "ground truth").value for t in gts])
    return n, rb, outs


def imp_sample(table, cam, rng, n, n_uniform, res_yx, fidx, xy, *, pidx=None, dirs=None, gts=(), appear=None, rng_next=None):
    """nsb_imp_sample.  gts: [(out [n, ...],)] in the table's gt order; appear = (appear_table [*, A], h_appear [n, A]) or None"""
    P = L.ptr
    n_gt, rb, outs = _gt_arrays(gts)
    at, ha = appear if appear is not None else (None, None)
    L.check(L.lib().nsb_imp_sample(P(table, "i64", "table"), P(cam, "i64", "cam"), P(rng, "i64", "rng"), L.c_i64(n), L.c_i64(n_uniform), L.c_i32(res_yx[0]),
                                   L.c_i32(res_yx[1]), L.c_i32(n_gt), rb, outs, P(at, "f32", "appear_table", allow_none=True),
                                   L.c_i32(at.shape[1] if at is not None else 0), P(ha, "f32", "h_appear", allow_none=True), P(fidx, "i64", "fidx"),
                                   P(xy, "f32", "xy"), P(pidx, "i64", "pidx", allow_none=True), P(dirs, "f32", "dirs", allow_none=True),
                                   P(rng_next, "i64", "rng_next", allow_none=True), L.stream_ptr()), "imp_sample")


def error_map_update(fidx, xy, val, flag, *, error_map=None, last=None, table=None, cam=None, n_images=None, res_yx=None, skip=None):
    """nsb_error_map_update on (error_map, last), or on camera *cam's row of the sampling table (n_images: the largest camera's); skip: a
    device int64 that leaves the map as it is when non-zero"""
    P = L.ptr
    if table is None:
        n_images, res_yx = error_map.shape[0], error_map.shape[1:]
    L.check(L.lib().nsb_error_map_update(P(error_map, "f32", "error_map", allow_none=True), P(last, "i32", "last", allow_none=True), L.c_i64(n_images),
                                         P(table, "i64", "table", allow_none=True), P(cam, "i64", "cam", allow_none=True), L.c_i32(res_yx[0]),
                                         L.c_i32(res_yx[1]), P(fidx, "i64", "fidx"), P(xy, "f32", "xy"), P(val, "f32", "val"), L.c_i64(fidx.shape[0]),
                                         P(flag, "i32", "flag"), P(skip, "i64", "skip", allow_none=True), L.stream_ptr()), "error_map_update")


# ---------------------------------------------------------------------------------------------------------------- modules
class ErrorMap(nn.Module):
    """nr3d_lib.models.importance.ErrorMap with its arguments, methods and persistent state-dict key `error_map`.  The cdf buffers are
    allocated here and rebuilt in place; sample_img_pixel and update_error_map run the kernels (CUDA only)."""

    def __init__(self, n_images, error_map_hw, *, min_pdf=0.01, max_pdf=None, n_steps_init=128, n_steps_max=None, n_steps_growth_factor=1.5,
                 dtype=torch.float, device=None):
        super().__init__()
        if dtype != torch.float32:
            raise RuntimeError(f"ErrorMap: dtype {dtype} is not built (float32 only)")
        n_images = int(n_images)
        if n_images < 1:
            raise RuntimeError(f"ErrorMap: n_images must be >= 1, got {n_images}")
        if len(error_map_hw) != 2 or min(int(v) for v in error_map_hw) < 2:
            raise RuntimeError(f"ErrorMap: error_map_hw must be two sizes >= 2, got {error_map_hw}")
        res_y, res_x = int(error_map_hw[0]), int(error_map_hw[1])
        self.dtype = dtype
        self.n_images, self.res_y, self.res_x = n_images, res_y, res_x
        self.register_buffer("error_map", torch.zeros([n_images, res_y, res_x], device=device, dtype=dtype), persistent=True)
        self.min_pdf, self.max_pdf = min_pdf, max_pdf
        self.register_buffer("min_cdf_x_cond_y", torch.arange(res_x, dtype=dtype, device=device).add_(1).div_(res_x).tile(n_images, res_y, 1), persistent=False)
        self.register_buffer("min_cdf_y", torch.arange(res_y, dtype=dtype, device=device).add_(1).div_(res_y).tile(n_images, 1), persistent=False)
        self.register_buffer("min_cdf_img", torch.arange(n_images, dtype=dtype, device=device).add_(1).div_(n_images), persistent=False)
        # the cdfs the kernels read, rebuilt in place (the reference assigns new tensors); `cdf_built` replaces its `cdf_img is None`
        self.register_buffer("cdf_x_cond_y", torch.zeros([n_images, res_y, res_x], dtype=dtype, device=device), persistent=False)
        self.register_buffer("cdf_y", torch.zeros([n_images, res_y], dtype=dtype, device=device), persistent=False)
        self.register_buffer("cdf_img", torch.zeros([n_images], dtype=dtype, device=device), persistent=False)
        self.register_buffer("last", torch.full([4, n_images, res_y, res_x], -1, dtype=torch.int32, device=device), persistent=False)
        self.register_buffer("flag", torch.zeros([1], dtype=torch.int32, device=device), persistent=False)
        self.cdf_built = False
        self.n_steps_since_update = 0
        self.n_steps_growth_factor = n_steps_growth_factor
        self.n_steps_between_update = n_steps_init
        self.n_steps_max = n_steps_max
        self._table = None

    @property
    def device(self):
        return self.error_map.device

    def _check_batch(self, i, xy, val):
        n = xy.shape[0] if isinstance(xy, torch.Tensor) and xy.dim() == 2 else -1
        if n < 0 or xy.shape[1] != 2 or xy.dtype != torch.float32:
            raise RuntimeError(f"ErrorMap: xy must be a float32 tensor [n, 2], got {getattr(xy, 'dtype', type(xy))} {tuple(getattr(xy, 'shape', ()))}")
        if isinstance(i, Number):
            i = torch.full([n], int(i), dtype=torch.long, device=xy.device)
        if not isinstance(i, torch.Tensor) or i.dtype != torch.long or tuple(i.shape) != (n,):
            raise RuntimeError(f"ErrorMap: i must be an int or an int64 tensor [{n}]")
        if not isinstance(val, torch.Tensor) or tuple(val.shape) != (n,) or val.dtype != torch.float32:
            raise RuntimeError(f"ErrorMap: val must be a float32 tensor [{n}], got {getattr(val, 'dtype', type(val))} {tuple(getattr(val, 'shape', ()))}")
        if n and (int(i.min()) < 0 or int(i.max()) >= self.n_images):
            raise RuntimeError(f"ErrorMap: frame indices out of [0, {self.n_images})")
        return i.contiguous(), xy.contiguous(), val.contiguous()

    @torch.no_grad()
    def update_error_map(self, i, xy, val):
        """the bilinear 4-corner update (importance.py:87-109) on the kernels; a negative val raises, as the reference's assert does"""
        i, xy, val = self._check_batch(i, xy, val)
        if bool((val < 0).any()):
            raise RuntimeError("ErrorMap.update_error_map: found a negative error; only non-negative errors may be accumulated")
        error_map_update(i, xy, val, self.flag, error_map=self.error_map, last=self.last)

    @torch.no_grad()
    def get_normalized_error_map(self, frame_ind=None):
        error_map = self.error_map[frame_ind] if frame_ind is not None else self.error_map
        if self.max_pdf is not None:
            return error_map.clone().clamp_max_(self.max_pdf)
        return error_map / error_map.max().clamp_min(1e-5)

    @torch.no_grad()
    def construct_cdf(self):
        """the reference's torch ops (cold: every >= 128 steps), written into the buffers the kernels read"""
        cdfs = recipe_construct_cdf(self.error_map, self.min_pdf, self.max_pdf, (self.min_cdf_x_cond_y, self.min_cdf_y, self.min_cdf_img))
        for dst, src in zip((self.cdf_x_cond_y, self.cdf_y, self.cdf_img), cdfs):
            dst.copy_(src)
        self.cdf_built = True

    @torch.no_grad()
    def construct_cdf_and_clean_error_map(self):
        self.construct_cdf()
        self.error_map.zero_()

    def count_step(self):
        """the host schedule of step_error_map (importance.py:154-160): -> True when this step rebuilt the cdfs"""
        self.n_steps_since_update += 1
        if self.n_steps_since_update >= self.n_steps_between_update:
            self.construct_cdf_and_clean_error_map()
            self.n_steps_since_update = 0
            self.n_steps_between_update = int(self.n_steps_growth_factor * self.n_steps_between_update)
            if self.n_steps_max is not None:
                self.n_steps_between_update = min(self.n_steps_between_update, self.n_steps_max)
            return True
        return False

    @torch.no_grad()
    def step_error_map(self, i, xy, val):
        self.update_error_map(i=i, xy=xy, val=val)
        self.count_step()

    @torch.no_grad()
    def get_pdf_image(self):
        cdf_img = self.cdf_img
        return cdf_img.diff(prepend=cdf_img.new_zeros([1]))

    def _require_cdf(self):
        if not self.cdf_built:
            raise RuntimeError("ErrorMap: construct_cdf() has not run yet")

    @torch.no_grad()
    def sample_pixel(self, num_samples, frame_ind, generator=None):
        self._require_cdf()
        return recipe_sample_pixel(self.cdf_x_cond_y, self.cdf_y, num_samples, frame_ind, generator)

    @torch.no_grad()
    def sample_img(self, num_samples, generator=None):
        self._require_cdf()
        return recipe_sample_img(self.cdf_img, num_samples, generator)

    def table_row(self):
        """this map's row of a sampling table (no camera)"""
        row = [0] * TABLE_WIDTH
        row[0], row[1], row[2] = self.cdf_img.data_ptr(), self.cdf_y.data_ptr(), self.cdf_x_cond_y.data_ptr()
        row[4], row[5], row[6] = self.n_images, 1, 1
        row[9], row[10] = self.error_map.data_ptr(), self.last.data_ptr()
        return row

    def _draw(self, num_samples, frac_uniform, generator):
        self._require_cdf()
        n = int(num_samples)
        if n < 1:
            raise RuntimeError(f"sample_img_pixel: num_samples must be >= 1, got {n}")
        dev = self.device
        if self._table is None:
            self._table = (torch.tensor([self.table_row()], dtype=torch.int64).to(dev), torch.zeros((), dtype=torch.int64, device=dev))
        rng = TR.take(TR.cuda_generator(generator, dev), sampler_inc(n, frac_uniform, TR.grid_cap(dev)))
        fidx = torch.empty(n, dtype=torch.int64, device=dev)
        xy = torch.empty(n, 2, dtype=torch.float32, device=dev)
        imp_sample(self._table[0], self._table[1], rng, n, split(n, frac_uniform)[0], (self.res_y, self.res_x), fidx, xy)
        return fidx, xy

    @torch.no_grad()
    def sample_img_pixel(self, num_samples, generator=None):
        """(frame indices [n], xy [n, 2]) from torch's CUDA generator (`generator`, else the default one), on the kernel"""
        return self._draw(num_samples, 0.0, generator)


class ImpSampler(nn.Module):
    """nr3d_lib.models.importance.ImpSampler over ONE error map (the shipped configs' 'rgb' map): error_maps = {name: (ErrorMap, frac)}."""

    def __init__(self, error_maps, frac_uniform=0.5):
        super().__init__()
        if len(error_maps) != 1:
            raise RuntimeError(f"ImpSampler: exactly one error map is built (the 'rgb' map), got {list(error_maps)}; "
                               "the 'mask' (frac_mask_err > 0) and 'focus_on' maps are not")
        if not 0.0 <= float(frac_uniform) <= 1.0:
            raise RuntimeError(f"ImpSampler: frac_uniform must lie in [0, 1], got {frac_uniform}")
        names = list(error_maps.keys())
        maps = [v[0] for v in error_maps.values()]
        fracs = [v[1] for v in error_maps.values()]
        for m in maps:
            if not isinstance(m, ErrorMap):
                raise RuntimeError(f"ImpSampler: the error maps must be neuralsim_b200.importance.ErrorMap, got {type(m)}")
            if not m.cdf_built:
                m.construct_cdf()
        self.error_maps = nn.ModuleDict(dict(zip(names, maps)))
        self.n_images = maps[0].n_images
        nu = np.array(fracs)
        self.error_map_fracs = ((1 - frac_uniform) * nu / nu.sum()).tolist()
        self.frac_uniform = frac_uniform
        self.error_map_names = names

    @property
    def device(self):
        return self.error_maps[self.error_map_names[0]].device

    @property
    def dtype(self):
        return self.error_maps[self.error_map_names[0]].dtype

    @property
    def error_map(self) -> ErrorMap:
        return self.error_maps[self.error_map_names[0]]

    @torch.no_grad()
    def get_pdf_image(self):
        pdf = []
        if self.frac_uniform > 0:
            pdf.append(self.frac_uniform * torch.full((self.n_images,), 1. / self.n_images, dtype=self.dtype, device=self.device))
        for frac, m in zip(self.error_map_fracs, self.error_maps.values()):
            pdf.append(frac * m.get_pdf_image())
        return torch.stack(pdf, 0).sum(0)

    @torch.no_grad()
    def sample_img(self, num_samples, generator=None):
        n_u, n_e = split(num_samples, self.frac_uniform)
        i = []
        if n_u > 0:
            i.append(torch.randint(self.n_images, [n_u], dtype=torch.long, device=self.device, generator=generator))
        if n_e > 0:
            i.append(self.error_map.sample_img(n_e, generator))
        return torch.cat(i, dim=0)

    @torch.no_grad()
    def sample_pixel(self, num_samples, frame_ind, generator=None):
        if not isinstance(frame_ind, Number):
            raise RuntimeError("ImpSampler.sample_pixel: frame_ind must be a single frame index")
        n_u, n_e = split(num_samples, self.frac_uniform)
        xy = []
        if n_u > 0:
            xy.append(torch.rand([n_u, 2], dtype=self.dtype, device=self.device, generator=generator).clamp_(1e-6, 1 - 1e-6))
        if n_e > 0:
            xy.append(self.error_map.sample_pixel(n_e, frame_ind, generator))
        return torch.cat(xy, dim=0)

    @torch.no_grad()
    def sample_img_pixel(self, num_samples, generator=None):
        """(frame indices [n], xy [n, 2]): the reference's split and draws, on the kernel"""
        return self.error_map._draw(num_samples, self.frac_uniform, generator)


class CameraSampler:
    """The batch source of StaticFrame(sampler=...): per camera k an ImpSampler, the ground-truth image stacks gts[k] = {key: [F_k, H_k,
    W_k, ...] device tensor} (float32 `image_rgb`, bool / uint8 masks; the same keys, dtypes and trailing shapes for every camera), the
    intrinsics intrs[k] [F_k, 3, 3] (float32), and the bases of its frames in the pose list (CameraPoses) and in the appearance-code table.
    `frame.step(cam=k)` draws camera k's batch inside the graph, as ImpSampler.sample_img_pixel does over its error map, and updates that
    map; one capture serves every camera.  `frame.d_h_appear` keeps its meaning: a trainer scatters it by `frame.rays_fidx`."""

    def __init__(self, samplers, gts, intrs, wh, pose_bases, appear_bases=None, appear_table=None):
        k = len(samplers)
        if k < 1 or not (len(gts) == len(intrs) == len(wh) == len(pose_bases) == k) or (appear_bases is not None and len(appear_bases) != k):
            raise RuntimeError("CameraSampler: samplers, gts, intrs, wh, pose_bases (and appear_bases) need one entry per camera")
        s0 = samplers[0]
        self.samplers = list(samplers)
        self.frac_uniform = s0.frac_uniform
        self.res_yx = (s0.error_map.res_y, s0.error_map.res_x)
        self.device = s0.device
        keys = list(gts[0].keys())
        if len(keys) > MAX_GT:
            raise RuntimeError(f"CameraSampler: at most {MAX_GT} ground-truth keys, got {keys}")
        self.gt_keys = keys
        self.gt_spec = {key: (gts[0][key].dtype, tuple(gts[0][key].shape[3:])) for key in keys}
        self.appear_table = appear_table
        if appear_table is not None and (appear_table.dtype != torch.float32 or appear_table.dim() != 2 or appear_bases is None):
            raise RuntimeError("CameraSampler: appear_table must be a float32 [n_codes, n_appear] tensor, with appear_bases")
        rows = []
        for c, s in enumerate(samplers):
            if not isinstance(s, ImpSampler):
                raise RuntimeError(f"CameraSampler: camera {c}: not an ImpSampler")
            m = s.error_map
            if s.frac_uniform != self.frac_uniform or (m.res_y, m.res_x) != self.res_yx or m.device != self.device:
                raise RuntimeError(f"CameraSampler: camera {c}: frac_uniform, error_map_hw and device must be the cameras' common ones")
            F = m.n_images
            W, H = int(wh[c][0]), int(wh[c][1])
            if list(gts[c].keys()) != keys:
                raise RuntimeError(f"CameraSampler: camera {c}: ground-truth keys {list(gts[c].keys())}, camera 0 has {keys}")
            for key, t in gts[c].items():
                dt, tail = self.gt_spec[key]
                if (not isinstance(t, torch.Tensor) or t.device != self.device or not t.is_contiguous() or tuple(t.shape[:3]) != (F, H, W)
                        or t.dtype != dt or tuple(t.shape[3:]) != tail):
                    raise RuntimeError(f"CameraSampler: camera {c}: {key} must be a contiguous {dt} tensor [{F}, {H}, {W}, *{tail}] on {self.device}, "
                                       f"got {getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
            K = intrs[c]
            if not isinstance(K, torch.Tensor) or K.dtype != torch.float32 or tuple(K.shape) != (F, 3, 3) or K.device != self.device or not K.is_contiguous():
                raise RuntimeError(f"CameraSampler: camera {c}: intrinsics must be a contiguous float32 tensor [{F}, 3, 3] on {self.device}")
            row = m.table_row()
            row[3], row[5], row[6], row[7] = K.data_ptr(), W, H, int(pose_bases[c])
            row[8] = int(appear_bases[c]) if appear_bases is not None else 0
            if appear_table is not None and (row[8] < 0 or row[8] + F > appear_table.shape[0]):
                raise RuntimeError(f"CameraSampler: camera {c}: codes [{row[8]}, {row[8] + F}) outside the table of {appear_table.shape[0]}")
            for j, key in enumerate(keys):
                row[_GT_SLOT + j] = gts[c][key].data_ptr()
            rows.append(row)
        self.gts, self.intrs = gts, intrs                  # the table points into them
        self.pose_end = max(int(pose_bases[c]) + s.n_images for c, s in enumerate(samplers))
        self.max_images = max(s.n_images for s in samplers)
        self.table = torch.tensor(rows, dtype=torch.int64).to(self.device)

    @property
    def n_cameras(self):
        return len(self.samplers)

    def inc(self, n, cap):
        return sampler_inc(n, self.frac_uniform, cap)

    def sample(self, cam, rng, n, fidx, xy, pidx, dirs, gts, h_appear, rng_next):
        """the draw of camera *cam (a device scalar) into the given buffers (nsb_imp_sample)"""
        imp_sample(self.table, cam, rng, n, split(n, self.frac_uniform)[0], self.res_yx, fidx, xy, pidx=pidx, dirs=dirs,
                   gts=[(gts[k],) for k in self.gt_keys], appear=(self.appear_table, h_appear) if h_appear is not None else None, rng_next=rng_next)

    def update(self, cam, fidx, xy, err, flag, skip=None):
        """camera *cam's error map += the batch's errors (nsb_error_map_update from the table)"""
        error_map_update(fidx, xy, err, flag, table=self.table, cam=cam, n_images=self.max_images, res_yx=self.res_yx, skip=skip)

    # -- the batch source of a StaticFrame: every per-frame buffer lives on the frame, so one sampler serves several frames
    def attach(self, frame):
        """check the frame, give it `cam` (a device index), `rays_fidx`, `rays_pix`, `ground_truth`, `err_flag`.  -> the draw's reservation"""
        if frame.pose is None:
            raise RuntimeError("StaticFrame(sampler=...): needs pose= (CameraPoses: the sampled rays are pose indices and camera-space directions)")
        if self.pose_end > frame.pose.n_poses:
            raise RuntimeError(f"StaticFrame(sampler=...): the cameras' frames reach pose {self.pose_end - 1}, the pose list holds {frame.pose.n_poses}")
        if self.appear_table is not None and (frame.h_appear is None or self.appear_table.shape[1] != frame.h_appear.shape[1]):
            raise RuntimeError("StaticFrame(sampler=...): the sampler's appearance codes do not match the model's code width")
        dev, n = frame.device, frame.n_rays
        frame.cam = torch.zeros((), dtype=torch.int64, device=dev)
        frame.rays_fidx = torch.zeros(n, dtype=torch.int64, device=dev)
        frame.rays_pix = torch.zeros(n, 2, device=dev)
        frame.ground_truth = {k: torch.zeros((n,) + tail, dtype=dt, device=dev) for k, (dt, tail) in self.gt_spec.items()}
        frame.err_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        return self.inc(n, TR.grid_cap(dev))

    def select(self, frame, cam, frame_ind, rays):
        """frame.step(cam=k), which takes no frame_ind or rays: k into frame.cam.  -> camera k's ErrorMap.count_step, run after the step"""
        if frame_ind is not None or any(v is not None for v in rays):
            raise RuntimeError("StaticFrame.step: a frame with sampler= draws its own batch; pass cam= only")
        if isinstance(cam, bool) or not isinstance(cam, int) or not 0 <= cam < self.n_cameras:
            raise RuntimeError(f"StaticFrame.step: cam must be an int in [0, {self.n_cameras}), got {cam!r}")
        frame.cam.fill_(cam)
        return self.samplers[cam].error_map.count_step

    def draw(self, frame, rng):
        """camera frame.cam's batch, drawn at the device block rng: `rays_fidx`, `rays_pix`, `ground_truth`, `pidx`, `dirs`, codes"""
        self.sample(frame.cam, rng, frame.n_rays, frame.rays_fidx, frame.rays_pix, frame.pidx, frame.dirs, frame.ground_truth,
                    frame.h_appear if self.appear_table is not None else None, frame.rng)

    def loss(self, frame, arg):
        """loss, err = frame.loss_fn(arg, frame.ground_truth), err [n_rays] the per-ray rgb error the reference feeds its error map.
        -> (loss, what runs after the backward: camera frame.cam's error map += err, unless the device flag `skip` is set)"""
        loss, err = frame.loss_fn(arg, frame.ground_truth)
        if not isinstance(err, torch.Tensor) or err.numel() != frame.n_rays:
            raise RuntimeError(f"StaticFrame(sampler=...): loss_fn must return (loss, err), err holding {frame.n_rays} per-ray errors")
        err = err.detach().reshape(-1).float().contiguous()
        return loss, lambda skip: self.update(frame.cam, frame.rays_fidx, frame.rays_pix, err, frame.err_flag, skip=skip)

    def check(self, frame):
        """raises if loss_fn gave the error map a negative error since the last check (one device-to-host read)"""
        if int(frame.err_flag) != 0:
            frame.err_flag.zero_()
            raise RuntimeError("StaticFrame.check: loss_fn returned a negative per-ray error; the error map accumulates non-negative errors only")
