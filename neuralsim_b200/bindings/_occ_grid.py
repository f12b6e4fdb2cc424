"""Drop-in for `nr3d_lib.bindings._occ_grid` (reference: nr3d_lib/csrc/occ_grid/src/occ_grid.cpp:21-33,
include/occ_grid/cpp_api.h:14-65): ray_marching / batched_ray_marching with AABB contraction."""
from __future__ import annotations

import ctypes
from enum import IntEnum

import torch

from .. import _lib as L


class ContractionType(IntEnum):
    AABB = 0
    UN_BOUNDED_TANH = 1
    UN_BOUNDED_SPHERE = 2


def _march(rays_o, rays_d, t_min, t_max, roi, grid_binary, batch_inds, type, step_size, max_step_size, dt_gamma,
           max_steps, return_gidx, who):
    if int(type) != int(ContractionType.AABB):
        raise RuntimeError(f"{who}: only ContractionType.AABB is built (no shipped config uses tanh/sphere contraction)")
    if grid_binary.dtype != torch.bool:
        raise RuntimeError(f"{who}: grid_binary must be a bool tensor")
    R = rays_o.shape[0]
    dev = rays_o.device
    g = grid_binary.contiguous().view(torch.uint8)
    res = grid_binary.shape[-3:]
    args = (L.c_i64(R), L.ptr(rays_o, "f32", "rays_o"), L.ptr(rays_d, "f32", "rays_d"), L.ptr(t_min, "f32", "t_min"),
            L.ptr(t_max, "f32", "t_max"), L.ptr(roi, "f32", "roi"), L.ptr(batch_inds, "i32", "batch_inds", allow_none=True),
            L.c_i32(res[0]), L.c_i32(res[1]), L.c_i32(res[2]), L.ptr(g, "u8"), L.c_f32(step_size), L.c_f32(max_step_size),
            L.c_f32(dt_gamma), ctypes.c_uint32(int(max_steps)))
    num_steps = torch.empty(R, dtype=torch.int32, device=dev)
    with L.KERNEL_TIMER.time("march", R):
        L.check(L.lib().nsb_ray_marching(*args, None, L.ptr(num_steps), None, None, None, None, None, L.stream_ptr()), who)
    cum = num_steps.cumsum(0, dtype=torch.int32)
    packed_info = torch.stack([cum - num_steps, num_steps], 1).contiguous()
    total = int(cum[-1].item()) if R > 0 else 0          # output size is data dependent: one sync, as the reference
    t_starts = torch.empty((total, 1), dtype=torch.float32, device=dev)
    t_ends = torch.empty((total, 1), dtype=torch.float32, device=dev)
    ridx = torch.empty(total, dtype=torch.int32, device=dev)
    gidx = torch.empty(total, dtype=torch.int32, device=dev) if return_gidx else None
    bidx = torch.empty(total, dtype=torch.int32, device=dev) if batch_inds is not None else None
    if total > 0:
        with L.KERNEL_TIMER.time("march", R):
            L.check(L.lib().nsb_ray_marching(*args, L.ptr(packed_info), None, L.ptr(t_starts), L.ptr(t_ends), L.ptr(ridx),
                                             L.ptr(gidx, allow_none=True), L.ptr(bidx, allow_none=True), L.stream_ptr()), who)
    return packed_info, t_starts, t_ends, ridx, gidx, bidx


def ray_marching(rays_o, rays_d, t_min, t_max, roi, grid_binary, type, step_size, max_step_size, dt_gamma, max_steps,
                 return_gidx):
    """-> [packed_info i32[R,2], t_starts[M,1], t_ends[M,1], ridx i32[M], gidx i32[M]]   (ray_marching.cu:136-244)"""
    if grid_binary.dim() != 3 or roi.numel() != 6:
        raise RuntimeError("ray_marching: expected grid_binary [X,Y,Z] and roi [6]")
    out = _march(rays_o, rays_d, t_min, t_max, roi, grid_binary, None, type, step_size, max_step_size, dt_gamma, max_steps,
                 return_gidx, "ray_marching")
    return list(out[:5])


def batched_ray_marching(rays_o, rays_d, t_min, t_max, batch_inds, batch_data_size, roi, grid_binary, type, step_size,
                         max_step_size, dt_gamma, max_steps, return_gidx):
    """-> [packed_info, t_starts, t_ends, ridx, bidx, gidx]   (batched_marching.cu:154-287)"""
    if grid_binary.dim() != 4:
        raise RuntimeError("batched_ray_marching: expected grid_binary [B,X,Y,Z]")
    if batch_data_size and rays_o.shape[0] % int(batch_data_size) != 0:        # batched_marching.cu:206
        raise RuntimeError(f"batched_ray_marching: Expect nonzero `batch_data_size`={int(batch_data_size)} to be a divisor of "
                           f"`n_rays`={rays_o.shape[0]}")
    if batch_inds is None:
        if not batch_data_size:
            raise RuntimeError("batched_ray_marching: need batch_inds or batch_data_size")
        batch_inds = (torch.arange(rays_o.shape[0], device=rays_o.device) // int(batch_data_size)).int()
    info, t0, t1, ridx, gidx, bidx = _march(rays_o, rays_d, t_min, t_max, roi.contiguous(), grid_binary,
                                            batch_inds.contiguous().int(), type, step_size, max_step_size, dt_gamma, max_steps,
                                            return_gidx, "batched_ray_marching")
    return [info, t0, t1, ridx, bidx, gidx]


def forest_ray_marching(*a, **k):
    """occ_grid.cpp:21-33 `forest_ray_marching(ForestMeta, ...)`: needs the forest block space (`_forest`, kaolin) -- not built (SURVEY §8 a13)"""
    raise RuntimeError("_occ_grid.forest_ray_marching is not built in neuralsim_b200 (forest block spaces, SURVEY.md §8 a13)")
