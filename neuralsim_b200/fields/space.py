"""Axis-aligned bounding space -- API of `nr3d_lib.models.spatial.AABBSpace` (reference: models/spatial/aabb.py:20-99)."""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn

from ..graphics.raytest import ray_box_intersection_fast_float_nocheck
from .. import _lib as L


# True: ray_test of fp32 CUDA rays runs as three launches of csrc/neus_glue.cu; False: as the chain of torch ops of the reference
# (aabb.py:71-99) -- same results (tests/test_glue_gpu.py); bench.py's reference-cuda arm switches it off.
FUSED_RAY_TEST = True


class AABBSpace(nn.Module):
    def __init__(self, bounding_size: float = 2.0, aabb=None, dtype=torch.float, device=None):
        super().__init__()
        if aabb is None:
            h = bounding_size / 2.
            aabb = [[-h, -h, -h], [h, h, h]]
        aabb = torch.as_tensor(aabb, dtype=dtype, device=device)
        self.register_buffer("aabb", aabb, persistent=True)
        self.register_buffer("radius3d_original", (aabb[1] - aabb[0]) / 2., persistent=True)

    @property
    def center(self):
        return (self.aabb[1] + self.aabb[0]) / 2.

    @property
    def radius3d(self):
        return (self.aabb[1] - self.aabb[0]) / 2.

    def normalize_coords(self, x):
        return (x - self.center) / self.radius3d

    def unnormalize_coords(self, x):
        return x * self.radius3d + self.center

    def normalize_rays(self, rays_o, rays_d):
        """So that o + d*t lands in [-1,1]^3 for the same depth t (|d| changes)."""
        return (rays_o - self.center) / self.radius3d, rays_d / self.radius3d

    def sample_pts_uniform(self, num_pts: int, generator=None):
        return torch.empty([num_pts, 3], dtype=self.aabb.dtype, device=self.aabb.device).uniform_(-1, 1, generator=generator)

    def ray_test(self, rays_o, rays_d, near=None, far=None, return_rays=True, normalized=False, **extra_ray_data):
        """Slab test against the unit cube -> dict(num_rays, rays_inds, near, far, rays_o, rays_d, **extras) of the hit rays."""
        if (FUSED_RAY_TEST and rays_o.is_cuda and rays_o.dim() == 2 and rays_o.dtype == torch.float32 and rays_d.dtype == torch.float32 and return_rays
                and not rays_o.requires_grad and not rays_d.requires_grad and not isinstance(near, torch.Tensor) and not isinstance(far, torch.Tensor)):
            ret = self._ray_test_fused(rays_o, rays_d, near, far, normalized, extra_ray_data)
            # per-ray data that requires grad (learnable appearance codes) is indexed here, outside the test's no_grad, so autograd reaches it
            ret.update({k: v[ret["rays_inds"]] for k, v in extra_ray_data.items() if isinstance(v, torch.Tensor) and v.requires_grad})
            return ret
        if not normalized:
            rays_o, rays_d = self.normalize_rays(rays_o, rays_d)
        with torch.no_grad():
            near_, far_ = ray_box_intersection_fast_float_nocheck(rays_o, rays_d, -1., 1.)
            if near is not None:
                near_.clamp_min_(near)
            if far is not None:
                far_.clamp_max_(far)
            mask = (far_ > near_) & (far_ > (0 if near is None else near))
            if far is not None:
                mask &= near_ < far
            ridx = mask.nonzero().long()[..., 0]
        ret = dict(num_rays=ridx.shape[0], rays_inds=ridx, near=near_[ridx], far=far_[ridx])
        ret.update({k: (v[ridx] if isinstance(v, torch.Tensor) else v) for k, v in extra_ray_data.items()})
        if return_rays:
            ret.update(rays_o=rays_o[ridx], rays_d=rays_d[ridx])
        return ret

    def _center_radius_c(self):
        """the box's centre and half-size as host float[3] arrays, read back only when the aabb changed"""
        if getattr(self, "_host_cr", None) is None or self._host_cr[0] != (self.aabb.data_ptr(), self.aabb._version):
            c, r = self.center.tolist(), self.radius3d.tolist()
            self._host_cr = ((self.aabb.data_ptr(), self.aabb._version), (ctypes.c_float * 3)(*c), (ctypes.c_float * 3)(*r))
        return self._host_cr[1], self._host_cr[2]

    @torch.no_grad()
    def _ray_test_fused(self, rays_o, rays_d, near, far, normalized, extra_ray_data):
        """The same test as below in three launches and one host read (csrc/neus_glue.cu: k_ray_test_aabb, k_scan_counts, k_gather_rays)."""
        from ..graphics import neus_fused as NF
        R, dev = rays_o.shape[0], rays_o.device
        if normalized:
            c3, r3 = (ctypes.c_float * 3)(0., 0., 0.), (ctypes.c_float * 3)(1., 1., 1.)
        else:
            c3, r3 = self._center_radius_c()
        pairs = torch.zeros(2, dtype=torch.int64, device=dev)              # coherent neighbour pairs, image row length
        tested = NF.ray_test_aabb(rays_o, rays_d, c3, r3, near, far, L.ptr(pairs), L.ptr(pairs[1:]))
        sc = NF.scan_counts(tested[4], want_index=True, extra=pairs)
        n, ridx = sc["n_nonzero"], sc["index"]
        o_c, d_c = torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev)
        n_c, f_c = torch.empty(n, device=dev), torch.empty(n, device=dev)
        # one per-ray fp32 payload (rays_h_appear) rides along in the gather kernel; anything else is indexed by torch
        fused_key = next((k for k, v in extra_ray_data.items() if isinstance(v, torch.Tensor) and v.is_cuda and v.dtype == torch.float32 and v.dim() == 2
                          and v.shape[0] == R and v.is_contiguous() and not v.requires_grad), None)
        ex = extra_ray_data[fused_key] if fused_key is not None else None
        ex_c = torch.empty(n, ex.shape[1], device=dev) if ex is not None else None
        NF.gather_rays(ridx, n, tested[:4], (o_c, d_c, n_c, f_c), ex, ex_c)
        ret = dict(num_rays=n, rays_inds=ridx, near=n_c, far=f_c)
        ret.update({k: (ex_c if k == fused_key else (v[ridx] if isinstance(v, torch.Tensor) else v)) for k, v in extra_ray_data.items()
                    if not (isinstance(v, torch.Tensor) and v.requires_grad)})                # those: ray_test, with grad
        ret.update(rays_o=o_c, rays_d=d_c)
        # image-ordered rays (>= 3/4 of the rays neighbour their predecessor): the queries traverse samples ray-tiled (csrc/fused_tc.cu)
        ret["rays_coherent"] = R > 64 and sc["extra"][0] >= 0.75 * (R - 1)
        if ret["rays_coherent"]:                       # what the queries need to walk the rays in 8 x 4 pixel blocks (graphics/neus.py)
            ret["rays_row"] = (R, pairs)
        return ret
