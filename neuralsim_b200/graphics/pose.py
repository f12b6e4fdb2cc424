"""Refined camera poses: world rays from per-ray pose indices, and the pose gradient, on the project's kernels (csrc/pose.cu).

StreetSurf refines the camera poses with LearnableParams(refine_ego_motion={class_name: Camera}) (app/models/scene/learnable_params.py:
85-113): each camera node's per-frame transform becomes TransformRT(rot=RotationQuaternionRefinedAdd(q0, dq), trans=
TranslationRefinedAdd(t0, dt)) with learnable zero-initialised deltas.  `CameraPoses` holds those poses flattened over (camera node,
frame): q0, dq [P, 4] (real part first), t0, dt [P, 3].  A ray is the pose index pidx (into the P poses) and the camera-space direction
(intrs.lift(...) of its pixel, a constant: intrinsics are not refined), and

    rays_o = t0 + dt,    rays_d = normalize(quat_apply(normalize_quat(q0 + dq), dirs))

in the reference's fp32 operation order (app/resources/observers/cameras.py:299-310).  `pose_rays` is the differentiable op; the
one-launch step (`StaticFrame(..., pose=...)`) runs the same two kernels inside its graph through a `FramePose`, so both give the same bits.
"""
from __future__ import annotations

import torch

from .. import _lib as L

__all__ = ["CameraPoses", "PoseRays", "pose_rays", "FramePose", "check_pose_cfg", "check_pidx", "pose_forward", "pose_backward"]

_UNSUPPORTED_ROT = ("RotationAxisAngle", "Rotation6D", "RotationMat3x3")


def check_pose_cfg(cfg):
    """Refuse the LearnableParams options this op does not build: refined intrinsics / extrinsics (refine_camera_intr,
    refine_camera_extr: the camera-space directions are constants here) and other motion (refine_other_motion)."""
    for k in ("refine_camera_intr", "refine_camera_extr", "refine_other_motion"):
        if cfg.get(k):
            raise RuntimeError(f"CameraPoses: {k} is not built (only refine_ego_motion of camera nodes: quaternion + translation deltas)")
    ego = cfg.get("refine_ego_motion")
    if ego and ego.get("class_name", "Camera") != "Camera":
        raise RuntimeError(f"CameraPoses: refine_ego_motion of {ego.get('class_name')!r} nodes is not built (camera nodes only)")


class CameraPoses(torch.nn.Module):
    """P refined camera poses: q0 [P, 4], t0 [P, 3] (buffers) and the learnable deltas dq [P, 4], dt [P, 3] (zeros).

    `rotation` names the reference's rotation class; only "RotationQuaternion" is built.  `cfg` (optional): the LearnableParams
    config, checked by check_pose_cfg."""

    def __init__(self, q0, t0, *, rotation="RotationQuaternion", cfg=None):
        super().__init__()
        if rotation != "RotationQuaternion":
            raise RuntimeError(f"CameraPoses: rotation {rotation!r} is not built (RotationQuaternion only; "
                               f"{', '.join(_UNSUPPORTED_ROT)} are refused)")
        if cfg is not None:
            check_pose_cfg(cfg)
        q0, t0 = torch.as_tensor(q0, dtype=torch.float32), torch.as_tensor(t0, dtype=torch.float32)
        if q0.dim() != 2 or q0.shape[1] != 4 or t0.shape != (q0.shape[0], 3):
            raise RuntimeError(f"CameraPoses: q0 must be [P, 4] and t0 [P, 3], got {tuple(q0.shape)} and {tuple(t0.shape)}")
        self.register_buffer("q0", q0.contiguous())
        self.register_buffer("t0", t0.contiguous())
        self.dq = torch.nn.Parameter(torch.zeros_like(self.q0))
        self.dt = torch.nn.Parameter(torch.zeros_like(self.t0))

    @property
    def n_poses(self):
        return self.q0.shape[0]

    @property
    def requires_grad(self):
        return self.dq.requires_grad or self.dt.requires_grad


def _check_f32(t, shape, name):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"pose_rays: {name} must be a float32 tensor of shape {tuple(shape)}, got "
                           f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
    if not t.is_cuda or not t.is_contiguous():
        raise RuntimeError(f"pose_rays: {name} must be a contiguous CUDA tensor")


def check_pidx(pidx, n_rays, n_poses):
    """the pose indices of n_rays rays: int64 [n_rays], contiguous, on the device, every index in [0, n_poses) (one host read)"""
    if not isinstance(pidx, torch.Tensor) or pidx.dtype != torch.int64 or tuple(pidx.shape) != (n_rays,):
        raise RuntimeError(f"pose_rays: pidx must be an int64 tensor of shape ({n_rays},), got {getattr(pidx, 'dtype', type(pidx))} "
                           f"{tuple(getattr(pidx, 'shape', ()))}")
    if n_rays:
        lo, hi = torch.aminmax(pidx)
        lo, hi = int(lo), int(hi)
        if lo < 0 or hi >= n_poses:
            raise RuntimeError(f"pose_rays: pidx out of range: indices span [{lo}, {hi}], the poses [0, {n_poses})")
    if not pidx.is_cuda or not pidx.is_contiguous():
        raise RuntimeError("pose_rays: pidx must be a contiguous CUDA tensor")


def pose_forward(poses, pidx, dirs, unit, nrm, rays_o, rays_d, count=None):
    """nsb_pose_rays into the given buffers (unit [P, 4], nrm [P], rays [n, 3]); count = (cnt, k): the rays below the device count"""
    P = L.ptr
    L.call(L.lib().nsb_pose_rays, "pose_rays", P(poses.q0, "f32", "q0"), P(poses.dq, "f32", "dq"), P(poses.t0, "f32", "t0"), P(poses.dt, "f32", "dt"),
           L.c_i64(poses.n_poses), P(pidx, "i64", "pidx"), P(dirs, "f32", "dirs"), L.c_i64(dirs.shape[0]), P(unit, "f32", "unit"), P(nrm, "f32", "nrm"),
           P(rays_o, "f32", "rays_o"), P(rays_d, "f32", "rays_d"), L.stream_ptr(), count=count)


def scratch_floats(n, n_poses):
    return int(L.lib().nsb_pose_grad_scratch_floats(L.c_i64(n), L.c_i64(n_poses)))


def pose_backward(unit, nrm, pidx, dirs, d_rays_o, d_rays_d, scratch, d_dq, d_dt, count=None):
    """nsb_pose_rays_backward: ADDS the pose gradient into d_dq [P, 4] / d_dt [P, 3] (None: not written)"""
    P = L.ptr
    L.call(L.lib().nsb_pose_rays_backward, "pose_rays_backward", P(unit, "f32", "unit"), P(nrm, "f32", "nrm"), L.c_i64(unit.shape[0]),
           P(pidx, "i64", "pidx"), P(dirs, "f32", "dirs"), L.c_i64(dirs.shape[0]), P(d_rays_o, "f32", "d_rays_o"), P(d_rays_d, "f32", "d_rays_d"),
           P(scratch, "f32", "scratch"), P(d_dq, "f32", "d_dq", allow_none=True), P(d_dt, "f32", "d_dt", allow_none=True), L.stream_ptr(), count=count)


class PoseRays(torch.autograd.Function):
    """(pidx, dirs, q0, dq, t0, dt) -> (rays_o, rays_d); the backward is nsb_pose_rays_backward onto zeros -- the gradient the graph
    step adds into dq.grad / dt.grad, bit for bit"""

    @staticmethod
    def forward(ctx, poses, pidx, dirs, dq, dt):
        n, dev = dirs.shape[0], dirs.device
        unit = torch.empty(poses.n_poses, 4, device=dev)
        nrm = torch.empty(poses.n_poses, device=dev)
        rays = torch.empty(2, n, 3, device=dev)
        pose_forward(poses, pidx, dirs, unit, nrm, rays[0], rays[1])
        ctx.save_for_backward(unit, nrm, pidx, dirs)
        ctx.need = (dq.requires_grad, dt.requires_grad)
        return rays[0], rays[1]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_o, g_d):
        unit, nrm, pidx, dirs = ctx.saved_tensors
        dev, n = dirs.device, dirs.shape[0]
        g_o = torch.zeros(n, 3, device=dev) if g_o is None else g_o.contiguous()
        g_d = torch.zeros(n, 3, device=dev) if g_d is None else g_d.contiguous()
        d_dq = torch.zeros(unit.shape[0], 4, device=dev) if ctx.need[0] else None
        d_dt = torch.zeros(unit.shape[0], 3, device=dev) if ctx.need[1] else None
        scratch = torch.empty(max(scratch_floats(n, unit.shape[0]), 4), device=dev)
        pose_backward(unit, nrm, pidx, dirs, g_o, g_d, scratch, d_dq, d_dt)
        return None, None, None, d_dq, d_dt


def pose_rays(poses, pidx, dirs):
    """world rays (rays_o, rays_d) [n, 3] of the camera-space directions dirs [n, 3] under poses[pidx]; differentiable in poses.dq,
    poses.dt.  pidx: int64 [n] in [0, P) (checked: one host read)."""
    n = dirs.shape[0] if isinstance(dirs, torch.Tensor) else -1
    _check_f32(dirs, (n, 3), "dirs")
    for name, t, w in (("q0", poses.q0, 4), ("dq", poses.dq, 4), ("t0", poses.t0, 3), ("dt", poses.dt, 3)):
        _check_f32(t, (poses.n_poses, w), name)
    check_pidx(pidx, n, poses.n_poses)
    return PoseRays.apply(poses, pidx, dirs, poses.dq, poses.dt)


class FramePose:
    """The pose's part of a one-launch step (StaticFrame(pose=poses)): the inputs `dirs` [n_rays, 3] (camera-space directions) and `pidx`
    [n_rays] (int64 pose indices), the rays built from them and the pose adjoint, which ADDS into `grads` (bound as dq.grad / dt.grad)."""

    def __init__(self, poses, n_rays, device):
        P, n = poses.n_poses, int(n_rays)
        self.poses, self.n_rays = poses, n
        self.dirs = torch.zeros(n, 3, device=device)
        self.pidx = torch.zeros(n, dtype=torch.int64, device=device)
        self.unit, self.nrm = torch.zeros(P, 4, device=device), torch.zeros(P, device=device)
        self.scratch = torch.zeros(max(scratch_floats(n, P), 4), device=device)
        self.d_rays = torch.zeros(2, n, 3, device=device).unbind(0)           # the rays' gradient when the step keeps none of its own
        self.grads = (torch.zeros(P, 4, device=device), torch.zeros(P, 3, device=device))

    def set_rays(self, dirs, pidx):
        """StaticFrame.set_rays: dirs [n_rays, 3] and pidx [n_rays] (int64 in [0, P), checked: one host read) into the inputs"""
        if not isinstance(dirs, torch.Tensor) or tuple(dirs.shape) != (self.n_rays, 3) or not dirs.is_floating_point():
            raise RuntimeError(f"StaticFrame.set_rays: dirs must be a float tensor [{self.n_rays}, 3], got {getattr(dirs, 'shape', type(dirs))}")
        check_pidx(pidx.to(self.pidx.device) if isinstance(pidx, torch.Tensor) else pidx, self.n_rays, self.poses.n_poses)
        self.dirs.copy_(dirs, non_blocking=True)
        self.pidx.copy_(pidx, non_blocking=True)

    def wants_grad(self):
        return self.poses.requires_grad and torch.is_grad_enabled()

    def bind_grads(self):
        """dq.grad / dt.grad := `grads`, for the deltas that require grad (a None .grad counts as zeros, another tensor is copied in)"""
        for p, buf in zip((self.poses.dq, self.poses.dt), self.grads):
            if not p.requires_grad:
                continue
            if p.grad is None:
                buf.zero_()
            elif p.grad is not buf:
                buf.copy_(p.grad)
            p.grad = buf

    def run(self, rays_o, rays_d, d_rays=None, zero_grads=False):
        """the world rays into rays_o, rays_d [n_rays, 3].  -> (d_rays, None) without grad; with grad (`grads` zeroed first if zero_grads)
        the buffers the rays' gradient goes to (d_rays, else the pose's own) and the hook that adds their pose adjoint into `grads`"""
        grad = self.wants_grad()
        if grad and zero_grads:
            for g in self.grads:
                g.zero_()
        with torch.no_grad():
            pose_forward(self.poses, self.pidx, self.dirs, self.unit, self.nrm, rays_o, rays_d)
        if not grad:
            return d_rays, None
        d = d_rays if d_rays is not None else self.d_rays
        q = self.poses
        return d, lambda: pose_backward(self.unit, self.nrm, self.pidx, self.dirs, d[0], d[1], self.scratch,
                                        self.grads[0] if q.dq.requires_grad else None, self.grads[1] if q.dt.requires_grad else None)
