"""Float64 statement of the pose op (nsb_pose_rays) and its adjoint (nsb_pose_rays_backward), the reference's torch formulation of the
same rays (the recipe a trainer runs without the op), and posed street batches.  TEST INFRASTRUCTURE.

The rays (app/resources/observers/cameras.py:299-310; nr3d_lib/models/attributes/transform.py:107-130; nr3d_lib/maths/transforms.py):
    u = standardize(q / max(|q|, 1e-12)),  q = q0 + dq       r = vec(u (0, v) conj(u))       rays_d = r / max(|r|, 1e-12),  rays_o = t0 + dt
The adjoint, per ray then summed per pose:  d_t = g_o;  d_r = g_d / c - [|r| >= eps] r (g_d . r) / (c^2 |r|);  d_u = -2 (0, d_r) u (0, v);
per pose  d_q = (s_u - u (u . s_u)) / (s |q|)  (s = -1 where the standardisation flipped u; |q| < eps: s_u / (s eps)).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

EPS = 1e-12


def qmul(a, b):
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def _unit(q0, dq):
    q = np.asarray(q0, np.float64) + np.asarray(dq, np.float64)
    n = np.linalg.norm(q, axis=-1)
    u = q / np.maximum(n, EPS)[:, None]
    s = np.where(u[:, 0] < 0, -1.0, 1.0)
    return u * s[:, None], s * n


def _rot(u, v):
    p = np.concatenate([np.zeros(v.shape[:-1] + (1,)), v], -1)
    return qmul(qmul(u, p), u * np.array([1.0, -1.0, -1.0, -1.0]))[..., 1:]


def forward(q0, dq, t0, dt, pidx, dirs):
    """-> rays_o, rays_d [n, 3] in float64"""
    u, _ = _unit(q0, dq)
    r = _rot(u[pidx], np.asarray(dirs, np.float64))
    rd = r / np.maximum(np.linalg.norm(r, axis=-1), EPS)[:, None]
    ro = (np.asarray(t0, np.float64) + np.asarray(dt, np.float64))[pidx]
    return ro, rd


def ray_terms(q0, dq, pidx, dirs, g_d, divide=True):
    """the per-ray cotangents d_u [n, 4] of the unit quaternion (before the per-pose sum); divide=False: a deliberately wrong one
    without the division by the rotated direction's norm"""
    u, _ = _unit(q0, dq)
    v = np.asarray(dirs, np.float64)
    ur = u[pidx]
    r = _rot(ur, v)
    nr = np.linalg.norm(r, axis=-1)
    c = np.maximum(nr, EPS)
    g = np.asarray(g_d, np.float64)
    k = np.where(nr >= EPS, (g * r).sum(-1) / (c * c * nr), 0.0)
    d_r = (g / c[:, None] if divide else g) - r * k[:, None]
    gq = np.concatenate([np.zeros((len(v), 1)), d_r], -1)
    p = np.concatenate([np.zeros((len(v), 1)), v], -1)
    return -2.0 * qmul(qmul(gq, ur), p)


def adjoint(q0, dq, pidx, dirs, g_o, g_d, n_poses):
    """-> d_dq [P, 4], d_dt [P, 3] in float64 (poses without rays: 0)"""
    u, sn = _unit(q0, dq)
    du = ray_terms(q0, dq, pidx, dirs, g_d)
    s_u = np.zeros((n_poses, 4))
    s_t = np.zeros((n_poses, 3))
    np.add.at(s_u, pidx, du)
    np.add.at(s_t, pidx, np.asarray(g_o, np.float64))
    ud = (u * s_u).sum(-1)
    clamped = np.abs(sn) < EPS
    d_q = np.where(clamped[:, None], s_u / np.copysign(EPS, sn)[:, None], (s_u - u * ud[:, None]) / np.where(clamped, 1.0, sn)[:, None])
    return d_q, s_t


def bound_terms(dirs):
    """per ray, the sum of |terms| of the forward's rotated direction relative to its norm: each output of the sandwich adds 16 products
    |u_a u_b v_c| <= |v|_1 (|u_k| <= 1), then the normalisation -> 4 |v|_1 / |v| + 1"""
    v = np.asarray(dirs, np.float64)
    return 4.0 * np.abs(v).sum(-1) / np.linalg.norm(v, axis=-1) + 1.0


# ---------------------------------------------------------------------------------------------------------------- the torch recipe
def torch_pose_rays(q0, dq, t0, dt, pidx, dirs):
    """the reference's own arithmetic as a trainer runs it in torch (differentiable in dq, dt): normalize_quat (F.normalize, then the
    standardisation), quat_apply (two quat_raw_multiply, quat_invert by [1, -1, -1, -1]), F.normalize of the rotated direction, and the
    translation as the origin (transforms.py:41-72, 150-193; transform.py:107-130; cameras.py:299-310)"""
    q = (q0 + dq)[pidx]
    q = F.normalize(q, dim=-1)
    q = torch.where(q[..., 0:1] < 0, -q, q)

    def mul(a, b):
        aw, ax, ay, az = torch.unbind(a, -1)
        bw, bx, by, bz = torch.unbind(b, -1)
        return torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw), -1)
    p = torch.cat((dirs.new_zeros(dirs.shape[:-1] + (1,)), dirs), -1)
    r = mul(mul(q, p), q * torch.tensor([1, -1, -1, -1], device=q.device))[..., 1:]
    return (t0 + dt)[pidx], F.normalize(r, dim=-1)


# ---------------------------------------------------------------------------------------------------------------- posed street batches
def rot_to_quat(R):
    """a unit quaternion (real part first) of a rotation matrix (float64)"""
    w = math.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = math.copysign(math.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2, R[2, 1] - R[1, 2])
    y = math.copysign(math.sqrt(max(0.0, 1.0 - R[0, 0] + R[1, 1] - R[2, 2])) / 2, R[0, 2] - R[2, 0])
    z = math.copysign(math.sqrt(max(0.0, 1.0 - R[0, 0] - R[1, 1] + R[2, 2])) / 2, R[1, 0] - R[0, 1])
    return np.array([w, x, y, z])


def street_poses(n_cams, n_frames, road_z, seed=0, y0=-60.0, dy=12.0):
    """camera-to-world poses of n_cams cameras (yaw offsets) on a car driving along +y, 2 m above the road: q0 [P, 4], t0 [P, 3],
    P = n_cams * n_frames, pose index cam * n_frames + frame.  Camera axes x right, y down, z forward (an OpenCV pinhole)."""
    rng = np.random.default_rng(seed)
    q0, t0 = [], []
    for c in range(n_cams):
        for f in range(n_frames):
            yaw = math.radians((c - (n_cams - 1) / 2) * 40.0 + rng.uniform(-5, 5))
            fwd = np.array([math.sin(yaw), math.cos(yaw), 0.0])
            right = np.array([math.cos(yaw), -math.sin(yaw), 0.0])
            down = np.array([0.0, 0.0, -1.0])
            q0.append(rot_to_quat(np.stack([right, down, fwd], 1)))
            t0.append([rng.uniform(-3, 3), y0 + dy * f, road_z + 2.0])
    return np.array(q0, np.float32), np.array(t0, np.float32)


def street_batch(n, n_poses, seed=0, W=1920, H=1280, focal=2000.0):
    """n random pixels of W x H pinhole cameras over n_poses poses: pose indices (int64, in random order) and the lifted camera-space
    directions (x / f, y / f, 1) of the pixel centres, as intrs.lift returns them"""
    rng = np.random.default_rng(seed)
    pidx = rng.integers(0, n_poses, n)
    i, j = np.floor(rng.uniform(0, W, n)) + 0.5, np.floor(rng.uniform(0, H, n)) + 0.5
    dirs = np.stack([(i - W / 2) / focal, (j - H / 2) / focal, np.ones(n)], -1)
    return pidx.astype(np.int64), dirs.astype(np.float32)
