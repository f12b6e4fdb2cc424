"""Generates tests/golden/ref_pose.npz, camera rays from refined poses and their pose gradient in float64, by EXECUTING THE REFERENCE'S
OWN normalize_quat and quat_apply (nr3d_lib/maths/transforms.py) where a checkout of the reference project is found
(oracle/build_ref.py: reference_root).  The reference is not part of this repository, so the vectors are committed.

    python tests/golden/make_golden_pose.py

transforms.py is imported as `nr3d_lib.maths.transforms` with `nr3d_lib` and `nr3d_lib.maths` registered as *empty* packages whose
__path__ points at the reference tree (no __init__.py runs; its one relative import, maths/common.py, is the reference's own).  The rays
are then composed as the camera observer composes them (app/resources/observers/cameras.py:299-310): rays_d = F.normalize(
quat_apply(normalize_quat(q0 + dq)[pidx], dirs)), rays_o = (t0 + dt)[pidx]; torch float64 autograd gives d_dq, d_dt for the stored
cotangents.  The cases (tests/test_pose_refine.py reads them from the file): quaternions of norm 0.3 and 7, real parts of q0 + dq below
zero, several rays per pose, poses without rays.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_root  # noqa: E402


def import_reference_transforms(ref):
    for name, sub in (("nr3d_lib", ""), ("nr3d_lib.maths", "/maths")):
        m = types.ModuleType(name)
        m.__path__ = [ref + sub]
        sys.modules[name] = m
    return importlib.import_module("nr3d_lib.maths.transforms")


def cases():
    """(q0, dq, t0, dt, pidx, dirs, g_o, g_d) per case, float64, from fixed seeds"""
    out = []
    for seed, (P, n, scale) in enumerate([(6, 40, 0.3), (6, 40, 7.0), (9, 25, 1.0), (1, 13, 2.5)]):
        g = np.random.default_rng(100 + seed)
        q0 = g.normal(size=(P, 4))
        q0 = q0 / np.linalg.norm(q0, axis=1, keepdims=True) * scale
        q0[::2, 0] = -np.abs(q0[::2, 0])                       # real parts below zero
        dq = g.normal(size=(P, 4)) * 0.05 * scale
        t0, dt = g.normal(size=(P, 3)) * 10, g.normal(size=(P, 3)) * 0.1
        used = np.arange(P) if P == 1 else np.arange(0, P, 2) if seed != 2 else np.array([0, 3, 4, 8])     # poses without rays
        pidx = g.choice(used, n)
        dirs = np.stack([g.uniform(-0.5, 0.5, n), g.uniform(-0.35, 0.35, n), np.ones(n)], -1)
        out.append((q0, dq, t0, dt, pidx.astype(np.int64), dirs, g.normal(size=(n, 3)), g.normal(size=(n, 3))))
    return out


def main():
    if reference_root() is None:
        raise SystemExit("make_golden_pose.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
    T = import_reference_transforms(os.path.join(reference_root(), "nr3d_lib", "nr3d_lib"))
    out = {}
    for k, (q0, dq, t0, dt, pidx, dirs, g_o, g_d) in enumerate(cases()):
        tq = torch.from_numpy(dq).requires_grad_(True)
        tt = torch.from_numpy(dt).requires_grad_(True)
        pi = torch.from_numpy(pidx)
        q = T.normalize_quat(torch.from_numpy(q0) + tq)[pi]
        rd = F.normalize(T.quat_apply(q, torch.from_numpy(dirs)), dim=-1)
        ro = (torch.from_numpy(t0) + tt)[pi]
        torch.autograd.backward([ro, rd], [torch.from_numpy(g_o), torch.from_numpy(g_d)])
        for name, v in dict(q0=q0, dq=dq, t0=t0, dt=dt, pidx=pidx, dirs=dirs, g_o=g_o, g_d=g_d, rays_o=ro.detach().numpy(),
                            rays_d=rd.detach().numpy(), d_dq=tq.grad.numpy(), d_dt=tt.grad.numpy()).items():
            out[f"case{k}.{name}"] = v
    path = os.path.join(ROOT, "tests", "golden", "ref_pose.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(cases())} cases, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
