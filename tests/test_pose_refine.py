"""CPU: the float64 statement of the pose op and its adjoint (tests/pose64.py, what nsb_pose_rays / nsb_pose_rays_backward compute)
pinned to the reference's own normalize_quat and quat_apply, executed (tests/golden/ref_pose.npz, tests/golden/make_golden_pose.py), and
to torch float64 autograd of the restated formula (pose64.torch_pose_rays, the recipe the profile and the GPU tests run); the argument
checks of the Python op, of the frame's pose inputs and of the C entry points (they fail before any launch: no GPU needed)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import pose64

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pose.npz")


def _gold():
    z = np.load(GOLD)
    n = len({k.split(".")[0] for k in z.files})
    return [{k.split(".", 1)[1]: z[k] for k in z.files if k.startswith(f"case{i}.")} for i in range(n)]


def _autograd(c):
    dq = torch.from_numpy(c["dq"]).requires_grad_(True)
    dt = torch.from_numpy(c["dt"]).requires_grad_(True)
    ro, rd = pose64.torch_pose_rays(torch.from_numpy(c["q0"]), dq, torch.from_numpy(c["t0"]), dt, torch.from_numpy(c["pidx"]), torch.from_numpy(c["dirs"]))
    torch.autograd.backward([ro, rd], [torch.from_numpy(c["g_o"]), torch.from_numpy(c["g_d"])])
    return ro.detach().numpy(), rd.detach().numpy(), dq.grad.numpy(), dt.grad.numpy()


def test_cases_cover_the_edges():
    cs = _gold()
    norms = [np.linalg.norm(c["q0"] + c["dq"], axis=1) for c in cs]
    assert any((n < 0.4).all() for n in norms) and any((n > 6).all() for n in norms)
    assert all(((c["q0"] + c["dq"])[:, 0] < 0).any() for c in cs if len(c["q0"]) > 1)
    assert all(np.bincount(c["pidx"]).max() > 1 for c in cs)
    assert sum(len(c["q0"]) - len(np.unique(c["pidx"])) for c in cs) >= 6          # poses without rays


@pytest.mark.parametrize("case", range(4))
def test_statement_matches_executed_reference(case):
    c = _gold()[case]
    ro, rd = pose64.forward(c["q0"], c["dq"], c["t0"], c["dt"], c["pidx"], c["dirs"])
    np.testing.assert_allclose(ro, c["rays_o"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(rd, c["rays_d"], rtol=1e-12, atol=1e-12)
    d_q, d_t = pose64.adjoint(c["q0"], c["dq"], c["pidx"], c["dirs"], c["g_o"], c["g_d"], len(c["q0"]))
    np.testing.assert_allclose(d_q, c["d_dq"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(d_t, c["d_dt"], rtol=1e-12, atol=1e-12)
    unused = np.setdiff1d(np.arange(len(c["q0"])), c["pidx"])
    assert (d_q[unused] == 0).all() and (d_t[unused] == 0).all()


@pytest.mark.parametrize("case", range(4))
def test_torch_recipe_matches_executed_reference(case):
    """the torch restatement the GPU tests and the profile use as the trainer's recipe is the executed reference (float64)"""
    c = _gold()[case]
    ro, rd, d_q, d_t = _autograd(c)
    for got, want in ((ro, "rays_o"), (rd, "rays_d"), (d_q, "d_dq"), (d_t, "d_dt")):
        np.testing.assert_allclose(got, c[want], rtol=1e-12, atol=1e-12)


def test_wrong_adjoints_fail():
    """the comparison can fail: without the standardisation's sign, or without the division by the rotated direction's norm (the
    lifted directions have |v| > 1).  The two projections are not such tests: rays_d does not change with the scale of u (u . s_u = 0),
    and a radial d_r moves no unit quaternion."""
    c = _gold()[0]
    u, sn = pose64._unit(c["q0"], c["dq"])
    du = pose64.ray_terms(c["q0"], c["dq"], c["pidx"], c["dirs"], c["g_d"])
    s_u = np.zeros_like(u)
    np.add.at(s_u, c["pidx"], du)
    no_sign = (s_u - u * (u * s_u).sum(-1, keepdims=True)) / np.abs(sn)[:, None]
    du_np = pose64.ray_terms(c["q0"], c["dq"], c["pidx"], c["dirs"], c["g_d"], divide=False)
    s_np = np.zeros_like(u)
    np.add.at(s_np, c["pidx"], du_np)
    no_div = (s_np - u * (u * s_np).sum(-1, keepdims=True)) / sn[:, None]
    for wrong in (no_sign, no_div):
        assert not np.allclose(wrong, c["d_dq"], rtol=1e-6, atol=1e-9)


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_pose_refusals():
    from neuralsim_b200.graphics.pose import CameraPoses, check_pose_cfg
    for rot in ("RotationAxisAngle", "Rotation6D"):
        with pytest.raises(RuntimeError, match=rot):
            CameraPoses(torch.zeros(2, 4), torch.zeros(2, 3), rotation=rot)
    for k in ("refine_camera_intr", "refine_camera_extr"):
        with pytest.raises(RuntimeError, match=k):
            check_pose_cfg({"refine_ego_motion": {"class_name": "Camera"}, k: {"class_name": "Camera"}})
        with pytest.raises(RuntimeError, match=k):
            CameraPoses(torch.zeros(2, 4), torch.zeros(2, 3), cfg={k: {"lr": 1e-3}})
    check_pose_cfg({"refine_ego_motion": {"class_name": "Camera"}, "refine_camera_intr": None, "refine_camera_extr": None, "enable_after": 500})
    with pytest.raises(RuntimeError, match=r"\[P, 4\]"):
        CameraPoses(torch.zeros(2, 3), torch.zeros(2, 3))


def test_python_op_argument_checks():
    from neuralsim_b200.graphics.pose import CameraPoses, check_pidx, pose_rays
    poses = CameraPoses(torch.tensor([[1.0, 0, 0, 0]] * 3), torch.zeros(3, 3))
    for bad, what in ((torch.tensor([0, 3]), "out of range"), (torch.tensor([-1, 0]), "out of range"),
                      (torch.tensor([0, 1], dtype=torch.int32), "int64"), (torch.tensor([0, 1, 2]), r"shape \(2,\)")):
        with pytest.raises(RuntimeError, match=what):
            check_pidx(bad, 2, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        check_pidx(torch.tensor([0, 2]), 2, 3)
    for dirs, what in ((torch.zeros(2, 3, dtype=torch.float64), "float32"), (torch.zeros(2, 4), "shape"), (torch.zeros(2, 3), "CUDA"),
                       (torch.zeros(3, 2).t(), "CUDA")):
        with pytest.raises(RuntimeError, match=what):
            pose_rays(poses, torch.tensor([0, 1]), dirs)


@pytest.fixture(scope="module")
def lib():
    from neuralsim_b200 import _lib, build
    build.build_library()
    return _lib.lib()


def test_c_entry_argument_checks(lib):
    from neuralsim_b200 import _lib as L
    buf = (ctypes.c_float * 64)()
    ib = (ctypes.c_int64 * 4)()
    f, i, N = ctypes.cast(buf, ctypes.c_void_p), ctypes.cast(ib, ctypes.c_void_p), ctypes.c_void_p(0)
    odd = ctypes.c_void_p(ctypes.addressof(buf) + 4)
    s = L.stream_ptr if False else (lambda: ctypes.c_void_p(0))
    fwd, bwd = lib.nsb_pose_rays, lib.nsb_pose_rays_backward
    I64 = ctypes.c_int64
    for args, what in (((N, f, f, f, I64(2), i, f, I64(4), f, f, f, f), "NULL pose"), ((f, f, f, f, I64(2), N, f, I64(4), f, f, f, f), "NULL ray"),
                       ((f, f, f, f, I64(-1), i, f, I64(4), f, f, f, f), "negative"), ((f, f, f, f, I64(0), i, f, I64(4), f, f, f, f), "at least one pose"),
                       ((f, f, f, f, I64(1 << 31), i, f, I64(4), f, f, f, f), "2\\^31"), ((f, f, f, f, I64(2), i, f, I64(4), odd, f, f, f), "aligned")):
        with pytest.raises(RuntimeError, match=what):
            L.check(fwd(*args, s()), "pose_rays")
    for args, what in (((N, f, I64(2), i, f, I64(4), f, f, f, f, f), "NULL pose"), ((f, f, I64(2), i, f, I64(4), f, N, f, f, f), "NULL ray"),
                       ((f, f, I64(2), i, f, I64(4), f, f, N, f, f), "NULL ray"), ((f, f, I64(2), i, f, I64(-4), f, f, f, f, f), "negative"),
                       ((f, f, I64(2), i, f, I64(4), f, f, odd, f, f), "aligned"), ((f, f, I64(2), i, f, I64(4096 * 65536), f, f, f, f, f), "65535")):
        with pytest.raises(RuntimeError, match=what):
            L.check(bwd(*args, s()), "pose_rays_backward")
    assert lib.nsb_pose_grad_scratch_floats(I64(8192), I64(24)) == 2 * 24 * 8
