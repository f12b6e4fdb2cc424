"""Camera rays from refined poses and the pose gradient (csrc/pose.cu: nsb_pose_rays, nsb_pose_rays_backward; graphics/pose.py;
StaticFrame(pose=...)) on the GPU.

Bounds.  The forward is the reference's fp32 op sequence: bit-equal to that sequence run in torch (tests/pose64.py torch_pose_rays), and
within 32 * 2^-24 * sum|terms| of float64 (pose64.bound_terms: the sandwich's 16 products per output, then the normalisation).  The
adjoint sums each pose's rays in a fixed order (per lane serially, then a butterfly, then the 4096-ray chunks): against float64 per
element within 2^-24 * (64 + n_p / 8) * sum over the pose's rays of |term| (n_p its rays; the lanes' serial sums hold n_p / 32 terms),
the terms scaled by the normalisation's 1 / |q|.  The graph step runs the host-sized path's kernels on the same rays, and its ray
cotangents are the host-sized path's bits (tests/test_graph_ray_grad_gpu.py), so its pose gradient is compared bit for bit; its model
gradients are compared to the order of the fp32 table atomics (ORDER_REL, tests/test_appear_grad_gpu.py).  Against the trainer's torch
recipe (torch pose, ray_grad=True, torch backward), whose index backward sums a pose's rays in another order, the pose gradient is held
to the float64 bound above on both sides."""
import gc
import json

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import pose64
import test_appear_grad_gpu as ag
from util import product_grads, rel_l2

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _poses(q0, t0, dq=None, dt=None, dev="cuda"):
    from neuralsim_b200.graphics.pose import CameraPoses
    p = CameraPoses(torch.as_tensor(q0, dtype=torch.float32), torch.as_tensor(t0, dtype=torch.float32)).to(dev)
    with torch.no_grad():
        if dq is not None:
            p.dq.copy_(torch.as_tensor(dq, dtype=torch.float32))
        if dt is not None:
            p.dt.copy_(torch.as_tensor(dt, dtype=torch.float32))
    return p


def _np(t):
    return t.detach().double().cpu().numpy()


def _random_case(P, n, seed, order="shuffled", used=None):
    g = np.random.default_rng(seed)
    q0 = g.normal(size=(P, 4)) * g.choice([0.3, 1.0, 7.0], size=(P, 1))
    dq, t0, dt = g.normal(size=(P, 4)) * 0.05, g.normal(size=(P, 3)) * 20, g.normal(size=(P, 3)) * 0.1
    pidx = g.choice(np.arange(P) if used is None else used, n)
    if order == "sorted":
        pidx = np.sort(pidx)
    dirs = np.stack([g.uniform(-0.5, 0.5, n), g.uniform(-0.35, 0.35, n), np.ones(n)], -1)
    return _poses(q0, t0, dq, dt), torch.from_numpy(pidx).cuda(), torch.from_numpy(dirs).float().cuda()


def _kernel_grad(poses, pidx, dirs, g_o, g_d, count=None):
    from neuralsim_b200.graphics.pose import pose_backward, pose_forward, scratch_floats
    P, n = poses.n_poses, dirs.shape[0]
    unit, nrm, rays = torch.empty(P, 4, device="cuda"), torch.empty(P, device="cuda"), torch.empty(2, n, 3, device="cuda")
    pose_forward(poses, pidx, dirs, unit, nrm, rays[0], rays[1])
    d_dq, d_dt = torch.zeros(P, 4, device="cuda"), torch.zeros(P, 3, device="cuda")
    scratch = torch.full((max(scratch_floats(n, P), 4),), float("nan"), device="cuda")
    pose_backward(unit, nrm, pidx, dirs, g_o, g_d, scratch, d_dq, d_dt, count=count)
    return d_dq, d_dt


def _check_adjoint(poses, pidx, dirs, g_o, g_d, d_dq, d_dt):
    q0, dq, p, v = _np(poses.q0), _np(poses.dq), pidx.cpu().numpy(), _np(dirs)
    P = q0.shape[0]
    want_q, want_t = pose64.adjoint(q0, dq, p, v, _np(g_o), _np(g_d), P)
    _, sn = pose64._unit(q0, dq)
    du = np.abs(pose64.ray_terms(q0, dq, p, v, _np(g_d))).sum(-1)
    n_p = np.bincount(p, minlength=P)
    a_q, a_t = np.zeros(P), np.zeros(P)
    np.add.at(a_q, p, du)
    np.add.at(a_t, p, np.abs(_np(g_o)).sum(-1))
    c = U * (64 + n_p / 8)
    b_q = 2 * c * a_q / np.maximum(np.abs(sn), 1e-12) + 1e-30          # 2: the normalisation's projection adds one more product per term
    b_t = c * a_t + 1e-30
    r_q = np.abs(_np(d_dq) - want_q).max(-1) / b_q
    r_t = np.abs(_np(d_dt) - want_t).max(-1) / b_t
    assert (r_q <= 1).all() and (r_t <= 1).all(), (float(r_q.max()), float(r_t.max()))
    none = n_p == 0
    assert (_np(d_dq)[none] == 0).all() and (_np(d_dt)[none] == 0).all()
    return float(max(r_q.max(), r_t.max()))


# ===================================================================================================================== kernels
@pytest.mark.parametrize("case", range(4))
def test_forward_matches_float64_and_the_torch_recipe(case):
    z = np.load(pose64.__file__.replace("pose64.py", "golden/ref_pose.npz"))
    c = {k.split(".", 1)[1]: z[k] for k in z.files if k.startswith(f"case{case}.")}
    poses = _poses(c["q0"], c["t0"], c["dq"], c["dt"])
    pidx, dirs = torch.from_numpy(c["pidx"]).cuda(), torch.from_numpy(c["dirs"]).float().cuda()
    from neuralsim_b200.graphics.pose import pose_rays
    with torch.no_grad():
        ro, rd = pose_rays(poses, pidx, dirs)
        to, td = pose64.torch_pose_rays(poses.q0, poses.dq, poses.t0, poses.dt, pidx, dirs)
    assert torch.equal(ro, to) and torch.equal(rd, td), "not the bits of the reference's torch ops"
    wo, wd = pose64.forward(_np(poses.q0), _np(poses.dq), _np(poses.t0), _np(poses.dt), c["pidx"], _np(dirs))
    assert (np.abs(_np(rd) - wd) <= 32 * U * pose64.bound_terms(_np(dirs))[:, None]).all()
    assert (np.abs(_np(ro) - wo) <= U * np.abs(wo)).all()


def test_forward_bits_on_a_street_batch():
    q0, t0 = pose64.street_poses(3, 8, C.ROAD_Z)
    pidx, dirs = pose64.street_batch(8192, 24, seed=3)
    poses, pidx, dirs = _poses(q0, t0, np.random.default_rng(1).normal(size=(24, 4)) * 1e-3), torch.from_numpy(pidx).cuda(), torch.from_numpy(dirs).cuda()
    from neuralsim_b200.graphics.pose import pose_rays
    with torch.no_grad():
        ro, rd = pose_rays(poses, pidx, dirs)
        to, td = pose64.torch_pose_rays(poses.q0, poses.dq, poses.t0, poses.dt, pidx, dirs)
    assert torch.equal(ro, to) and torch.equal(rd, td)


SIZES = [(1, 1), (5, 1), (1, 300), (7, 127), (7, 128), (7, 129), (64, 3 * 4096 + 77), (1, 70000), (300, 20000), (1000, 8192)]


@pytest.mark.parametrize("order", ["shuffled", "sorted"])
@pytest.mark.parametrize("P,n", SIZES)
def test_adjoint_matches_float64(P, n, order):
    used = np.arange(0, P, 2) if P > 4 else None                      # every other pose has no ray
    poses, pidx, dirs = _random_case(P, n, seed=P * 7 + n, order=order, used=used)
    if P > 4 and n > 2:
        pidx[1] = P - 1                                                # a pose with one ray only
        if order == "sorted":
            pidx = torch.sort(pidx).values
    g = torch.Generator(device="cuda").manual_seed(n)
    g_o, g_d = torch.randn(n, 3, device="cuda", generator=g), torch.randn(n, 3, device="cuda", generator=g)
    d_dq, d_dt = _kernel_grad(poses, pidx, dirs, g_o, g_d)
    r = _check_adjoint(poses, pidx, dirs, g_o, g_d, d_dq, d_dt)
    print(f"METRIC pose adjoint P={P} n={n} {order} err/bound={r:.3f}")


def test_device_count_below_capacity_ignores_nan_rows():
    from neuralsim_b200.graphics.pose import pose_backward, pose_forward, scratch_floats
    P, cap, live = 40, 3 * 4096 + 11, 5000
    poses, pidx, dirs = _random_case(P, cap, seed=5)
    g_o, g_d = torch.randn(cap, 3, device="cuda"), torch.randn(cap, 3, device="cuda")
    g_o[live:], g_d[live:], dirs[live:] = float("nan"), float("nan"), float("nan")
    cnt = torch.tensor([live], dtype=torch.int64, device="cuda")
    d_dq, d_dt = _kernel_grad(poses, pidx, dirs, g_o, g_d, count=(cnt, 0))
    e_dq, e_dt = _kernel_grad(poses, pidx[:live].contiguous(), dirs[:live].contiguous(), g_o[:live].contiguous(), g_d[:live].contiguous())
    assert torch.isfinite(d_dq).all() and torch.isfinite(d_dt).all()
    assert torch.equal(d_dq, e_dq) and torch.equal(d_dt, e_dt)
    # the forward too: rays past the count are not written
    unit, nrm, rays = torch.empty(P, 4, device="cuda"), torch.empty(P, device="cuda"), torch.full((2, cap, 3), 7.0, device="cuda")
    pose_forward(poses, pidx, dirs, unit, nrm, rays[0], rays[1], count=(cnt, 0))
    assert bool((rays[:, live:] == 7.0).all()) and bool(torch.isfinite(rays[:, :live]).all())


def test_adjoint_is_deterministic_on_shuffled_rays():
    poses, pidx, dirs = _random_case(24, 8192, seed=11)
    g_o, g_d = torch.randn(8192, 3, device="cuda"), torch.randn(8192, 3, device="cuda")
    runs = [_kernel_grad(poses, pidx, dirs, g_o, g_d) for _ in range(3)]
    for a, b in runs[1:]:
        assert torch.equal(a, runs[0][0]) and torch.equal(b, runs[0][1])


def test_accumulates_into_the_given_buffers():
    from neuralsim_b200.graphics.pose import pose_backward, pose_forward, scratch_floats
    poses, pidx, dirs = _random_case(6, 500, seed=2)
    g_o, g_d = torch.randn(500, 3, device="cuda"), torch.randn(500, 3, device="cuda")
    a_q, a_t = _kernel_grad(poses, pidx, dirs, g_o, g_d)
    unit, nrm, rays = torch.empty(6, 4, device="cuda"), torch.empty(6, device="cuda"), torch.empty(2, 500, 3, device="cuda")
    pose_forward(poses, pidx, dirs, unit, nrm, rays[0], rays[1])
    b_q, b_t = torch.ones(6, 4, device="cuda"), torch.ones(6, 3, device="cuda")
    pose_backward(unit, nrm, pidx, dirs, g_o, g_d, torch.empty(scratch_floats(500, 6), device="cuda"), b_q, b_t)
    assert torch.equal(b_q, 1 + a_q) and torch.equal(b_t, 1 + a_t)


# ===================================================================================================================== the graph step
_ST = {}
N_RAYS = 8192


def _street(cuda):
    if "r" not in _ST:
        model = C.build_model(cuda).train()
        q0, t0 = pose64.street_poses(3, 8, C.ROAD_Z)
        pidx, dirs = pose64.street_batch(N_RAYS, 24, seed=4)
        g = torch.Generator().manual_seed(9)
        w = torch.tensor([-1.0, -0.5, 0.5, 1.0])[torch.randint(0, 4, (N_RAYS, 3), generator=g)].to(cuda)
        dq0 = np.random.default_rng(2).normal(size=(24, 4)) * 2e-3
        _ST["r"] = dict(model=model, q0=q0, t0=t0, dq0=dq0, pidx=torch.from_numpy(pidx).to(cuda), dirs=torch.from_numpy(dirs).to(cuda),
                        loss=lambda r: ag._loss(r, w))
    return _ST["r"]


def _host(s, poses):
    """the host-sized fused path through the same autograd op -> rendered, model grads, dq.grad, dt.grad"""
    from neuralsim_b200.graphics.pose import pose_rays
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = s["model"]
    model.zero_grad(set_to_none=True)
    poses.zero_grad(set_to_none=True)
    o, d = pose_rays(poses, s["pidx"], s["dirs"])
    na = model.radiance_net.blocks.layers[0].in_features - 22 - model.implicit_surface.encoding.out_features if model.use_h_appear else 0
    codes = torch.zeros(N_RAYS, na, device=o.device) if na else None           # the frame's codes when none are passed
    out = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train().render(model, o, d, rays_h_appear=codes)["rendered"]
    s["loss"](out).backward()
    return ({k: v.detach().clone() for k, v in out.items()}, product_grads(model), poses.dq.grad.clone(), poses.dt.grad.clone())


def _frame(s, poses, **kw):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    s["model"].zero_grad(set_to_none=True)
    gc.collect()
    return StaticFrame(s["model"], N_RAYS, loss_fn=s["loss"], near=C.NEAR, far=C.FAR, zero_grads=True, pose=poses, **kw)


def _same(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(a, b), f"{what}: not bit-equal, max |diff| {float((a - b).abs().max()):.3e}"


def _grads_close(g, h):
    rep = {}
    for k, v in h.items():
        if v is None:
            continue
        rep[k] = rel_l2(g[k], v)
        assert rep[k] <= ag.ORDER_REL, (k, rep[k])
    return rep


def test_graph_step_matches_host_sized_path(cuda):
    s = _street(cuda)
    poses = _poses(s["q0"], s["t0"], s["dq0"])
    r_host, g_host, gq, gt = _host(s, poses)
    poses.zero_grad(set_to_none=True)
    fr = _frame(s, poses, ray_grad=True)
    fr.step(dirs=s["dirs"], pidx=s["pidx"])
    assert fr.counts()["overflow"] == 0
    for k, v in r_host.items():
        _same(fr.rendered[k], v, k)
    _same(poses.dq.grad, gq, "dq.grad")
    _same(poses.dt.grad, gt, "dt.grad")
    rep = _grads_close(product_grads(s["model"]), g_host)
    assert float(gq.abs().max()) > 0 and float(gt.abs().max()) > 0
    # a second replay (zero_grads: the pose gradient is overwritten, not doubled), and one set to None by the trainer
    fr.step()
    _same(poses.dq.grad, gq, "second replay dq.grad")
    poses.dq.grad = None
    fr.step(dirs=s["dirs"], pidx=s["pidx"])
    _same(poses.dq.grad, gq, "dq.grad after set_to_none")
    # ray_grad still fills d_rays: the pose adjoint of those cotangents is the same gradient
    from neuralsim_b200.graphics.pose import pose_rays
    o, d = pose_rays(poses, s["pidx"], s["dirs"])
    poses.zero_grad(set_to_none=True)
    torch.autograd.backward([o, d], [fr.d_rays_o, fr.d_rays_d])
    _same(poses.dq.grad, gq, "dq.grad from d_rays")
    assert fr.captures == 1
    print("METRIC pose graph host-sized", json.dumps(dict(model_grads=rep, max_dq=float(gq.abs().max()))))


def test_requires_grad_toggle(cuda):
    """enable_after: a pose without grad runs the forward only (no .grad); switching requires_grad on re-captures once"""
    s = _street(cuda)
    poses = _poses(s["q0"], s["t0"], s["dq0"])
    r_host, _, gq, gt = _host(s, poses)
    poses.zero_grad(set_to_none=True)
    poses.requires_grad_(False)
    fr = _frame(s, poses)
    fr.step(dirs=s["dirs"], pidx=s["pidx"])
    for k, v in r_host.items():
        _same(fr.rendered[k], v, f"no-grad {k}")
    assert poses.dq.grad is None and poses.dt.grad is None and fr.captures == 1
    poses.requires_grad_(True)
    fr.step(dirs=s["dirs"], pidx=s["pidx"])
    assert fr.captures == 2
    _same(poses.dq.grad, gq, "dq.grad after the toggle")
    _same(poses.dt.grad, gt, "dt.grad after the toggle")
    fr.step()
    assert fr.captures == 2


def test_graph_step_against_the_torch_recipe(cuda):
    """the trainer's current recipe: torch pose, copy_, replay with ray_grad, torch backward through the pose"""
    s = _street(cuda)
    poses = _poses(s["q0"], s["t0"], s["dq0"])
    fr = _frame(s, poses, ray_grad=True)
    fr.step(dirs=s["dirs"], pidx=s["pidx"])
    rend = {k: v.clone() for k, v in fr.rendered.items()}
    g_new = (poses.dq.grad.clone(), poses.dt.grad.clone())
    d_rays = (fr.d_rays_o.clone(), fr.d_rays_d.clone())
    del fr
    ref = _poses(s["q0"], s["t0"], s["dq0"])
    fr = _frame(s, None, ray_grad=True)
    o, d = pose64.torch_pose_rays(ref.q0, ref.dq, ref.t0, ref.dt, s["pidx"], s["dirs"])
    fr.step(o.detach(), d.detach())
    for k, v in rend.items():
        _same(fr.rendered[k], v, k)
    _same(fr.d_rays_o, d_rays[0], "d_rays_o")
    _same(fr.d_rays_d, d_rays[1], "d_rays_d")
    torch.autograd.backward([o, d], [fr.d_rays_o, fr.d_rays_d])
    for g in (g_new, (ref.dq.grad, ref.dt.grad)):
        _check_adjoint(ref, s["pidx"], s["dirs"], d_rays[0], d_rays[1], g[0], g[1])
    print("METRIC pose graph vs torch recipe", json.dumps(dict(dq_rel=rel_l2(g_new[0], ref.dq.grad), dt_rel=rel_l2(g_new[1], ref.dt.grad))))


def test_frame_refusals(cuda):
    s = _street(cuda)
    poses = _poses(s["q0"], s["t0"])
    fr = _frame(s, poses)
    bad = s["pidx"].clone()
    bad[17] = 24
    with pytest.raises(RuntimeError, match="out of range"):
        fr.set_rays(s["dirs"], bad)
    with pytest.raises(RuntimeError, match="dirs and pidx"):
        fr.step(s["dirs"], s["dirs"])
    with pytest.raises(RuntimeError, match="set_rays"):
        fr.capture()
    plain = _frame(s, None)
    with pytest.raises(RuntimeError, match="without pose"):
        plain.set_rays(s["dirs"], s["pidx"])
