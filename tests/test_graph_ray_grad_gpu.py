"""The gradient to learnable rays from the one-launch graph step (`StaticFrame(..., ray_grad=True)`): the boundary query's and the colour
query's per-ray sums (nsb_fused_sdf_bwd_rays, nsb_fused_color_bwd_grads through the ray map of the codes) and the adjoint of the ray test
and the view directions (nsb_gather_rays_backward), against the host-sized render of the same rays built from a learnable pose, and the
800x600 benchmark frame against a float64 replay of its step (oracle/step64.py, tests/rays64.py, tests/ray_adjoint64.py).

Bounds.  The graph step runs the host-sized path's kernels on the same samples and adds the three contributions to a ray's direction in
the order torch autograd adds them there (tests/test_graph_ray_grad.py), so its ray gradient is compared bit for bit.  Parameter
gradients are compared up to ORDER_REL, the bound of two runs that differ only in the order of the fp32 table atomics
(tests/test_appear_grad_gpu.py).  The bound of the ray-gradient entry points against float64 (tests/test_ray_grad_gpu.py RAY_REL, 6e-3)
would let a reference without the view-direction term pass at the 800x600 frame (it is 5.9e-4 off there on an H100), so the frame's
bound follows the step's own error budget instead (tests/test_step_grad_frame_gpu.py: fp16 values that round the other way move a
gradient of the 4096-ray subset by ~1e-4 relative): FRAME_RAY_REL = 2e-4, against 4.2e-5 measured on an H100.  The Adam steps keep
tests/test_ray_grad_gpu.py's bound."""
import gc
import json

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import test_appear_grad_gpu as ag
import test_partial_levels_gpu as pl
import test_ray_grad_gpu as rg
from oracle import fused64, neus64, step64
from ray_adjoint64 import adjoint
from rays64 import color_rows, ray_grads, sdf_rows
from util import make_pair, product_grads, rel_l2

pytestmark = pytest.mark.gpu

ORDER_REL = ag.ORDER_REL
FRAME_RAY_REL = 2e-4
P0 = [0.01, -0.02, 0.015, 0.01, 0.02, -0.01]


def _host(model, ro, rd, params, loss_fn, cfg, codes=None):
    """the host-sized render of the posed rays -> (rendered, d_rays_o, d_rays_d, d_codes | None)"""
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model.zero_grad(set_to_none=True)
    o, d = rg._pose(params, ro, rd)
    o.retain_grad()
    d.retain_grad()
    kw = dict(rays_h_appear=codes) if codes is not None else {}
    out = SingleVolumeRenderer(cfg).train().render(model, o, d, **kw)["rendered"]
    loss_fn(out).backward()
    return {k: v.detach().clone() for k, v in out.items()}, o.grad.clone(), d.grad.clone(), None if codes is None else codes.grad.clone()


def _frame(model, n, loss_fn, cfg, **kw):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model.zero_grad(set_to_none=True)
    gc.collect()
    return StaticFrame(model, n, loss_fn=loss_fn, near=cfg.get("near"), far=cfg.get("far"), with_rgb=cfg.get("with_rgb", True),
                       with_normal=cfg.get("with_normal", True), zero_grads=True, **kw)


def _posed(ro, rd, p=P0):
    with torch.no_grad():
        return rg._pose(torch.tensor(p, device=ro.device), ro, rd)


def _same(a, b, what):
    assert a.shape == b.shape, what
    if not torch.equal(a, b):
        raise AssertionError(f"{what}: not bit-equal, max |diff| {float((a - b).abs().max()):.3e}, rel-L2 {rel_l2(a, b):.3e}")


# ===================================================================================================================== camera rays
_CAM = {}
CAM_CFG = dict(near=0.01)


def _cam(cuda):
    if "r" not in _CAM:
        _, model = make_pair(cuda)
        model.train()
        ro, rd, codes0, w = ag._frame_rays(cuda)
        loss = lambda r: ag._loss(r, w)
        params = torch.tensor(P0, device=cuda, requires_grad=True)
        host = _host(model, ro, rd, params, loss, CAM_CFG, codes0.clone().requires_grad_(True))
        _CAM["r"] = dict(model=model, ro=ro, rd=rd, codes0=codes0, w=w, loss=loss, host=host)
    return _CAM["r"]


def test_camera_rays_bit_equal_to_host_sized(cuda):
    """a camera batch from a learnable SE(3) pose with learnable codes: rendered buffers, the code gradient and the ray gradient of the
    graph step are the host-sized render's bits; a second replay overwrites; a parameter update is followed; one capture"""
    c = _cam(cuda)
    model, (r_host, g_o, g_d, g_codes) = c["model"], c["host"]
    o, d = _posed(c["ro"], c["rd"])
    fr = _frame(model, o.shape[0], c["loss"], CAM_CFG, h_appear_grad=True, ray_grad=True)
    fr.step(o, d, c["codes0"])
    assert fr.counts()["overflow"] == 0
    for k, v in r_host.items():
        _same(fr.rendered[k], v, k)
    _same(fr.d_h_appear, g_codes, "d_h_appear")
    _same(fr.d_rays_o, g_o, "d_rays_o")
    _same(fr.d_rays_d, g_d, "d_rays_d")
    print("METRIC graph raygrad camera", json.dumps(dict(max_o=float(g_o.abs().max()), max_d=float(g_d.abs().max()))))
    assert float(g_o.abs().max()) > 0 and float(g_d.abs().max()) > 0
    assert bool((fr.d_rays_o[-40:] == 0).all()) and bool((fr.d_rays_d[-40:] == 0).all())        # the 40 rays that miss the box
    first = (fr.d_rays_o.clone(), fr.d_rays_d.clone())
    fr.step(o, d, c["codes0"])
    _same(fr.d_rays_o, first[0], "second replay d_rays_o")
    _same(fr.d_rays_d, first[1], "second replay d_rays_d")
    R1 = model.radiance_net.blocks.layers[0].weight
    saved = R1.detach().clone()
    try:
        with torch.no_grad():
            R1.mul_(1.25)
        fr.step(o, d, c["codes0"])
        upd = (fr.d_rays_o.clone(), fr.d_rays_d.clone())
        _, h_o, h_d, _ = _host(model, c["ro"], c["rd"], torch.tensor(P0, device=cuda, requires_grad=True), c["loss"], CAM_CFG,
                                  c["codes0"].clone().requires_grad_(True))
    finally:
        with torch.no_grad():
            R1.copy_(saved)
    assert not torch.equal(upd[1], first[1])
    _same(upd[0], h_o, "updated d_rays_o")
    _same(upd[1], h_d, "updated d_rays_d")
    assert fr.captures == 1


def test_option_changes_nothing_else(cuda):
    """ray_grad on vs off: rendered buffers, loss and d_h_appear bit-equal; parameter gradients to the order of the fp32 atomics"""
    c = _cam(cuda)
    model = c["model"]
    o, d = _posed(c["ro"], c["rd"])
    runs = []
    for on in (False, True, False):
        fr = _frame(model, o.shape[0], c["loss"], CAM_CFG, h_appear_grad=True, ray_grad=on)
        fr.step(o, d, c["codes0"])
        runs.append(({k: v.clone() for k, v in fr.rendered.items()}, fr.loss.clone(), fr.d_h_appear.clone(), product_grads(model)))
        assert (fr.d_rays_o is not None) == on
        del fr
    (r0, l0, h0, g0), (r1, l1, h1, g1), (_, _, _, g2) = runs
    for k in r0:
        _same(r1[k], r0[k], k)
    _same(l1, l0, "loss")
    _same(h1, h0, "d_h_appear")
    rep = {}
    for k, v in g0.items():
        if v is None:
            assert g1[k] is None, k
            continue
        rep[k] = (rel_l2(g1[k], v), rel_l2(g2[k], v))
        assert rep[k][0] <= max(ORDER_REL, 2 * rep[k][1]), (k, rep[k])
    print("METRIC graph raygrad option", json.dumps(rep))


def test_use_graph_false_and_overflow_recapture(cuda):
    """the same gradient without a CUDA graph, and after an arena overflow that check() re-captures"""
    c = _cam(cuda)
    model, (_, g_o, g_d, g_codes) = c["model"], c["host"]
    o, d = _posed(c["ro"], c["rd"])
    fr = _frame(model, o.shape[0], c["loss"], CAM_CFG, h_appear_grad=True, ray_grad=True, use_graph=False)
    fr.step(o, d, c["codes0"])
    _same(fr.d_rays_o, g_o, "eager d_rays_o")
    _same(fr.d_rays_d, g_d, "eager d_rays_d")
    for caps in (dict(march_cap=4096, kept_cap=1 << 20), dict(march_cap=1 << 22, kept_cap=4096)):
        fr = _frame(model, o.shape[0], c["loss"], CAM_CFG, h_appear_grad=True, ray_grad=True, **caps)
        fr.coherent = True
        fr.step(o, d, c["codes0"])
        assert fr.counts()["overflow"] != 0, caps
        assert fr.check() is False and fr.captures == 2
        assert fr.counts()["overflow"] == 0
        _same(fr.d_rays_o, g_o, f"re-captured d_rays_o {caps}")
        _same(fr.d_rays_d, g_d, f"re-captured d_rays_d {caps}")
        _same(fr.d_h_appear, g_codes, f"re-captured d_h_appear {caps}")


# ===================================================================================================================== LiDAR rays
def _lidar_case(model, cfg, n=4096, seed=1):
    lo, ld = C.lidar_rays(seed, n)
    lo, ld = lo.cuda(), ld.cuda()
    loss = C.loss_lidar if cfg.get("with_normal", True) else (lambda r: r["depth_volume"].mean() + r["mask_volume"].mean())
    host = _host(model, lo, ld, torch.tensor(P0, device=lo.device, requires_grad=True), loss, cfg)
    o, d = _posed(lo, ld)
    fr = _frame(model, n, loss, cfg, ray_grad=True)
    fr.step(o, d)
    assert fr.counts()["overflow"] == 0
    for k, v in host[0].items():
        _same(fr.rendered[k], v, k)
    _same(fr.d_rays_o, host[1], "d_rays_o")
    _same(fr.d_rays_d, host[2], "d_rays_d")
    hit = host[0]["mask_volume"] > 0
    assert float(host[2].abs().max()) > 0 and bool((fr.d_rays_o[~hit] == 0).all())
    return fr


@pytest.mark.parametrize("with_normal", [True, False], ids=["normals", "depth-only"])
def test_lidar_rays_on_cfg3_colour_model(cuda, with_normal):
    """with_rgb=False on the cfg3 colour model: no view-direction term; without normals no kept-sample query runs (boundary term only)"""
    model = C.build_model(cuda).train()
    _lidar_case(model, dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=with_normal))


def test_lidar_rays_on_12_level_geometry_only_model(cuda):
    model = pl._cfg3_geo12(cuda)
    _lidar_case(model, dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True))


# ===================================================================================================================== training
def test_adam_steps_on_pose_move_it_as_host_sized_path(cuda):
    """four Adam steps on a pose alone (the model fixed: no parameter requires grad), each step's rays replayed through StaticFrame and
    the pose's backward run outside the graph, take the pose where the host-sized path takes it"""
    _, model = make_pair(cuda)
    model.train()
    for p in model.parameters():
        p.requires_grad_(False)
    ro, rd, codes, w = ag._frame_rays(cuda)
    loss = lambda r: ag._loss(r, w)
    start = [0.02, -0.01, 0.01, 0.03, 0.0, -0.02]
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    gc.collect()
    fr = StaticFrame(model, ro.shape[0], loss_fn=loss, near=0.01, ray_grad=True, slack=2.0)

    def steps(graph):
        params = torch.tensor(start, device=cuda, requires_grad=True)
        opt = torch.optim.Adam([params], lr=2e-3)
        for _ in range(4):
            opt.zero_grad()
            o, d = rg._pose(params, ro, rd)
            if graph:
                fr.step(o.detach(), d.detach(), codes)
                torch.autograd.backward([o, d], [fr.d_rays_o, fr.d_rays_d])
            else:
                loss(SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=codes)["rendered"]).backward()
            opt.step()
        return params.detach().clone()

    a, b = steps(True), steps(False)
    s = torch.tensor(start, device=cuda)
    print("METRIC graph raygrad adam", json.dumps(dict(moved_rel=rel_l2(a - s, b - s), captures=fr.captures)))
    assert float((b - s).abs().min()) > 0
    assert rel_l2(a - s, b - s) <= 0.1


# ===================================================================================================================== the 800x600 frame
_FRAME = {}


def _frame_case(cuda, monkeypatch):
    """bench.py's model and 800x600 frame (view 0), rgb loss weighted per ray; the graph step's ray gradient on a 4096-ray subset of its
    solid hit rays and, from the float64 replay of those rays on the host-sized step's decisions, the per-ray gradients to the compacted
    rays from the colour (kept) samples and the boundary samples, and the view-direction gradient.  The bench box is [-1, 1]^3, where
    the division by its half-size is the identity; here box and rays are scaled by 2 (exact in fp32), which leaves the normalised rays,
    and so every sample, bit-identical and makes the world-frame gradient half the normalised one."""
    if "r" in _FRAME:
        return _FRAME["r"]
    import bench
    import test_step_grad_frame_gpu as sf
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = bench.build_model(cuda).train()
    with torch.no_grad():
        model.space.aabb.mul_(2.0)
    assert model.space.radius3d.tolist() == [2.0, 2.0, 2.0] and model.space.center.tolist() == [0.0, 0.0, 0.0]
    o, d = sf._rays(0, False, cuda)
    o, d = o * 2.0, d * 2.0
    n = o.shape[0]
    g = torch.Generator().manual_seed(21)
    w = torch.tensor([-1.0, -0.5, 0.5, 1.0])[torch.randint(0, 4, (n, 3), generator=g)].to(cuda)
    loss = lambda r: (r["rgb_volume"] * w).sum()
    codes = torch.zeros(n, 4, device=cuda)
    cap = sf._Capture(monkeypatch, model)
    with torch.no_grad():
        out = SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=codes)["rendered"]
    r_host = {k: v.detach().clone() for k, v in out.items()}
    c = cap.host()
    del out
    monkeypatch.undo()
    fr = _frame(model, n, loss, dict(near=0.01), ray_grad=True)
    fr.step(o, d, codes)
    assert fr.counts()["overflow"] == 0
    for k in r_host:
        _same(fr.rendered[k], r_host[k], k)
    hit = c["compact"]["rays_inds_hit"]
    solid = np.nonzero(r_host["mask_volume"].cpu().numpy()[hit] > 0.5)[0]
    packs = np.sort(np.random.default_rng(5).choice(solid, sf.N_SUBSET, replace=False))
    dec = sf._decisions(c, packs)
    ref = fused64.Fused64.from_model(model)
    R = packs.shape[0]
    g_rgb = w[torch.from_numpy(hit[packs]).to(cuda)].double().cpu().numpy()
    seen = {}
    orig_cb, orig_sb, orig_ab = ref.color_backward, ref.sdf_backward, neus64.alpha_backward

    def color_backward(fwd, *a, **k):
        seen.update(fwd=fwd, g_nablas=k.get("g_nablas"), g_rgb=k.get("g_rgb"))
        return orig_cb(fwd, *a, **k)

    def sdf_backward(x, d_sdf, *a, **k):
        seen.update(x=x, d_sdf=d_sdf)
        return orig_sb(x, d_sdf, *a, **k)

    def alpha_backward(*a, **k):
        out_ = orig_ab(*a, **k)
        seen.update(nz=np.nonzero(out_["d_sdf"])[0])
        return out_
    ref.color_backward, ref.sdf_backward = color_backward, sdf_backward
    with monkeypatch.context() as mp:
        mp.setattr(neus64, "alpha_backward", alpha_backward)
        step64.step_grads(ref, dec, c["compact"]["inv_s"], g_mask=np.zeros(R), g_depth=np.zeros(R), g_rgb=g_rgb, g_nablas=np.zeros((R, 3)),
                          ln_inv_s_factor=model.ctrl_var.ln_inv_s_factor)
    kpi = np.asarray(dec["kept_pinfo"], np.int64)
    ray_k = neus64.pack_of(kpi, int(kpi[:, 1].sum()))
    gx_c, gv_c = color_rows(ref, seen["fwd"], np.asarray(dec["view"])[ray_k], g_nablas=seen["g_nablas"], g_rgb=seen["g_rgb"])
    col = ray_grads(gx_c, dec["t_kept"], ray_k, R, gv_c)
    pinfo = np.asarray(dec["pinfo"], np.int64)
    ray_b = neus64.pack_of(pinfo, int(pinfo[:, 1].sum()))[seen["nz"]]
    bnd = ray_grads(sdf_rows(ref, seen["x"], seen["d_sdf"]), np.asarray(dec["t1"])[seen["nz"]], ray_b, R)
    rows = torch.from_numpy(hit[packs]).to(cuda)
    got = (fr.d_rays_o[rows].double().cpu().numpy(), fr.d_rays_d[rows].double().cpu().numpy())
    miss = np.setdiff1d(np.arange(n), hit)
    miss_t = torch.from_numpy(miss).to(cuda)
    _FRAME["r"] = dict(got=got, col=col, bnd=bnd, vnorm=np.linalg.norm(np.asarray(dec["d"], np.float64), axis=1).clip(1e-10),
                       r3=model.space.radius3d.double().cpu().numpy(), R=R, n_miss=int(miss.shape[0]),
                       miss_zero=bool((fr.d_rays_o[miss_t] == 0).all()) and bool((fr.d_rays_d[miss_t] == 0).all()))
    return _FRAME["r"]


def _ref_rays(r, view=True, divide=True, boundary=True):
    """the float64 reference of the subset's ray gradient, or a deliberately wrong one"""
    col, bnd = r["col"], r["bnd"]
    g_o = col[0] + (bnd[0] if boundary else 0)
    g_d = col[1] + (bnd[1] if boundary else 0)
    return adjoint(np.arange(r["R"]), r["R"], r["r3"] if divide else np.ones(3), g_o, g_d, col[2] if view else None, r["vnorm"])


def _err(r, ref):
    return max(ag._rel(r["got"][0], ref[0]), ag._rel(r["got"][1], ref[1]))


def test_frame_ray_gradient_matches_float64_replay(cuda, monkeypatch):
    r = _frame_case(cuda, monkeypatch)
    ref = _ref_rays(r)
    e = _err(r, ref)
    print(f"METRIC graph raygrad frame800x600 subset={r['R']} rel={e:.2e} (bound {FRAME_RAY_REL:.0e}) misses={r['n_miss']}")
    assert np.abs(ref[1]).max() > 0 and np.abs(r["bnd"][1]).max() > 0 and np.abs(r["col"][2]).max() > 0
    assert e <= FRAME_RAY_REL, e
    assert r["miss_zero"]


def test_frame_wrong_references_fail(cuda, monkeypatch):
    """the bound can fail: references without the view-direction term, without the division by the box's half-size, and without the
    boundary samples' contribution fail the comparison the kernels pass"""
    r = _frame_case(cuda, monkeypatch)
    errs = dict(no_view=_err(r, _ref_rays(r, view=False)), no_divide=_err(r, _ref_rays(r, divide=False)),
                no_boundary=_err(r, _ref_rays(r, boundary=False)))
    print("METRIC graph raygrad frame wrong references", json.dumps({k: f"{v:.2e}" for k, v in errs.items()}), f"(bound {FRAME_RAY_REL:.0e})")
    assert all(e > FRAME_RAY_REL for e in errs.values()), errs
