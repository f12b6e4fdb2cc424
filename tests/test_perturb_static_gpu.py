"""Perturbed samples in the one-launch step, against torch's own random stream (graphics/perturb.py, csrc/perturb.cu).

1. The draw.  nsb_coarse_depths_perturbed equals batch_sample_step_linear(near, far, nc1, perturb=True) bit for bit from the same
   generator state, at 1 ray, at the block edges and on both sides of torch's grid cap (256 cap and 4 * 256 cap values), with a device
   count below the capacity (rows past it untouched); its next offset is the generator's offset after torch's draw.
2. The stage sampler.  nsb_packed_invert_cdf_perturbed equals packed_sample_cdf(..., perturb=True) at offsets chained after the coarse
   and marcher draws and an earlier stage, at nf 8 and 32, with hit counts below the capacity and beyond the grid cap.
3. The step.  From the same generator state the perturbed graph step (StaticFrame(perturb=True)) and the host-sized perturbed step
   (SingleVolumeRenderer(perturb=True)) give bit-equal images, loss, code and ray gradients, and parameter gradients to the order of the
   fp32 atomics: camera rays with codes and LiDAR rays under LidarLoss, 4096 and 8192 rays, on the 16-level cfg3 model.
4. StaticFrame(perturb=True): one capture across a level schedule with a learnable pose, each replay the host-sized step from the state
   recorded before it; fresh draws per replay; the generator advanced by the reservation; manual_seed reproduces a replay; no host
   synchronisation in step(); an arena overflow's retry redraws the same values."""
import gc

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import pose64
import test_lidar_loss_gpu as ll
import test_lotd_anneal_gpu as la
from util import rel_l2

pytestmark = pytest.mark.gpu
ORDER_REL = ll.ORDER_REL


def _cap():
    from neuralsim_b200 import torch_rng as TR
    return TR.grid_cap(torch.device("cuda"))


def _gen(seed=1234, offset=40):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    g.set_offset(offset)
    return g


def _rng(g):
    return torch.tensor([g.initial_seed(), g.get_offset()], dtype=torch.int64, device="cuda")


def _same(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.equal(a, b), f"{what}: not bit-equal, max |diff| {float((a - b).abs().max()):.3e}"


# ===================================================================================================================== the draw
def _coarse_sizes():
    cap = _cap()
    out = [(1, 129), (2, 129), (1, 256), (2, 128), (3, 9)]
    for edge in (256 * cap, 4 * 256 * cap):
        out += [(edge // 129, 129), (edge // 129 + 1, 129), (edge // 8 - 1, 8), (edge // 8, 8), (edge // 8 + 1, 8)]
    return out


@pytest.mark.parametrize("k", range(15))
def test_coarse_draw_equals_torch(k):
    from neuralsim_b200 import torch_rng as TR
    from neuralsim_b200.graphics import perturb as PT
    from neuralsim_b200.graphics.raysample import batch_sample_step_linear
    n, nc1 = _coarse_sizes()[k]
    gi = torch.Generator(device="cuda").manual_seed(k)
    near = torch.rand(n, device="cuda", generator=gi) * 2 + 0.05
    far = near + torch.rand(n, device="cuda", generator=gi) * 200 + 1
    for cap_extra in (0, 37):                                        # the capacity equal to the count, and above it with NaN rows
        g = _gen(seed=99 + k, offset=8 * k)
        rng = _rng(g)
        R = n + cap_extra
        near_c = torch.cat([near, torch.ones(cap_extra, device="cuda")])
        far_c = torch.cat([far, torch.full((cap_extra,), 2.0, device="cuda")])
        cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
        cnt[0] = n
        t = torch.full((R, nc1), float("nan"), device="cuda")
        nxt = torch.zeros(1, dtype=torch.int64, device="cuda")
        PT.coarse_depths(near_c, far_c, nc1, rng, cnt, [(0, nc1)], t, nxt)
        ref = batch_sample_step_linear(near, far, nc1, prefix_shape=[n], perturb=True, generator=g)
        _same(t[:n], ref, f"n={n} nc1={nc1}")
        assert bool(t[n:].isnan().all())
        assert int(nxt) == g.get_offset() and g.get_offset() - 8 * k == TR.uniform_inc(n * nc1, _cap())


def _packs(P, seed):
    g = np.random.default_rng(seed)
    lens = g.integers(1, 60, P)
    first = np.concatenate([[0], np.cumsum(lens)[:-1]])
    S = int(lens.sum())
    bins, cdf = np.empty(S, np.float32), np.empty(S, np.float32)
    for p in range(P):
        a, n = first[p], lens[p]
        bins[a:a + n] = np.sort(g.uniform(0.1, 80, n)).astype(np.float32)
        c = np.cumsum(g.exponential(1.0, n) * (g.uniform(0, 1, n) > 0.3))
        cdf[a:a + n] = (np.concatenate([[0], c[:-1]]) / max(c[-1], 1e-5)).astype(np.float32)
    pi = np.stack([first, lens], 1).astype(np.int64)
    return torch.from_numpy(bins).cuda(), torch.from_numpy(cdf).cuda(), torch.from_numpy(pi).cuda()


@pytest.mark.parametrize("P,extra", [(1, 0), (300, 50), (40000, 100)])
def test_stage_sampler_equals_torch_at_chained_offsets(P, extra):
    from neuralsim_b200.graphics import perturb as PT
    from neuralsim_b200.graphics.raysample import packed_sample_cdf
    bins, cdf, pi = _packs(P, P)
    n_rays, M = P + 17, int(pi[:, 1].sum())
    pi_c = torch.cat([pi, torch.zeros(extra, 2, dtype=torch.int64, device="cuda")])
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[0], cnt[12], cnt[13] = n_rays, M, P
    g = _gen(seed=P, offset=4 * P)
    rng = _rng(g)
    draws = [(0, 129), (12, 1)]
    torch.rand([n_rays, 129], device="cuda", generator=g)            # the coarse depths' and the marcher's draws, as the step makes them
    torch.rand([M], device="cuda", generator=g)
    for nf in (8, 32):
        draws = draws + [(13, nf)]
        out = torch.full((P + extra, nf), float("nan"), device="cuda")
        nxt = torch.zeros(1, dtype=torch.int64, device="cuda")
        PT.invert_cdf(bins, cdf, pi_c, nf, rng, cnt, draws, out, nxt)
        ref = packed_sample_cdf(bins, cdf, pi, nf, perturb=True, generator=g)[0]
        _same(out[:P], ref, f"P={P} nf={nf}")
        assert bool(out[P:].isnan().all()) and int(nxt) == g.get_offset()
    assert P * 32 < 256 * _cap() or P * 32 > 256 * _cap()            # (40000 x 32 lies beyond the grid cap: several calls per thread)


# ===================================================================================================================== the step
_M = {}


def _model():
    if "m" not in _M:
        _M["m"] = C.build_model(torch.device("cuda"), max_num_levels=16, log2_hashmap_size=16, target_num_params=18 * 2 ** 17).train()
    return _M["m"]


def _host_cam(model, co, cd, codes, cfg):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    for p in model.parameters():
        if p.grad is not None:
            p.grad.zero_()
    o, d, h = co.clone().requires_grad_(True), cd.clone().requires_grad_(True), codes.clone().requires_grad_(True)
    r = SingleVolumeRenderer(cfg).train().render(model, o, d, rays_h_appear=h)["rendered"]
    loss = C.loss_cam(r)
    loss.backward()
    return ({k: v.detach().clone() for k, v in r.items()}, loss.detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None},
            o.grad, d.grad, h.grad)


def _check_grads(model, h, h2, what):
    for n, p in model.named_parameters():
        if n in h[2]:
            e, spread = rel_l2(p.grad, h[2][n]), rel_l2(h2[2][n], h[2][n])
            assert e <= max(ORDER_REL, 2 * spread), (what, n, e, spread)


@pytest.mark.parametrize("n", [4096, 8192])
def test_graph_step_equals_host_sized_perturbed_step_camera(n):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model = _model()
    co, cd = (t[:n].cuda() for t in C.camera_rays(3, n))
    codes = torch.randn(n, 4, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 0.3
    cfg = dict(near=C.NEAR, far=C.FAR, perturb=True)
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, zero_grads=True, h_appear_grad=True, ray_grad=True, perturb=True)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    fr.step(co, cd, codes)                                           # the capture
    for step in range(2):
        s0 = gen.get_offset()
        h = _host_cam(model, co, cd, codes, cfg)
        gen.set_offset(s0)
        h2 = _host_cam(model, co, cd, codes, cfg)
        gen.set_offset(s0)
        fr.step(co, cd, codes)
        assert gen.get_offset() == s0 + fr.rng_reservation
        assert fr.counts()["overflow"] == 0
        for k, v in h[0].items():
            _same(fr.rendered[k], v, f"step {step} {k}")
        _same(fr.loss, h[1], f"step {step} loss")
        _check_grads(model, h, h2, f"step {step}")
        _same(fr.d_rays_o, h[3], "d_rays_o")
        _same(fr.d_rays_d, h[4], "d_rays_d")
        _same(fr.d_h_appear, h[5], "d_h_appear")
    assert fr.captures == 1


@pytest.mark.parametrize("n", [4096, 8192])
def test_graph_step_equals_host_sized_perturbed_step_lidar(n):
    model = _model()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    fr, lidar, terms, lo, ld, ranges = ll._frame_case(model, cfg, n=n)
    from neuralsim_b200.graphics.neus_static import StaticFrame
    fr = StaticFrame(model, n, loss_fn=fr.loss_fn, loss_on_ret=True, near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True, zero_grads=True, perturb=True)
    hcfg = dict(cfg, perturb=True)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    lidar.set_step(ranges, 100)
    fr.step(lo, ld)                                                  # the capture
    s0 = gen.get_offset()
    host = ll._host_step(model, lidar, lo, ld, ranges, 100, hcfg)
    gen.set_offset(s0)
    host2 = ll._host_step(model, lidar, lo, ld, ranges, 100, hcfg)
    gen.set_offset(s0)
    lidar.set_step(ranges, 100)
    fr.step(lo, ld)
    assert fr.counts()["overflow"] == 0 and gen.get_offset() == s0 + fr.rng_reservation
    got_terms = {k: v.clone() for k, v in terms.items()}
    for k, v in host[0].items():
        _same(fr.rendered[k], v, k)
    for k, v in host[1].items():
        _same(got_terms[k], v, k)
    _same(fr.loss, host[2], "loss")
    g = ll._grads(model)
    for k, v in host[3].items():
        e, spread = rel_l2(g[k], v), rel_l2(host2[3][k], v)
        assert e <= max(ORDER_REL, 2 * spread), (k, e, spread)


def test_render_static_eager_draws_from_the_default_generator():
    """render_static(perturb=True) without rng_dev: the default generator's state at the call, advanced by the reservation"""
    from neuralsim_b200.graphics import perturb as PT
    from neuralsim_b200.graphics.neus import query_config
    from neuralsim_b200.graphics.neus_static import render_static
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = _model()
    n = 4096
    co, cd = (t[:n].cuda() for t in C.camera_rays(2, n))
    codes = torch.zeros(n, 4, device="cuda")
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    with torch.no_grad():
        rt = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train().ray_query(model, co, cd, codes, return_buffer=True, return_details=True)["ray_tested"]
        s0 = gen.get_offset()
        r, cnt, _ = render_static(model, co, cd, codes, near=C.NEAR, far=C.FAR, march_cap=n * 300, kept_cap=n * 200,
                                  coherent=bool(rt.get("rays_coherent", False)), perturb=True)
        cfg = query_config(**(model.ray_query_cfg.get("query_param", {}) or {}), upsample_s_divisor=model.upsample_s_divisor)
        assert gen.get_offset() == s0 + PT.reservation(n, cfg, _cap())
        assert int(cnt[20]) == 0
        gen.set_offset(s0)
        h = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, perturb=True)).train().render(model, co, cd, rays_h_appear=codes)["rendered"]
    for k in ("rgb_volume", "depth_volume", "mask_volume", "normals_volume"):
        _same(r[k], h[k], k)


def test_perturb_before_march_is_refused():
    from neuralsim_b200.graphics.neus_static import render_static
    model = _model()
    co, cd = (t[:256].cuda() for t in C.camera_rays(1, 256))
    qp = model.ray_query_cfg.setdefault("query_param", {})
    saved = qp.get("march_cfg")
    qp["march_cfg"] = dict(saved or {}, perturb_before_march=True)
    try:
        with pytest.raises(RuntimeError, match="perturb_before_march"):
            render_static(model, co, cd, near=C.NEAR, far=C.FAR, march_cap=1 << 20, kept_cap=1 << 20, perturb=True)
    finally:
        if saved is None:
            qp.pop("march_cfg")
        else:
            qp["march_cfg"] = saved


# ===================================================================================================================== StaticFrame
def test_frame_follows_a_level_schedule_with_a_pose():
    """one capture over four replays crossing level changes with a learnable pose: each replay is the host-sized perturbed step from the
    state recorded before it; consecutive replays draw different depths; the generator moves by the reservation; manual_seed repeats a
    replay; step() has no host synchronisation"""
    import test_pose_refine_gpu as pr
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.graphics.pose import pose_rays
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from util import product_grads
    model = la._annealed_cfg3()
    n = 4096
    q0, t0 = pose64.street_poses(3, 8, C.ROAD_Z)
    pidx, dirs = pose64.street_batch(n, 24, seed=4)
    pidx, dirs = torch.from_numpy(pidx).cuda(), torch.from_numpy(dirs).cuda()
    poses = pr._poses(q0, t0, np.random.default_rng(2).normal(size=(24, 4)) * 2e-3)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]

    def host(s0):
        gen.set_offset(s0)
        for p in model.parameters():                  # in place: the captured step accumulates into these tensors
            if p.grad is not None:
                p.grad.zero_()
        poses.zero_grad(set_to_none=True)
        o, d = pose_rays(poses, pidx, dirs)
        codes = torch.zeros(n, 4, device="cuda")
        out = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, perturb=True)).train().render(model, o, d, rays_h_appear=codes)["rendered"]
        loss = C.loss_cam(out)
        loss.backward()
        return ({k: v.detach().clone() for k, v in out.items()}, loss.detach(), product_grads(model), poses.dq.grad.clone(), poses.dt.grad.clone())

    la._set_iter(model, la.STOP_IT)                  # the arenas sized at all levels
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, zero_grads=True, pose=poses, perturb=True, slack=2.0,
                     kept_cap=n * la.KEPT_PER_RAY)
    fr.set_rays(dirs, pidx)
    depths, levels = [], set()
    for it in (2, 3, 4, 5):
        la._set_iter(model, it)
        levels.add(model.implicit_surface.encoding.max_level)
        s0 = gen.get_offset()
        fr.step()
        assert gen.get_offset() == s0 + fr.rng_reservation
        assert fr.counts()["overflow"] == 0, it
        got = ({k: v.clone() for k, v in fr.rendered.items()}, fr.loss.clone(), product_grads(model), poses.dq.grad.clone(), poses.dt.grad.clone())
        depths.append(fr.buffers["t"][:fr.counts()["kept"]].clone())
        h = host(s0)
        h2 = host(s0)
        for k, v in h[0].items():
            _same(got[0][k], v, f"it {it} {k}")
        _same(got[1], h[1], f"it {it} loss")
        _same(got[3], h[3], f"it {it} dq.grad")
        _same(got[4], h[4], f"it {it} dt.grad")
        for k, v in h[2].items():
            if v is not None:
                e, spread = rel_l2(got[2][k], v), rel_l2(h2[2][k], v)
                assert e <= max(ORDER_REL, 2 * spread), (it, k, e, spread)
        poses.zero_grad(set_to_none=True)
        gen.set_offset(s0 + fr.rng_reservation)
    assert len(levels) == 4 and fr.captures == 1
    assert all(not (a.shape == b.shape and torch.equal(a, b)) for a, b in zip(depths, depths[1:]))
    # the same seed twice: the same replay
    outs = []
    for _ in range(2):
        torch.manual_seed(77)
        fr.step()
        outs.append({k: v.clone() for k, v in fr.rendered.items()})
    for k in outs[0]:
        _same(outs[0][k], outs[1][k], f"manual_seed {k}")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fr.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert fr.captures == 1


def test_overflow_retry_redraws_the_same_values():
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = _model()
    n = 4096
    co, cd = (t[:n].cuda() for t in C.camera_rays(1, n))
    codes = torch.zeros(n, 4, device="cuda")
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, zero_grads=True, march_cap=1024, kept_cap=256, coherent=False, perturb=True)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    s0 = gen.get_offset()
    fr.step(co, cd, codes)
    assert fr.counts()["overflow"] != 0
    assert fr.check() is False
    assert fr.counts()["overflow"] == 0 and gen.get_offset() == s0 + fr.rng_reservation
    gen.set_offset(s0)
    with torch.no_grad():
        h = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, perturb=True)).train().render(model, co, cd, rays_h_appear=codes)["rendered"]
    for k, v in h.items():
        _same(fr.rendered[k], v, k)
