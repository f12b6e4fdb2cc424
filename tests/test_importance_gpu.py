"""Error-map importance sampling inside the step (csrc/importance.cu, neuralsim_b200/importance.py), against torch's own ops on the GPU.

1. The draws.  nsb_imp_sample's in-kernel torch.randint / torch.rand are bit-equal to torch's from the same generator state, at 1 value,
   at the block edges and on both sides of torch's grid cap, and the offset it leaves is the generator's after torch's draws.
2. The batch.  nsb_imp_sample over two cameras of different image sizes (CameraSampler) equals the reference recipe run with torch ops on
   the GPU: frame indices, xy, pose indices, camera-space directions, ground-truth rows (float rgb, bool mask) and appearance codes.
3. The update.  nsb_error_map_update equals the reference's update on the CPU and CUDA torch under deterministic algorithms on
   collision-heavy batches; a negative error sets the flag StaticFrame.check() raises on.
4. The step.  StaticFrame(sampler=...) with pose refinement, perturbation and appearance codes on the cfg3 model at 4096 and 8192 rays,
   over a run that switches cameras and crosses a cdf rebuild: each replay equals the host-sized sequence from the same generator state
   (sample, set rays, host perturbed step, loss, update): batch, images, loss and error maps bit-equal, parameter gradients to the order of
   the fp32 atomics; one capture; no host synchronisation in step()."""
import gc

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import pose64
from util import product_grads, rel_l2

pytestmark = pytest.mark.gpu
ORDER_REL = 3e-6


def _I():
    from neuralsim_b200 import importance as I
    return I


def _cap():
    from neuralsim_b200 import torch_rng as TR
    return TR.grid_cap(torch.device("cuda"))


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(a, b), f"{what}: not bit-equal ({int((a != b).sum())} elements differ)"


def _gen(seed, offset):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    g.set_offset(offset)
    return g


def _rng(g):
    return torch.tensor([g.initial_seed(), g.get_offset()], dtype=torch.int64, device="cuda")


def _map(n_images, hw=(32, 64), seed=0, **kw):
    I = _I()
    m = I.ErrorMap(n_images, hw, device="cuda", **kw)
    g = torch.Generator("cuda").manual_seed(seed)
    m.error_map.copy_(torch.rand(m.error_map.shape, device="cuda", generator=g) * (torch.rand(m.error_map.shape, device="cuda", generator=g) > 0.5))
    m.construct_cdf()
    return m


# ===================================================================================================================== 1. the draws
def _sizes():
    cap = _cap()
    e1, e4 = 256 * cap, 4 * 256 * cap
    return [1, 2, 255, 256, 257, 1023, 1024, 1025, e1 - 1, e1, e1 + 1, e4 // 2 - 1, e4 // 2 + 3, e4 + 5]


@pytest.mark.parametrize("k", range(14))
@pytest.mark.parametrize("frac", [1.0, 0.5, 0.0])
def test_draws_equal_torch(k, frac):
    """frac 1: randint([n]) and rand([n, 2]) alone; 0.5 and 0: the four draws at chained offsets, against the recipe"""
    I = _I()
    n = _sizes()[k]
    m = _map(5, seed=k)
    s = I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=frac)
    g = _gen(31 + k, 4 * k)
    rng = _rng(g)
    table = torch.tensor([m.table_row()], dtype=torch.int64).cuda()
    cam = torch.zeros((), dtype=torch.int64, device="cuda")
    fidx = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    xy = torch.full((n, 2), float("nan"), device="cuda")
    nxt = torch.zeros(2, dtype=torch.int64, device="cuda")
    I.imp_sample(table, cam, rng, n, I.split(n, frac)[0], (32, 64), fidx, xy, rng_next=nxt)
    ri, rxy = I.recipe_sample_img_pixel((m.cdf_x_cond_y, m.cdf_y, m.cdf_img), 5, n, frac, generator=g)
    _same(fidx, ri, f"n={n} frac={frac} fidx")
    _same(xy, rxy, f"n={n} frac={frac} xy")
    assert nxt.tolist() == [rng[0].item(), g.get_offset()]
    assert g.get_offset() - 4 * k == I.sampler_inc(n, frac, _cap())
    if frac == 1.0 and n >= 1024:
        assert set(fidx.unique().tolist()) == set(range(5))
    del s


def test_module_draw_uses_the_default_generator():
    """ImpSampler.sample_img_pixel / ErrorMap.sample_img_pixel: the kernel from the default generator's state, which moves past the draw"""
    I = _I()
    m = _map(4, seed=3)
    s = I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=0.5)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    for f, obj in ((0.5, s), (0.0, m)):
        s0 = gen.get_offset()
        i, xy = obj.sample_img_pixel(999)
        s1 = gen.get_offset()
        gen.set_offset(s0)
        ri, rxy = I.recipe_sample_img_pixel((m.cdf_x_cond_y, m.cdf_y, m.cdf_img), 4, 999, f)
        assert gen.get_offset() == s1
        _same(i, ri, "i")
        _same(xy, rxy, "xy")


# ===================================================================================================================== 2. the batch
def _cameras(n_appear=4, seed=0):
    """two cameras: 6 frames of 96 x 64 (no skew) and 9 frames of 80 x 48 (skew 0.7), rgb + occupancy mask, pose bases 0 / 6"""
    I = _I()
    g = torch.Generator("cuda").manual_seed(seed)
    specs = [(6, 96, 64, 100.0, 0.0), (9, 80, 48, 90.0, 0.7)]
    samplers, gts, intrs, wh = [], [], [], []
    for c, (F, W, H, f, sk) in enumerate(specs):
        m = _map(F, seed=10 + c, n_steps_init=2)
        samplers.append(I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=0.5))
        gts.append(dict(image_rgb=torch.rand(F, H, W, 3, device="cuda", generator=g),
                        image_occupancy_mask=torch.rand(F, H, W, device="cuda", generator=g) > 0.3))
        K = torch.tensor([[f, sk, W / 2 + 0.3], [0, f * 1.01, H / 2 - 0.2], [0, 0, 1]], dtype=torch.float32)
        K = K.repeat(F, 1, 1)
        K[:, 0, 0] += torch.arange(F) * 0.5                          # per-frame intrinsics
        intrs.append(K.cuda().contiguous())
        wh.append((W, H))
    table = torch.randn(6 + 9 + 3, n_appear, device="cuda", generator=g)
    return I.CameraSampler(samplers, gts, intrs, wh, pose_bases=[0, 6], appear_bases=[3, 9], appear_table=table), specs


def _recipe_batch(cs, cam, n, generator=None):
    """the reference's batch of camera `cam` with torch ops on the GPU: -> dict"""
    I = _I()
    m = cs.samplers[cam].error_map
    fidx, xy = I.recipe_sample_img_pixel((m.cdf_x_cond_y, m.cdf_y, m.cdf_img), m.n_images, n, cs.frac_uniform, generator=generator)
    W, H = int(cs.table[cam, 5]), int(cs.table[cam, 6])
    w, h, dirs = I.recipe_pixels(xy, fidx, torch.tensor([W, H], device="cuda"), cs.intrs[cam])
    base, abase = int(cs.table[cam, 7]), int(cs.table[cam, 8])
    gt = {k: v[fidx, h, w] for k, v in cs.gts[cam].items()}
    return dict(fidx=fidx, xy=xy, pidx=base + fidx, dirs=dirs, gt=gt, codes=cs.appear_table[abase + fidx])


@pytest.mark.parametrize("n", [1, 777, 8192])
def test_batch_equals_recipe_on_two_cameras(n):
    I = _I()
    cs, _ = _cameras()
    for cam in (1, 0):
        g = _gen(5 + cam, 8 * n)
        rng = _rng(g)
        camt = torch.tensor(cam, dtype=torch.int64, device="cuda")
        out = dict(fidx=torch.empty(n, dtype=torch.int64, device="cuda"), xy=torch.empty(n, 2, device="cuda"),
                   pidx=torch.empty(n, dtype=torch.int64, device="cuda"), dirs=torch.empty(n, 3, device="cuda"))
        gts = {k: torch.empty((n,) + tail, dtype=dt, device="cuda") for k, (dt, tail) in cs.gt_spec.items()}
        ha = torch.empty(n, 4, device="cuda")
        nxt = torch.zeros(2, dtype=torch.int64, device="cuda")
        cs.sample(camt, rng, n, out["fidx"], out["xy"], out["pidx"], out["dirs"], gts, ha, nxt)
        ref = _recipe_batch(cs, cam, n, generator=g)
        for k in ("fidx", "xy", "pidx", "dirs"):
            _same(out[k], ref[k], f"cam {cam} n={n} {k}")
        for k in gts:
            _same(gts[k], ref["gt"][k], f"cam {cam} n={n} {k}")
        _same(ha, ref["codes"], f"cam {cam} n={n} codes")
        assert int(nxt[1]) == g.get_offset()


# ===================================================================================================================== 3. the update
def _collide(n, n_images, hw, seed):
    g = np.random.default_rng(seed)
    fidx = g.integers(0, min(n_images, 2), n)
    cells = g.integers(0, 4, (n, 2))
    xy = ((cells + g.choice([0.0, 0.5, 0.999], (n, 2))) / np.array([hw[1], hw[0]])).astype(np.float32)
    xy[:4] = np.array([[1e-6, 1e-6], [1 - 1e-6, 1 - 1e-6], [1e-6, 1 - 1e-6], [0.5, 0.5]], np.float32)[:n]
    val = g.exponential(1.0, n).astype(np.float32)
    return torch.from_numpy(fidx), torch.from_numpy(xy), torch.from_numpy(val)


@pytest.mark.parametrize("n,n_images,hw", [(1, 1, (2, 2)), (5000, 3, (32, 64)), (65536, 7, (32, 64)), (3000, 2, (5, 7))])
def test_update_equals_reference(n, n_images, hw):
    I = _I()
    m = I.ErrorMap(n_images, hw, device="cuda")
    start = torch.rand(n_images, *hw) * (torch.rand(n_images, *hw) > 0.5)
    m.error_map.copy_(start)
    cpu, gpu = start.clone(), start.cuda()
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for b in range(3):
            fidx, xy, val = _collide(n, n_images, hw, 10 * n + b)
            m.update_error_map(fidx.cuda(), xy.cuda(), val.cuda())
            I.recipe_update_error_map(cpu, fidx, xy, val)
            I.recipe_update_error_map(gpu, fidx.cuda(), xy.cuda(), val.cuda())
            _same(m.error_map.cpu(), cpu, f"b{b} vs CPU")
            _same(m.error_map, gpu, f"b{b} vs CUDA deterministic")
    finally:
        torch.use_deterministic_algorithms(was)
    assert bool((m.last == -1).all()) and int(m.flag) == 0


def test_negative_error_sets_the_flag():
    I = _I()
    m = I.ErrorMap(2, (4, 8), device="cuda")
    fidx, xy = torch.zeros(3, dtype=torch.int64, device="cuda"), torch.full((3, 2), 0.5, device="cuda")
    with pytest.raises(RuntimeError, match="negative"):
        m.update_error_map(fidx, xy, torch.tensor([0.1, -0.2, 0.3], device="cuda"))
    I.error_map_update(fidx, xy, torch.tensor([0.1, -0.2, 0.3], device="cuda"), m.flag, error_map=m.error_map, last=m.last)
    assert int(m.flag) == 1


# ===================================================================================================================== 4. the step
_M = {}


def _model():
    if "m" not in _M:
        _M["m"] = C.build_model(torch.device("cuda"), max_num_levels=16, log2_hashmap_size=16, target_num_params=18 * 2 ** 17).train()
    return _M["m"]


def _loss(rendered, gt):
    """an L1 rgb loss and its per-ray error, occupancy-masked as the trainer's error_map_ignore_not_occupied does"""
    diff = (rendered["rgb_volume"] - gt["image_rgb"]).abs()
    err = diff.mean(-1) * gt["image_occupancy_mask"].float()
    return diff.mean() + rendered["depth_volume"].mean() * 1e-3, err


def _street_poses(n_poses):
    import test_pose_refine_gpu as pr
    q0, t0 = pose64.street_poses(1, n_poses, C.ROAD_Z)
    return pr._poses(q0, t0, np.random.default_rng(2).normal(size=(n_poses, 4)) * 2e-3)


@pytest.mark.parametrize("n", [4096, 8192])
def test_graph_step_equals_host_sequence(n):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.graphics.pose import pose_rays
    from neuralsim_b200.renderer import SingleVolumeRenderer
    I = _I()
    model = _model()
    cs, specs = _cameras()
    poses = _street_poses(15)
    host_maps = [I.ErrorMap(s.error_map.n_images, (32, 64), device="cuda", n_steps_init=2) for s in cs.samplers]
    for hm, s in zip(host_maps, cs.samplers):
        hm.error_map.copy_(s.error_map.error_map)
        hm.construct_cdf()
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=_loss, near=C.NEAR, far=C.FAR, zero_grads=True, h_appear_grad=True, pose=poses, perturb=True, sampler=cs,
                     slack=2.0)

    def host(cam, s0):
        gen.set_offset(s0)
        for p in model.parameters():
            if p.grad is not None:
                p.grad.zero_()
        poses.zero_grad(set_to_none=True)
        m = host_maps[cam]
        fidx, xy = I.recipe_sample_img_pixel((m.cdf_x_cond_y, m.cdf_y, m.cdf_img), m.n_images, n, 0.5)
        W, H = specs[cam][1], specs[cam][2]
        w, h, dirs = I.recipe_pixels(xy, fidx, torch.tensor([W, H], device="cuda"), cs.intrs[cam])
        gt = {k: v[fidx, h, w] for k, v in cs.gts[cam].items()}
        codes = cs.appear_table[int(cs.table[cam, 8]) + fidx].clone().requires_grad_(True)
        o, d = pose_rays(poses, int(cs.table[cam, 7]) + fidx, dirs)
        out = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, perturb=True)).train().render(model, o, d, rays_h_appear=codes)["rendered"]
        loss, err = _loss(out, gt)
        loss.backward()
        return dict(fidx=fidx, xy=xy, gt=gt, rendered={k: v.detach().clone() for k, v in out.items()}, loss=loss.detach(), err=err.detach(),
                    grads=product_grads(model), dq=poses.dq.grad.clone(), dt=poses.dt.grad.clone(), d_codes=codes.grad.clone())

    was = torch.are_deterministic_algorithms_enabled()
    for step, cam in enumerate([0, 1, 1, 0, 0, 1]):
        s0 = gen.get_offset()
        fr.step(cam=cam)
        assert gen.get_offset() == s0 + fr.sampler_reservation + fr.rng_reservation
        assert fr.counts()["overflow"] == 0 and fr.check()
        got = dict(fidx=fr.rays_fidx.clone(), xy=fr.rays_pix.clone(), gt={k: v.clone() for k, v in fr.ground_truth.items()},
                   rendered={k: v.clone() for k, v in fr.rendered.items()}, loss=fr.loss.clone(), grads=product_grads(model), dq=poses.dq.grad.clone(),
                   dt=poses.dt.grad.clone(), d_codes=fr.d_h_appear.clone())
        maps = [(s.error_map.error_map.clone(), s.error_map.cdf_y.clone(), s.error_map.cdf_x_cond_y.clone()) for s in cs.samplers]
        h = host(cam, s0)
        h2 = host(cam, s0)
        torch.use_deterministic_algorithms(True)
        try:
            I.recipe_update_error_map(host_maps[cam].error_map, h["fidx"], h["xy"], h["err"])
        finally:
            torch.use_deterministic_algorithms(was)
        host_maps[cam].count_step()
        for k in ("fidx", "xy", "loss", "dq", "dt", "d_codes"):
            _same(got[k], h[k], f"step {step} {k}")
        for k in h["gt"]:
            _same(got["gt"][k], h["gt"][k], f"step {step} {k}")
        for k, v in h["rendered"].items():
            _same(got["rendered"][k], v, f"step {step} {k}")
        for k, v in h["grads"].items():
            if v is not None:
                e, spread = rel_l2(got["grads"][k], v), rel_l2(h2["grads"][k], v)
                assert e <= max(ORDER_REL, 2 * spread), (step, k, e, spread)
        for c, hm in enumerate(host_maps):
            _same(maps[c][0], hm.error_map, f"step {step} camera {c} error map")
            _same(maps[c][1], hm.cdf_y, f"step {step} camera {c} cdf_y")
            _same(maps[c][2], hm.cdf_x_cond_y, f"step {step} camera {c} cdf_x")
        gen.set_offset(s0 + fr.sampler_reservation + fr.rng_reservation)
    assert fr.captures == 1
    assert [s.error_map.n_steps_between_update for s in cs.samplers] == [3, 3]            # each camera rebuilt once, at its own 2nd step
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fr.step(cam=1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert fr.captures == 1


def test_negative_error_raises_at_check():
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model = _model()
    cs, _ = _cameras()
    poses = _street_poses(15)
    maps = [s.error_map.error_map.clone() for s in cs.samplers]

    def bad(rendered, gt):
        loss, err = _loss(rendered, gt)
        return loss, err - 0.5
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, 4096, loss_fn=bad, near=C.NEAR, far=C.FAR, zero_grads=True, pose=poses, sampler=cs, slack=2.0)
    fr.step(cam=0)
    with pytest.raises(RuntimeError, match="negative"):
        fr.check()
    assert fr.check()                                                # reported once
    assert not torch.equal(cs.samplers[0].error_map.error_map, maps[0]) and torch.equal(cs.samplers[1].error_map.error_map, maps[1])


def test_frame_refusals():
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model = _model()
    cs, _ = _cameras()
    with pytest.raises(RuntimeError, match="pose="):
        StaticFrame(model, 256, loss_fn=_loss, near=C.NEAR, far=C.FAR, sampler=cs)
    with pytest.raises(RuntimeError, match="pose list"):
        StaticFrame(model, 256, loss_fn=_loss, near=C.NEAR, far=C.FAR, sampler=cs, pose=_street_poses(10))
    fr = StaticFrame(model, 256, loss_fn=_loss, near=C.NEAR, far=C.FAR, sampler=cs, pose=_street_poses(15))
    for kw, match in ((dict(cam=2), "cam"), (dict(cam=None), "cam"), (dict(cam=0, dirs=torch.zeros(256, 3, device="cuda")), "cam= only")):
        with pytest.raises(RuntimeError, match=match):
            fr.step(**kw)
