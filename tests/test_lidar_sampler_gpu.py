"""The LiDAR batch drawn inside the step (csrc/lidar_sample.cu, neuralsim_b200/lidar_sampler.py), against torch's own ops on the GPU.

1. The draw.  nsb_lidar_sample equals recipe_sample_merged (the reference's sample_merged in torch ops) run on CUDA from the same
   generator state: li, the gathered lidar-local beams (the kernel run with identity transforms), ranges and rays_fidx bit for bit, and the
   offset it leaves is the generator's after the recipe's per-lidar randints -- at 8192 rays, at a size that is not a multiple of the
   block, at one ray, on frames with an empty lidar and with a truncation remainder.
2. The world rays match a float64 transform of the recipe's beams within 3 roundings of sum_j |R_ij x_j| (+ |t_i|): the kernel's three
   fp32 operations per component (csrc/lidar_sample.cu states their order), each off by at most 2^-24 of a partial sum bounded by that.
3. The step.  StaticFrame(sampler=LidarSampler, loss_on_ret=True) with LidarLoss on the 12-level LiDAR-only street model, with and
   without perturb=True, across frames of different beam counts under one capture: each replay's batch is the sampler's own draw, and its
   images, loss terms and loss are the bits of the host-sized step on that draw from the same generator state (the perturbed draws
   follow the sampler's); parameter gradients agree to the order of the fp32 atomics.  step() makes no host synchronisation.
4. An overflowed step: check() re-sizes and replays the same draw without touching the generator."""
import gc
import math

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import test_graph_ray_grad_gpu as gr
import test_partial_levels_gpu as pl
from test_lidar_loss_gpu import LIDAR_CFG
from util import rel_l2

pytestmark = pytest.mark.gpu
ORDER_REL = gr.ORDER_REL
COUNTS = [[6000, 900, 800, 700, 850], [5000, 0, 900, 800, 700], [7000, 1000, 1100, 0, 600], [0, 1200, 1300, 1250, 1100]]
WEIGHT = [0.4, 0.1, 0.1, 0.1, 0.1]                    # the shipped StreetSurf configs' lidar_weight
MOUNTS = [(0.0, 0.0, 2.2, 0.0), (1.5, 1.0, 0.8, 0.6), (1.5, -1.0, 0.8, -0.6), (-2.0, 0.7, 0.9, 2.5), (-2.0, -0.7, 0.9, -2.5)]


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(a, b), f"{what}: not bit-equal ({int((a != b).sum())} elements differ)"


def _gen(seed, offset):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    g.set_offset(offset)
    return g


def _rot_z(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def _data(seed=0):
    """5 lidars on a car driving along the street (y axis): lidar-local beams of a 64-line spinning pattern, per-frame transforms (car
    pose with a small roll / pitch / yaw, times each lidar's mount), ranges to the road plane (0 for beams that miss it)"""
    g = np.random.default_rng(seed)
    F, Ln = len(COUNTS), len(COUNTS[0])
    l2w = np.zeros((F, Ln, 3, 4))
    os_, ds, rs = [], [], []
    for f, cf in enumerate(COUNTS):
        car_R = _rot_z(0.05 * f) @ np.array([[1, 0, 0], [0, math.cos(0.01), -math.sin(0.01)], [0, math.sin(0.01), math.cos(0.01)]])
        car_t = np.array([0.3 * f, -60.0 + 12.0 * f, C.ROAD_Z])
        for li, n in enumerate(cf):
            mx, my, mz, yaw = MOUNTS[li]
            R, t = car_R @ _rot_z(yaw), car_R @ np.array([mx, my, mz]) + car_t
            l2w[f, li, :, :3], l2w[f, li, :, 3] = R, t
            elev = np.radians(g.choice(np.linspace(-17.6, 2.4, 64), n))
            azim = g.uniform(0, 2 * math.pi, n)
            d = np.stack([np.cos(elev) * np.sin(azim), np.cos(elev) * np.cos(azim), np.sin(elev)], -1).astype(np.float32)
            o = g.normal(scale=0.02, size=(n, 3)).astype(np.float32)
            dw, ow = d.astype(np.float64) @ R.T, o.astype(np.float64) @ R.T + t
            hit = dw[:, 2] < -1e-3
            r = np.where(hit, (C.ROAD_Z - ow[:, 2]) / np.where(hit, dw[:, 2], -1.0), 0.0) * (1 + 0.01 * g.normal(size=n))
            os_.append(o), ds.append(d), rs.append(np.clip(r, 0.0, 150.0).astype(np.float32))
    cat = lambda v: torch.from_numpy(np.concatenate(v)).cuda().contiguous()
    return cat(os_), cat(ds), cat(rs), torch.from_numpy(l2w.astype(np.float32)).cuda().contiguous()


_D = {}


def _sampler(n, identity=False, mode="merged_weighted"):
    from neuralsim_b200.lidar_sampler import LidarSampler
    if "d" not in _D:
        _D["d"] = _data()
    o, d, r, l2w = _D["d"]
    if identity:
        l2w = torch.zeros_like(l2w)
        l2w[..., 0, 0] = l2w[..., 1, 1] = l2w[..., 2, 2] = 1.0
    kw = dict(multi_lidar_weight=WEIGHT) if mode == "merged_weighted" else dict(lidar_sample_mode=mode)
    return LidarSampler(o, d, r, COUNTS, l2w, n, **kw)


# ===================================================================================================================== 1. the draw
@pytest.mark.parametrize("n", [8192, 1000, 1])
@pytest.mark.parametrize("mode", ["merged_weighted", "merged_equal"])
def test_kernel_equals_recipe(n, mode):
    s = _sampler(n, identity=True, mode=mode)
    if n == 8192 and mode == "merged_weighted":
        assert s.split[1][0] > int(8192 * 0.5 / 0.875) and s.split[1][1] == 0           # an empty lidar and a truncation remainder
    for f in range(s.n_frames):
        start = 1000 * f + 4 * n
        g_k, g_r = _gen(7 + f, start), _gen(7 + f, start)
        rng = torch.tensor([g_k.initial_seed(), start], dtype=torch.int64, device="cuda")
        frame = torch.tensor(f, dtype=torch.int64, device="cuda")
        out = dict(rays_o=torch.full((n, 3), float("nan"), device="cuda"), rays_d=torch.full((n, 3), float("nan"), device="cuda"),
                   ranges=torch.full((n,), float("nan"), device="cuda"), li=torch.full((n,), -1, dtype=torch.int64, device="cuda"),
                   rays_fidx=torch.full((n,), -1, dtype=torch.int64, device="cuda"))
        nxt = torch.zeros(2, dtype=torch.int64, device="cuda")
        s.launch(frame, rng, out["rays_o"], out["rays_d"], out["ranges"], out["li"], out["rays_fidx"], rng_next=nxt)
        ref = s.recipe(f, generator=g_r)
        for k in ("li", "rays_o", "rays_d", "ranges"):
            _same(out[k], ref[k], f"frame {f} n={n} {k}")
        _same(out["rays_fidx"], torch.full((n,), f, dtype=torch.int64, device="cuda"), f"frame {f} rays_fidx")
        assert nxt.tolist() == [rng[0].item(), g_r.get_offset()]
        assert g_r.get_offset() - start == s.frame_inc(f, _cap()) <= s.inc(n, _cap())
        got = s.sample(f, generator=g_k)                          # the module call: the generator moves as the recipe moved it
        assert g_k.get_offset() == g_r.get_offset()
        _same(got["li"], out["li"], "sample() li")


def _cap():
    from neuralsim_b200 import torch_rng as TR
    return TR.grid_cap(torch.device("cuda"))


# ===================================================================================================================== 2. world rays
@pytest.mark.parametrize("n", [8192, 1000])
def test_world_rays_against_float64(n):
    s, local = _sampler(n), _sampler(n, identity=True)
    for f in range(s.n_frames):
        got = s.sample(f, generator=_gen(3, 64 * f))
        ref = local.recipe(f, generator=_gen(3, 64 * f))
        _same(got["li"], ref["li"], "li")
        _same(got["ranges"], ref["ranges"], "ranges")
        T = s.l2w[f].double()[ref["li"]]                         # [n, 3, 4]
        R, t = T[..., :3], T[..., 3]
        for key, tt in (("rays_o", t), ("rays_d", torch.zeros_like(t))):
            x = ref[key].double()
            exact = (R * x.unsqueeze(-2)).sum(-1) + tt
            scale = (R.abs() * x.abs().unsqueeze(-2)).sum(-1) + tt.abs()
            err = (got[key].double() - exact).abs()
            worst = float((err / scale.clamp_min(1e-300)).max())
            assert worst <= 3.001 * 2.0 ** -24, (f, key, worst)


# ===================================================================================================================== 3. the step
_M = {}


def _model():
    if "m" not in _M:
        _M["m"] = pl._cfg3_geo12(torch.device("cuda")).train()
    return _M["m"]


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _frame(model, sampler, lidar, terms, perturb, **kw):
    from neuralsim_b200.graphics.neus_static import StaticFrame

    def loss_fn(ret, gt):
        terms.update(lidar(None, ret, ground_truth=gt))
        return sum(terms.values())
    model.zero_grad(set_to_none=True)
    gc.collect()
    return StaticFrame(model, sampler.num_rays, loss_fn=loss_fn, loss_on_ret=True, near=C.NEAR, far=C.FAR, with_rgb=False, zero_grads=True,
                       perturb=perturb, sampler=sampler, **kw)


def _host(model, lidar, o, d, ranges, it, perturb):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    for p in model.parameters():
        if p.grad is not None:
            p.grad.zero_()
    ret = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True, perturb=perturb)).train().render(
        model, o, d, return_buffer=True)
    terms = lidar(None, ret, None, {"ranges": ranges}, it=it)
    loss = sum(terms.values())
    loss.backward()
    return dict(rendered={k: v.detach().clone() for k, v in ret["rendered"].items()}, terms={k: v.detach().clone() for k, v in terms.items()},
                loss=loss.detach(), grads=_grads(model))


@pytest.mark.parametrize("perturb", [False, True])
def test_graph_step_equals_host_sized_step(perturb):
    from neuralsim_b200.loss import LidarLoss
    model = _model()
    s = _sampler(8192)
    lidar, terms = LidarLoss(**LIDAR_CFG), {}
    host_lidar = LidarLoss(**LIDAR_CFG)
    fr = _frame(model, s, lidar, terms, perturb, slack=2.0)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    for step, (f, it) in enumerate([(0, 100), (2, 100), (1, 5000), (3, 5000), (0, 12000)]):
        s0 = gen.get_offset()
        lidar.set_step(None, it)
        fr.step(frame_ind=f)
        assert gen.get_offset() == s0 + fr.sampler_reservation + fr.rng_reservation
        assert fr.counts()["overflow"] == 0 and fr.check()
        got = dict(o=fr.rays_o.clone(), d=fr.rays_d.clone(), ranges=fr.ground_truth["ranges"].clone(), li=fr.rays_li.clone(),
                   rendered={k: v.clone() for k, v in fr.rendered.items()}, terms={k: v.clone() for k, v in terms.items()}, loss=fr.loss.clone(),
                   grads=_grads(model))
        own = s.sample(f, generator=_gen(gen.initial_seed(), s0))            # the sampler's own draw from the step's generator state
        for k, v in (("o", own["rays_o"]), ("d", own["rays_d"]), ("ranges", own["ranges"]), ("li", own["li"])):
            _same(got[k], v, f"step {step} {k}")
        _same(fr.rays_fidx, torch.full_like(fr.rays_fidx, f), f"step {step} rays_fidx")
        hs = []
        for _ in range(2):
            gen.set_offset(s0 + s.frame_inc(f, _cap()))                     # the perturbed draws follow the sampler's
            hs.append(_host(model, host_lidar, got["o"], got["d"], got["ranges"], it, perturb))
        h, h2 = hs
        for k, v in h["rendered"].items():
            _same(got["rendered"][k], v, f"step {step} {k}")
        for k, v in h["terms"].items():
            _same(got["terms"][k], v, f"step {step} {k}")
        _same(got["loss"], h["loss"], f"step {step} loss")
        assert set(got["grads"]) == set(h["grads"])
        for k, v in h["grads"].items():
            e, spread = rel_l2(got["grads"][k], v), rel_l2(h2["grads"][k], v)
            assert e <= max(ORDER_REL, 2 * spread), (step, k, e, spread)
        gen.set_offset(s0 + fr.sampler_reservation + fr.rng_reservation)
    assert fr.captures == 1
    assert len({int(v) for v in (fr.sampler.split[0][0], fr.sampler.split[1][0], fr.sampler.split[3][0])}) == 3
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lidar.set_step(None, 100)
        fr.step(frame_ind=2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert fr.captures == 1


# ===================================================================================================================== 4. overflow
def test_overflow_retry_keeps_the_generator_and_the_draw():
    from neuralsim_b200.loss import LidarLoss
    model = _model()
    s = _sampler(4096)
    lidar, terms = LidarLoss(**LIDAR_CFG), {}
    fr = _frame(model, s, lidar, terms, True, march_cap=1024, kept_cap=256, coherent=False)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    s0 = gen.get_offset()
    lidar.set_step(None, 100)
    fr.step(frame_ind=1)
    assert fr.counts()["overflow"] != 0
    before = (fr.rays_o.clone(), fr.rays_d.clone(), fr.ground_truth["ranges"].clone(), fr.rays_li.clone())
    assert fr.check() is False
    after = (fr.rays_o, fr.rays_d, fr.ground_truth["ranges"], fr.rays_li)
    assert fr.counts()["overflow"] == 0 and gen.get_offset() == s0 + fr.sampler_reservation + fr.rng_reservation
    for k, a, b in zip(("rays_o", "rays_d", "ranges", "li"), before, after):
        _same(b, a, f"retry {k}")
    gen.set_offset(s0 + s.frame_inc(1, _cap()))
    h = _host(model, LidarLoss(**LIDAR_CFG), before[0], before[1], before[2], 100, True)
    for k, v in h["rendered"].items():
        _same(fr.rendered[k], v, k)
    _same(fr.loss, h["loss"], "loss")
    gen.set_offset(s0 + fr.sampler_reservation + fr.rng_reservation)


def test_frame_refusals():
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model = _model()
    s = _sampler(256)
    lf = lambda ret, gt: ret["rendered"]["depth_volume"].mean()
    with pytest.raises(RuntimeError, match="with_rgb=False"):
        StaticFrame(model, 256, loss_fn=lf, near=C.NEAR, far=C.FAR, sampler=s)
    with pytest.raises(RuntimeError, match="loss_fn"):
        StaticFrame(model, 256, near=C.NEAR, far=C.FAR, with_rgb=False, sampler=s)
    with pytest.raises(RuntimeError, match="num_rays"):
        StaticFrame(model, 512, loss_fn=lf, near=C.NEAR, far=C.FAR, with_rgb=False, sampler=s)
    fr = StaticFrame(model, 256, loss_fn=lf, near=C.NEAR, far=C.FAR, with_rgb=False, sampler=s)
    for kw, match in ((dict(frame_ind=4), "frame_ind"), (dict(), "frame_ind"), (dict(frame_ind=0, cam=0), "frame_ind= only"),
                      (dict(frame_ind=0, rays_o=torch.zeros(256, 3, device="cuda")), "frame_ind= only")):
        with pytest.raises(RuntimeError, match=match):
            fr.step(**kw)
