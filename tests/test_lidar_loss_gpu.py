"""The StreetSurf LiDAR loss on the fused kernels (csrc/lidar_loss.cu, neuralsim_b200/loss/lidar.py): the device median against torch.sort,
the loss terms and their cotangents against the float64 restatement (oracle/lidar64.py) on capacity-sized buffers with device counts, the
host-sized render with the fused loss against the reference's torch formulation, and the loss inside the one-launch step
(`StaticFrame(loss_on_ret=True)`) against the host-sized step.

Bounds.  The terms are fp64 sums of fp32 rows rounded once, so they are within a few fp32 ulp of float64 (FWD_REL = 1e-6).  Each cotangent
element is two to six correctly rounded fp32 operations away from its float64 value (GRAD_RTOL = 1e-6, about 8 ulp).  The fused loss and
the reference's torch formulation see the same rendered buffers and differ in the loss's last bits only, so the parameter gradients are
held to tests/test_cfg3_gpu.py's fused-vs-module bound (2e-2 rel-L2) and the terms to FWD_REL.  The graph step runs the host-sized
path's kernels on the same samples: its rendered buffers, loss terms and loss are compared bit for bit.  Its parameter gradients are sums of
fp32 atomics whose order differs from run to run on either path, so they are held to ORDER_REL, or twice the spread of two host-sized
runs (tests/test_graph_ray_grad_gpu.py does the same)."""
import gc
import json

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import test_graph_ray_grad_gpu as gr
import test_partial_levels_gpu as pl
from oracle import lidar64
from util import rel_l2

pytestmark = pytest.mark.gpu

FWD_REL = 1e-6
GRAD_RTOL = 1e-6
MODULE_REL = 2e-2
ORDER_REL = gr.ORDER_REL
LIDAR_CFG = dict(discard_outliers=0, discard_outliers_median=100.0, discard_toofar=80.0, depth=dict(w=0.05, fn_type="l1"),
                 line_of_sight=dict(w=0.1, fn_type="neus_unisim", fn_param=dict(epsilon_anneal=dict(type="milestones", milestones=[5000, 10000],
                                                                                                     vals=[1.5, 0.75, 0.5]))))


def _kth(v, k):
    from neuralsim_b200 import _lib as L
    lib = L.lib()
    out = torch.full((1,), -1.0, device=v.device)
    scratch = torch.empty(int(lib.nsb_kth_smallest_scratch_bytes()), dtype=torch.uint8, device=v.device)
    L.call(lib.nsb_kth_smallest, "kth_smallest", L.ptr(v, "f32"), L.c_i64(v.numel()), L.c_i64(k), L.ptr(out), L.ptr(scratch), L.stream_ptr())
    return out


@pytest.mark.parametrize("R", [1, 2, 3, 8191, 8192, 8193, 2 ** 20 + 3])
@pytest.mark.parametrize("kind", ["ties", "zeros", "inf", "nan", "nan-median"])
def test_median_bit_equal_to_torch_sort(cuda, R, kind):
    g = torch.Generator(device=cuda).manual_seed(R)
    v = torch.randint(0, 40, (R,), device=cuda, generator=g).float() / 8         # heavy ties
    if kind == "zeros":
        v[torch.rand(R, device=cuda, generator=g) < 0.6] = 0.0
    elif kind == "inf":
        v[torch.rand(R, device=cuda, generator=g) < 0.3] = float("inf")
    elif kind == "nan":
        v[torch.rand(R, device=cuda, generator=g) < 0.3] = float("nan")
    elif kind == "nan-median":
        v[torch.rand(R, device=cuda, generator=g) < 0.7] = float("nan")
        v[:1] = 0.0
    want = torch.sort(v).values[R // 2:R // 2 + 1]
    got = _kth(v, R // 2)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (R, kind, float(got), float(want))
    if R > 2:
        for k in (0, R - 1):
            assert torch.equal(_kth(v, k).view(torch.int32), torch.sort(v).values[k:k + 1].view(torch.int32)), k


# ===================================================================================================================== against float64
def _packed_static(cuda, R, n_hit, n_per, kept_cap, seed=0):
    """capacity-sized buffers as the graph step leaves them: n_hit kept rays of n_per samples, rows past the counts NaN / garbage"""
    rng = np.random.default_rng(seed)
    gt = rng.uniform(1, 100, R).astype(np.float32)
    gt[::17] = 0.0
    pred = (gt + rng.normal(0, 2, R)).astype(np.float32)
    pred[5] = gt[5] + 500.0                                  # an outlier
    mask_pred = rng.uniform(0, 1, R).astype(np.float32)
    mask_pred[::13] = 0.0
    rih = np.sort(rng.choice(R, n_hit, replace=False)).astype(np.int64)
    K = n_hit * n_per
    t = np.concatenate([gt[r] + rng.normal(0, 2, n_per) for r in rih]).astype(np.float32) if K else np.zeros(0, np.float32)
    if K:
        t[0] = gt[rih[0]] + np.float32(1.5)                 # a sample at |t - gt| = eps, up to the rounding of t
    vw = rng.uniform(0, 0.3, K).astype(np.float32)
    pinfo = np.stack([np.arange(n_hit) * n_per, np.full(n_hit, n_per)], -1).astype(np.int64)
    T = torch.full((kept_cap,), float("nan"), device=cuda)
    V = torch.full((kept_cap,), float("nan"), device=cuda)
    T[:K], V[:K] = torch.from_numpy(t).to(cuda), torch.from_numpy(vw).to(cuda)
    PI = torch.full((R, 2), 1 << 40, dtype=torch.int64, device=cuda)
    RI = torch.full((R,), 1 << 40, dtype=torch.int64, device=cuda)
    PI[:n_hit], RI[:n_hit] = torch.from_numpy(pinfo).to(cuda), torch.from_numpy(rih).to(cuda)
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS
    cnt = torch.zeros(32, dtype=torch.int64, device=cuda)
    cnt[CNT_SLOTS["kept_rays"]], cnt[CNT_SLOTS["kept"]] = n_hit, K
    np_case = dict(pred=pred, mask_pred=mask_pred, gt=gt, t=t, vw=vw, pinfo=pinfo, rih=rih)
    V.requires_grad_(True)
    vb = dict(type="packed_static", t=T, vw=V, rays_inds_hit=RI, pack_infos_hit=PI, ridx=None, cnt=cnt, CNT_SLOTS=CNT_SLOTS)
    return np_case, vb, torch.from_numpy(pred).to(cuda).requires_grad_(True), torch.from_numpy(mask_pred).to(cuda), torch.from_numpy(gt).to(cuda)


def _run_fused(lidar, vb, pred, mask_pred, gt, it):
    lidar.set_step(gt, it)
    out = lidar(None, dict(rendered=dict(depth_volume=pred, mask_volume=mask_pred), volume_buffer=vb))
    sum(out.values()).backward()
    return out


@pytest.mark.parametrize("n_per", [1, 31, 32, 33])
@pytest.mark.parametrize("fn_type", ["l1", "l2_relative"])
def test_terms_and_cotangents_against_float64(cuda, n_per, fn_type):
    from neuralsim_b200.loss import LidarLoss
    cfg = dict(LIDAR_CFG, depth=dict(w=0.05, fn_type=fn_type))
    R, n_hit, kept_cap = 3000, 1700, 1700 * n_per + 999
    case, vb, pred, mask_pred, gt = _packed_static(cuda, R, n_hit, n_per, kept_cap, seed=n_per)
    lidar = LidarLoss(**cfg)
    out = _run_fused(lidar, vb, pred, mask_pred, gt, it=100)
    o = lidar64.lidar_loss(case["pred"], case["mask_pred"], case["gt"], case["t"], case["vw"], case["pinfo"], case["rih"], fn_type=fn_type, w_depth=0.05,
                           w_los=0.1, epsilon=1.5, discard_toofar=80.0, median_factor=100.0)
    assert np.array_equal(lidar.mask.bool().cpu().numpy(), o["mask"])
    assert not o["mask"][5] and o["los"] > 0 and o["depth"] > 0
    d, s = float(out["lidar_loss.depth"].detach()), float(out["lidar_loss.los.empty"].detach())
    rep = dict(depth=abs(d - o["depth"]) / o["depth"], los=abs(s - o["los"]) / o["los"])
    print("METRIC lidar terms vs f64", json.dumps(dict(n_per=n_per, fn=fn_type, **rep)))
    assert rep["depth"] <= FWD_REL and rep["los"] <= FWD_REL, rep
    # l2_relative's gradient is the sum of two terms, 2 g d / den and -2 g d^2 x / den^2, that can cancel: the bound is relative to their
    # magnitudes (each rounds within a few ulp), not to their sum
    x, y = case["pred"].astype(np.float64), case["gt"].astype(np.float64)
    d, den = x - y, x * x + 1e-2
    g = 0.05 * o["mask"] / R
    scale = np.abs(o["g_depth"]) if fn_type == "l1" else g * (np.abs(2 * d / den) + np.abs(2 * d * d * x / (den * den)))
    err = np.abs(pred.grad.cpu().numpy().astype(np.float64) - o["g_depth"])
    assert bool(np.all(err <= GRAD_RTOL * scale + 1e-30)), float(np.max(err / (scale + 1e-30)))
    K = n_hit * n_per
    g_vw = vb["vw"].grad
    np.testing.assert_allclose(g_vw[:K].cpu().numpy(), o["g_vw"], rtol=GRAD_RTOL, atol=1e-30)
    assert bool((g_vw[K:] == 0).all())                       # capacity rows past the kept samples: untouched (zero-filled)


def test_no_kept_ray_gives_zero_line_of_sight(cuda):
    from neuralsim_b200.loss import LidarLoss
    case, vb, pred, mask_pred, gt = _packed_static(cuda, 500, 0, 4, 4096)
    lidar = LidarLoss(**LIDAR_CFG)
    out = _run_fused(lidar, vb, pred, mask_pred, gt, it=0)
    assert float(out["lidar_loss.los.empty"]) == 0.0 and float(out["lidar_loss.depth"]) > 0
    assert not bool(vb["vw"].grad.any())
    o = lidar64.lidar_loss(case["pred"], case["mask_pred"], case["gt"], fn_type="l1", w_depth=0.05, discard_toofar=80.0)
    assert abs(float(out["lidar_loss.depth"]) - o["depth"]) <= FWD_REL * o["depth"]


def test_loss_reads_nothing_back_to_the_host(cuda):
    """the loss forward and backward on capacity-sized buffers under torch's sync debug mode, at a size that takes the multi-CTA median"""
    from neuralsim_b200.loss import LidarLoss
    _, vb, pred, mask_pred, gt = _packed_static(cuda, (1 << 16) + 5, 3000, 8, 40000)
    lidar = LidarLoss(**LIDAR_CFG)
    lidar.set_step(gt, 0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = _run_fused(lidar, vb, pred, mask_pred, gt, it=7000)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert float(out["lidar_loss.los.empty"]) > 0


@pytest.mark.parametrize("kind", ["batched", "nerf_buffer"])
def test_unbuilt_buffer_types_raise(cuda, kind):
    from neuralsim_b200.loss import LidarLoss
    _, vb, pred, mask_pred, gt = _packed_static(cuda, 64, 8, 2, 64)
    vb = dict(vb, type="batched" if kind == "batched" else "nerf_buffer")
    with pytest.raises(RuntimeError, match=vb["type"]):
        LidarLoss(**LIDAR_CFG)(None, dict(rendered=dict(depth_volume=pred, mask_volume=mask_pred), volume_buffer=vb), None, {"ranges": gt}, it=0)


# ===================================================================================================================== rendered rays
def _ranges(model, lo, ld, cfg, seed=0):
    """LiDAR returns near the model's surface: the rendered depth with noise, some rays without a return and some beyond discard_toofar"""
    from neuralsim_b200.renderer import SingleVolumeRenderer
    with torch.no_grad():
        d = SingleVolumeRenderer(cfg).train().render(model, lo, ld)["rendered"]["depth_volume"]
    g = torch.Generator(device=lo.device).manual_seed(seed)
    r = d * (1 + 0.05 * torch.randn(d.shape, device=d.device, generator=g)) + 0.5 * torch.randn(d.shape, device=d.device, generator=g)
    r = r.clamp_min(0.5)
    r[::17] = 0.0
    r[::23] = 120.0
    return r


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _host_step(model, lidar, lo, ld, ranges, it, cfg, torch_loss=False):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    for p in model.parameters():                            # in place: a captured step keeps accumulating into these tensors
        if p.grad is not None:
            p.grad.zero_()
    ret = SingleVolumeRenderer(cfg).train().render(model, lo, ld, return_buffer=True)
    terms = _torch_lidar(ret, ranges, it) if torch_loss else lidar(None, ret, None, {"ranges": ranges}, it=it)
    loss = sum(terms.values())
    loss.backward()
    return {k: v.detach().clone() for k, v in ret["rendered"].items()}, {k: v.detach().clone() for k, v in terms.items()}, loss.detach(), _grads(model)


def _torch_lidar(ret, ranges, it):
    """the reference's LidarLoss.forward (l1 depth, neus_unisim line of sight, the shipped settings) in plain torch"""
    depth_pred, mask_pred = ret["rendered"]["depth_volume"], ret["rendered"]["mask_volume"]
    gt = ranges.view(depth_pred.shape)
    mask = gt <= 80.0
    err = (depth_pred - gt).abs() * mask
    sv, _ = torch.sort(err.data)
    mask[err > sv[depth_pred.numel() // 2] * 100.0] = False
    out = {"lidar_loss.depth": 0.05 * ((depth_pred - gt).abs() * mask).mean()}
    vb = ret["volume_buffer"]
    rih, t, vw, pi = vb["rays_inds_hit"], vb["t"], vb["vw"], vb["pack_infos_hit"]
    eps = _eps(it)
    gt_ex = torch.repeat_interleave(gt[rih], pi[:, 1], dim=0)
    per = torch.zeros(pi.shape[0], device=vw.device).index_add(0, torch.repeat_interleave(torch.arange(pi.shape[0], device=vw.device), pi[:, 1]),
                                                               ((t - gt_ex).abs() > eps) * vw ** 2)
    out["lidar_loss.los.empty"] = 0.1 * (per * mask[rih]).mean()
    return out


def _eps(it):
    from neuralsim_b200.loss.lidar import anneal_milestones
    return anneal_milestones(it, [5000, 10000], [1.5, 0.75, 0.5])


def test_host_sized_fused_loss_against_torch_formulation(cuda):
    from neuralsim_b200.loss import LidarLoss
    model = C.build_model(cuda).train()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    lo, ld = (x.to(cuda) for x in C.lidar_rays(1, C.N_LIDAR))
    ranges = _ranges(model, lo, ld, cfg)
    lidar = LidarLoss(**LIDAR_CFG)
    r_f, t_f, _, g_f = _host_step(model, lidar, lo, ld, ranges, 100, cfg)
    r_t, t_t, _, g_t = _host_step(model, lidar, lo, ld, ranges, 100, cfg, torch_loss=True)
    for k in r_f:
        assert torch.equal(r_f[k], r_t[k]), k
    rep = {k: abs(float(t_f[k]) - float(t_t[k])) / abs(float(t_t[k])) for k in t_t}
    assert all(float(v) > 0 for v in t_t.values())
    assert all(v <= FWD_REL * 10 for v in rep.values()), rep
    grel = {k: rel_l2(g_f[k], g_t[k]) for k in g_t}
    print("METRIC lidar host fused vs torch", json.dumps(dict(terms=rep, grads=grel)))
    assert set(g_f) == set(g_t) and all(v <= MODULE_REL for v in grel.values()), grel


def _frame_case(model, cfg, n=4096, seed=1):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.loss import LidarLoss
    lo, ld = (x.to(model.device) for x in C.lidar_rays(seed, n))
    ranges = _ranges(model, lo, ld, cfg)
    lidar = LidarLoss(**LIDAR_CFG)
    terms = {}

    def loss_fn(ret):
        terms.update(lidar(None, ret))
        return sum(terms.values())
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=loss_fn, loss_on_ret=True, near=cfg["near"], far=cfg["far"], with_rgb=False, with_normal=cfg["with_normal"],
                     zero_grads=True)
    return fr, lidar, terms, lo, ld, ranges


def _compare_to_host(model, fr, lidar, terms, lo, ld, ranges, it, cfg, what):
    host = _host_step(model, lidar, lo, ld, ranges, it, cfg)
    host2 = _host_step(model, lidar, lo, ld, ranges, it, cfg)
    lidar.set_step(ranges, it)
    fr.step(lo, ld)
    assert fr.counts()["overflow"] == 0
    for k, v in host[0].items():
        gr._same(fr.rendered[k], v, f"{what} {k}")
    for k, v in host[1].items():
        gr._same(terms[k], v, f"{what} {k}")
    gr._same(fr.loss, host[2], f"{what} loss")
    g = _grads(model)
    rep = {}
    for k, v in host[3].items():
        rep[k] = (rel_l2(g[k], v), rel_l2(host2[3][k], v))
        assert rep[k][0] <= max(ORDER_REL, 2 * rep[k][1]), (what, k, rep[k])
    print("METRIC lidar graph vs host", json.dumps(dict(what=what, terms={k: float(v) for k, v in host[1].items()}, grads=rep)))
    return {k: v.clone() for k, v in terms.items()}


@pytest.mark.parametrize("which", ["cfg3-colour-16", "lidar-only-12"])
def test_graph_step_bit_equal_to_host_sized_and_follows_replays(cuda, which):
    """the fused loss inside the captured step: rendered buffers, both terms and the loss are the host-sized step's bits; new ranges and an
    epsilon milestone reach the replay through set_step without a re-capture"""
    model = (C.build_model(cuda) if which == "cfg3-colour-16" else pl._cfg3_geo12(cuda)).train()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    fr, lidar, terms, lo, ld, ranges = _frame_case(model, cfg)
    a = _compare_to_host(model, fr, lidar, terms, lo, ld, ranges, 100, cfg, "first")
    assert all(float(v) > 0 for v in a.values())
    ranges2 = ranges.flip(0).contiguous()
    b = _compare_to_host(model, fr, lidar, terms, lo, ld, ranges2, 100, cfg, "new ranges")
    assert not torch.equal(b["lidar_loss.depth"], a["lidar_loss.depth"])
    c = _compare_to_host(model, fr, lidar, terms, lo, ld, ranges2, 5000, cfg, "milestone")
    assert torch.equal(c["lidar_loss.depth"], b["lidar_loss.depth"])
    assert not torch.equal(c["lidar_loss.los.empty"], b["lidar_loss.los.empty"])
    assert fr.captures == 1


def test_static_step_with_loss_has_no_host_read(cuda):
    """the static (non-graph) step with the loss, after its first call sized the arenas, under torch's sync debug mode"""
    model = C.build_model(cuda).train()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    fr, lidar, terms, lo, ld, ranges = _frame_case(model, cfg, n=2048)
    fr.use_graph = False
    lidar.set_step(ranges, 100)
    fr.step(lo, ld)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lidar.set_step(ranges, 100)
        fr.step(lo, ld)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert float(terms["lidar_loss.los.empty"]) > 0
