"""LoTD tables of L = 1..15 levels (2 features each) on the wgmma kernels: k_fused_sdf_tc, k_sdf_bwd_tc, k_upsample_persistent,
k_color_fwd<true|false>, k_color_rad_bwd and k_color_sdf_bwd take L from the meta, gather and scatter only levels < L and write zero
feature columns 2L..31.

1. Kernels against the float64 reference (oracle/fused64.py through tests/fused64_levels.py) at L in {1, 2, 7, 11, 12, 15}, with and without max_level, at 1, 127, 128
   and 129 points and at a size where every persistent CTA loops over three or more tiles, with a device count below the capacity.  The
   fp16 table and the W1 image sit at the start of allocations whose tails are fp16 NaN: a read past the table or past column 2L of W1
   would show as a non-finite output.  The persistent up-sampling kernel at 12 levels is bit-equal to the stage kernels.
2. Models: the LiDAR-only StreetSurf configuration at 12 levels on the cfg3 box (fused == chain, graph step == host-sized step), the
   colour model at 12 levels on camera rays, extract_mesh and adapter.accelerate at 12 levels, and which tables the predicates accept."""
import ctypes

import numpy as np
import pytest
import torch

import bench_cfg3 as C
from fused64_levels import Fused64Levels
from oracle import lotd as olotd
from test_geometry_only_gpu import _launch
from test_tc_kernels_gpu import (BWD_REL, NAB_FRAC_1E5, NAB_MAX_REL, RGB_FLIP_FRAC, RGB_MAX_ULP, SDF_FLIP_FRAC, SDF_MAX_ULP, TILE, _fp16_metrics,
                                 _inputs, _rel, _sms)
from util import rel_l2

pytestmark = pytest.mark.gpu

LEVELS = [1, 2, 7, 11, 12, 15]
CASES = [(L, ml) for L in LEVELS for ml in (None, L - 3) if ml is None or ml >= 0]
SDF_KEYS = ("grid", "W1", "b1", "W2", "b2")


def _model(levels, seed, n_appear=4, radiance=True):
    from neuralsim_b200.fields.neus import LoTDNeuS
    gen = torch.Generator("cuda").manual_seed(seed)
    model = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg(log2_hashmap_size=16, num_levels=levels)),
                                      decoder_cfg=dict(W=64)),
                     radiance_cfg=dict(W=64, n_appear_embedding=n_appear) if radiance else False, device="cuda", generator=gen)
    with torch.no_grad():
        model.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=gen)
    s = model.implicit_surface
    assert s.encoding.meta.n_pseudo_levels == levels and tuple(s.decoder.layers[0].weight.shape) == (64, 2 * levels)
    assert s._fusable() and (model._color_fusable() if radiance else model._geometry_fusable())
    return model


def _nan_tailed(t, extra=1 << 16):
    """t copied to the start of an allocation whose remaining `extra` elements are fp16 NaN"""
    buf = torch.full((t.numel() + extra,), float("nan"), dtype=torch.half, device=t.device)
    buf[:t.numel()].copy_(t.reshape(-1))
    return buf[:t.numel()].view(t.shape)


def _install_nan_tails(model):
    """replace the cached fp16 images of the table and of W1 (the fused SDF, colour and geometry states) by NaN-tailed copies"""
    from neuralsim_b200.fields.fused_color import color_net_c
    from neuralsim_b200.fields.networks import sdf_decoder_c
    s = model.implicit_surface
    s._fused_state()
    key, t, _ = s._fused_cache
    t = [_nan_tailed(t[0]), _nan_tailed(t[1])] + list(t[2:])
    s._fused_cache = (key, t, sdf_decoder_c(t[1:], s.decoder.layers))
    model._geo_cache = None
    if model.radiance_net is not None:
        model._fused_color_state()
        key, tc, _ = model._color_cache
        tc = [_nan_tailed(tc[0])] + list(tc[1:])
        model._color_cache = (key, tc, color_net_c(tc, s.decoder.layers, model.radiance_net.blocks.layers, model._nablas_fac()))


def _params(model):
    s, r = model.implicit_surface, model.radiance_net.blocks.layers
    d = s.decoder.layers
    return dict(grid=s.encoding.flattened_params, W1=d[0].weight, b1=d[0].bias, W2=d[1].weight, b2=d[1].bias, R1=r[0].weight,
                rb1=r[0].bias, R2=r[1].weight, rb2=r[1].bias, R3=r[2].weight, rb3=r[2].bias)


def _run_all(model, inp, ml):
    """every kernel once on the points of `inp`: the fused SDF query (points, rays), its backward, the colour forward (full and geometry-only)
    and the colour backward -> dict of numpy outputs and gradients"""
    s = model.implicit_surface
    model.max_level = ml
    x, ridx, t, o, d, v, ha = (inp[k].cuda() for k in ("x", "ridx", "t", "o", "d", "v", "ha"))
    c_sdf, c_nab, c_rgb = (c.cuda() for c in inp["cot"])
    with torch.no_grad():
        out = dict(sdf_pts=s.fused_sdf(x, max_level=ml), sdf_rays=s.fused_sdf_rays(ridx, t, o, d, max_level=ml))
        geo = model.forward_on_rays(ridx, t, o, d, with_rgb=False)
    out["geo_sdf"], out["geo_nablas"] = geo["sdf"], geo["nablas"]
    p = _params(model)
    sdf = s.fused_sdf_autograd(x, max_level=ml)
    out["sdf_bwd"] = dict(zip(SDF_KEYS, torch.autograd.grad((sdf * c_sdf).sum(), [p[k] for k in SDF_KEYS])))
    col = model.forward_on_rays(ridx, t, o, d, v, ha)
    out["sdf"], out["nablas"], out["rgb"] = col["sdf"].detach(), col["nablas"].detach(), col["rgb"].detach()
    loss = (col["sdf"] * c_sdf).sum() + (col["nablas"] * c_nab).sum() + (col["rgb"] * c_rgb).sum()
    out["color_bwd"] = dict(zip(p, torch.autograd.grad(loss, list(p.values()))))
    model.max_level = None
    for k, g in list(out["sdf_bwd"].items()) + list(out["color_bwd"].items()):
        assert bool(torch.isfinite(g).all()), k
    return {k: ({kk: vv.detach().double().cpu().numpy() for kk, vv in v.items()} if isinstance(v, dict) else v.cpu().numpy())
            for k, v in out.items()}


def _check(got, ref, inp, full_metrics):
    """got (_run_all) against the float64 reference: the 16-level tests' bounds; with few points only the per-element bounds (one
    flip among 129 values already exceeds a flip-fraction bound)"""
    fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy())
    for k in ("sdf_pts", "sdf_rays", "geo_sdf", "sdf", "nablas", "rgb", "geo_nablas"):
        assert np.isfinite(got[k]).all(), k
    for k in ("sdf_pts", "sdf_rays", "geo_sdf", "sdf"):
        frac, ulp = _fp16_metrics(got[k], fwd["sdf"], fwd["sdf_scale"])
        assert ulp <= SDF_MAX_ULP and (not full_metrics or frac <= SDF_FLIP_FRAC), (k, frac, ulp)
    frac, ulp = _fp16_metrics(got["rgb"], fwd["rgb"], 0.5)
    assert ulp <= RGB_MAX_ULP and (not full_metrics or frac <= RGB_FLIP_FRAC), ("rgb", frac, ulp)
    for k in ("nablas", "geo_nablas"):
        nab = np.abs(got[k] - fwd["nablas"]) / (fwd["nablas_scale"] + 1e-30)
        assert float(nab.max()) <= NAB_MAX_REL and (not full_metrics or float((nab > 1e-5).mean()) <= NAB_FRAC_1E5), (k, nab.max())
    assert np.array_equal(got["geo_sdf"], got["sdf"]) and np.array_equal(got["geo_nablas"], got["nablas"])
    if not full_metrics and inp["x"].shape[0] < TILE + 1:
        return
    want = ref.color_backward(fwd, *(c.numpy() for c in inp["cot"]))
    for k, w in want.items():
        e = _rel(got["color_bwd"][k].reshape(w.shape), w)
        assert e < BWD_REL[k], ("color_bwd", k, e)
    want = ref.sdf_backward(inp["x"].numpy(), inp["cot"][0].numpy())
    for k in SDF_KEYS:
        e = _rel(got["sdf_bwd"][k].reshape(want[k].shape), want[k])
        assert e < BWD_REL[k], ("sdf_bwd", k, e)


# ===================================================================================================================== 1. kernels
@pytest.mark.parametrize("levels,max_level", CASES, ids=[f"L{L}-ml{ml}" for L, ml in CASES])
def test_kernels_against_float64_small_sizes(levels, max_level):
    model = _model(levels, seed=levels)
    _install_nan_tails(model)
    ref = Fused64Levels.from_model(model, max_level=max_level)
    assert ref.nh == 2 * levels
    for n in (1, 127, 128, 129):
        inp = _inputs(n, 4, seed=n + levels)
        _check(_run_all(model, inp, max_level), ref, inp, full_metrics=False)


@pytest.mark.parametrize("levels,max_level", [(11, None), (11, 8), (12, None), (12, 9)])
def test_kernels_against_float64_multi_tile(levels, max_level):
    """every CTA of every persistent grid loops over three or more tiles (4 CTAs / SM is the largest grid: k_fused_sdf_tc, k_sdf_bwd_tc)"""
    model = _model(levels, seed=100 + levels)
    _install_nan_tails(model)
    n = (3 * _sms() * 4 + 1) * TILE - 51
    assert -(-n // TILE) >= 3 * _sms() * 4 and n % TILE
    inp = _inputs(n, 4, seed=levels)
    ref = Fused64Levels.from_model(model, max_level=max_level)
    _check(_run_all(model, inp, max_level), ref, inp, full_metrics=True)


def test_colour_forward_device_count_below_capacity():
    model = _model(12, seed=3)
    _install_nan_tails(model)
    n = (2 * _sms() * 2 + 1) * TILE - 51
    live = n - _sms() * TILE - 37
    inp = _inputs(n, 4, seed=5)
    for rad in (True, False):
        full = _launch(model, inp, rad)
        part = _launch(model, inp, rad, count=live)
        for k in ("sdf", "nablas", "x"):
            assert torch.equal(full[k][:live], part[k][:live]), (rad, k)
            assert bool(torch.isnan(part[k][live:]).all()), (rad, k)
        assert bool(torch.isfinite(part["sdf"][:live]).all() and torch.isfinite(part["nablas"][:live]).all())


def test_upsample_persistent_at_12_levels_equals_stage_kernels():
    from test_ray_upsample_edges_gpu import LAYOUTS, Rays, _chain, _kernel
    model = _model(12, seed=9).train()
    surf = model.implicit_surface
    _install_nan_tails(model)
    layout = next(iter(LAYOUTS))
    R = Rays(12)
    for k in range(3 * _sms() * 2):
        R.add("hit", int(R.rng.integers(8, 200)))
    rt = R.tensors()
    rows = np.arange(len(R.n))
    for ml in (None, 9):
        with torch.no_grad():
            ref, _, _, _ = _chain(surf, rt, rows, layout, ml=surf._ml(ml), est=False, thre=0.0)
            got, ovf = _kernel(surf, rt, layout, ml=surf._ml(ml), est=False, thre=0.0, entry="wrapper")
        assert int(ovf.sum()) == 0 and bool(torch.isfinite(ref).all())
        assert torch.equal(got, ref), ml


# ===================================================================================================================== 2. models
def test_fusable_predicates():
    for levels in (1, 11, 12, 16):
        m = _model(levels, seed=levels, n_appear=0)
        assert m.implicit_surface._fusable() and m._color_fusable() and m._geometry_fusable()
    from neuralsim_b200.fields.neus import LoTDNeuS
    m17 = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg(log2_hashmap_size=14, num_levels=17))),
                   radiance_cfg=dict(W=64, n_appear_embedding=0), device="cuda")
    assert not m17.implicit_surface._fusable() and not m17._color_fusable() and not m17._geometry_fusable()
    wide = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg(log2_hashmap_size=14, num_levels=12))),
                    radiance_cfg=dict(W=64, n_appear_embedding=9), device="cuda")          # 22 + 24 + 9 inputs: more than 8 appearance channels
    assert wide.implicit_surface._fusable() and not wide._color_fusable()


def _cfg3_geo12(cuda):
    """bench_cfg3's street model at 12 levels (the shipped LiDAR-only table count) with a small hashmap and radiance_cfg=False"""
    from neuralsim_b200.fields import LoTDNeuSModel
    gen = torch.Generator(device=cuda).manual_seed(42)
    model = LoTDNeuSModel(
        surface_cfg=dict(aabb=C.AABB, sdf_scale=C.SDF_SCALE,
                         encoding_cfg=dict(lotd_use_cuboid=True,
                                           lotd_auto_compute_cfg=dict(type="ngp", target_num_params=14 * 2 ** 17, min_res=16, n_feats=2,
                                                                      log2_hashmap_size=16, max_num_levels=12),
                                           param_init_cfg=dict(type="uniform_to_type", bound=2.0e-3))),
        radiance_cfg=False,
        var_ctrl_cfg=dict(ln_inv_s_init=0.5298, ln_inv_s_factor=10.0),
        accel_cfg=dict(vox_size=1.0, occ_val_fn_cfg=dict(type="sdf", inv_s=256.0), occ_thre=0.3, ema_decay=0.95, update_from_samples_cfg=None),
        ray_query_cfg=dict(query_mode="march_occ_multi_upsample_compressed", query_param=dict(
            nablas_has_grad=True, num_coarse=128, num_fine=[8, 8, 32], coarse_step_cfg=dict(step_mode="linear"),
            march_cfg=dict(step_size=0.2, max_steps=4096), upsample_inv_s=64.0, upsample_inv_s_factors=[1, 4, 16],
            upsample_use_estimate_alpha=False)),
        device=cuda, generator=gen)
    C.install_plane(model, C.ROAD_Z)
    assert model.implicit_surface.encoding.meta.n_pseudo_levels == 12 and model.radiance_net is None and model._geometry_fusable()
    return model.train()


def _render(model, r, rays, fused, ha=None, loss=C.loss_lidar):
    import neuralsim_b200.graphics.neus as GN
    import neuralsim_b200.fields.space as SP
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.fields.networks import LoTDSDF
    model.zero_grad(set_to_none=True)
    saved = (GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable)
    if not fused:
        GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable = False, False, (lambda self: False)
    L.KERNEL_TIMER.enable()
    try:
        out = r.render(model, *rays, rays_h_appear=ha)["rendered"] if ha is not None else r.render(model, *rays)["rendered"]
        loss(out).backward()
        launched = L.KERNEL_TIMER.summary()
    finally:
        L.KERNEL_TIMER.disable()
        GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable = saved
    s = model.implicit_surface
    grads = (s.encoding.flattened_params.grad.clone(), s.decoder.layers[0].weight.grad.clone())
    return {k: v.detach().clone() for k, v in out.items()}, grads, launched


def _fused_vs_chain_and_static(model, rays, ha, with_rgb, loss, keys):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=with_rgb, with_normal=True)).train()
    a, ga, launched = _render(model, r, rays, True, ha, loss)
    assert "fused_color_fwd" in launched and ("fused_sdf_fwd" in launched or "ray_upsample" in launched), sorted(launched)
    b, gb, _ = _render(model, r, rays, False, ha, loss)
    assert float(a["mask_volume"].sum()) > 100
    for k in keys:
        assert rel_l2(a[k], b[k]) <= 1e-4, (k, rel_l2(a[k], b[k]))
    for x, y in zip(ga, gb):
        assert rel_l2(x, y) <= 2e-2, rel_l2(x, y)
    # the one-launch graph step: images bit-equal to the host-sized step, gradients to fp32 summation order
    n = rays[0].shape[0]
    model.zero_grad(set_to_none=True)
    fr = StaticFrame(model, n, loss_fn=loss, near=C.NEAR, far=C.FAR, with_rgb=with_rgb, slack=2.0, zero_grads=True)
    fr.step(*rays, ha)
    assert fr.counts()["overflow"] == 0 and fr.captures == 1
    assert set(fr.rendered) == set(a)
    for k, v in a.items():
        assert torch.equal(fr.rendered[k], v), k
    s = model.implicit_surface
    assert rel_l2(s.encoding.flattened_params.grad, ga[0]) <= 2e-5 and rel_l2(s.decoder.layers[0].weight.grad, ga[1]) <= 2e-5


def test_lidar_only_12_levels_fused_chain_and_static_frame(cuda):
    model = _cfg3_geo12(cuda)
    lo, ld = C.lidar_rays(1, 4096)
    _fused_vs_chain_and_static(model, (lo.cuda(), ld.cuda()), None, False, C.loss_lidar, ("depth_volume", "normals_volume", "mask_volume"))


def test_colour_model_12_levels_camera_rays(cuda):
    model = C.build_model(cuda, max_num_levels=12, log2_hashmap_size=16, target_num_params=14 * 2 ** 17).train()
    assert model.implicit_surface.encoding.meta.n_pseudo_levels == 12 and model._color_fusable()
    co, cd = C.camera_rays(1, 4096)
    ha = torch.zeros(4096, model.radiance_net.blocks.layers[0].in_features - 22 - 24, device=cuda)
    _fused_vs_chain_and_static(model, (co.cuda(), cd.cuda()), ha, True, C.loss_cam,
                               ("depth_volume", "normals_volume", "mask_volume", "rgb_volume"))


def test_extract_mesh_at_12_levels_launches_the_fused_query(cuda):
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    model = C.build_model(cuda, max_num_levels=12, log2_hashmap_size=16, target_num_params=14 * 2 ** 17).eval()
    assert model.implicit_surface._fusable()
    q = lambda x: model.forward_sdf(model.space.normalize_coords(x))["sdf"]
    L.KERNEL_TIMER.enable()
    try:
        out = extract_mesh(q, filepath=None, N=24, chunk=20000, bmin=[-6., -12., -7.5], bmax=[6., 12., -3.5], show_progress=False, device=cuda)
        launched = L.KERNEL_TIMER.summary()
    finally:
        L.KERNEL_TIMER.disable()
    assert "lotd_gather" in launched, sorted(launched)
    v = out["verts"].cpu().numpy()
    assert v.shape[0] > 1000 and np.abs(v[:, 2] - C.ROAD_Z).max() < 0.02


def test_accelerate_12_level_reference_model(cuda):
    from neuralsim_b200.adapter import accelerate, describe
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from test_geometry_only_gpu import _RefLike
    src = _cfg3_geo12(cuda)
    ref = _RefLike(src).train()
    assert describe(ref)["radiance_cfg"] is False
    ours = accelerate(ref)
    assert ours.implicit_surface._fusable() and ours._geometry_fusable()
    assert ours.implicit_surface.encoding.flattened_params is ref.implicit_surface.encoding.flattened_params
    lo, ld = C.lidar_rays(4, 2048)
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()
    with torch.no_grad():
        want = r.render(src, lo.cuda(), ld.cuda())["rendered"]
        got = r.render(ref, lo.cuda(), ld.cuda())["rendered"]
    assert float(want["mask_volume"].sum()) > 100
    for k in ("depth_volume", "normals_volume", "mask_volume"):
        assert torch.equal(got[k], want[k]), k
