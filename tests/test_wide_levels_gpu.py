"""LoTD tables of L = 17..24 levels (2 features each) on the 48-column form of the wgmma kernels (k_fused_sdf_tc in its three modes,
k_sdf_bwd_tc, k_upsample_persistent, k_color_fwd<true|false>, k_color_rad_bwd, k_color_sdf_bwd), enabled per model with
max_fused_levels=24.

1. Kernels against the float64 reference in the 48-column layout (tests/fused64_wide.py) at L in {17, 18, 19, 23, 24}, with and without
   max_level (bounds below 16 included), at 1, 127, 128 and 129 points and at a size where every persistent CTA loops over three or more
   tiles, with the table and W1 images in NaN-tailed allocations, and with a device count below the capacity.
2. A 17-level table at max_level = 15 against the 16-level model with the same first 16 levels and W1 columns: the extra feature columns
   add exact zeros, so every output is bit-equal; the gradients agree to the order of the fp32 atomics (which already varies from run to
   run of one model), and the 17th level's table rows and W1 / R1 columns get exact zeros.
3. The persistent up-sampling kernel at 17 levels is bit-equal to the stage kernels.
4. bench_cfg3's street model at 17 levels with the option: fused == chain and graph step == host-sized step for LiDAR and camera rays,
   one capture with the error-map sampler, pose refinement, perturbation and code gradients across a hard-mask level schedule whose bound
   crosses 16, extract_mesh and adapter.accelerate.
5. The gradients to learnable rays, view directions and codes through every ray- and code-gradient instantiation of the 48-column backward
   kernels against the module path, and the wide radiance column map at 0 and 8 codes against float64."""
import numpy as np
import pytest
import torch

import bench_cfg3 as C
from fused64_wide import Fused64Wide
from oracle import lotd as olotd
from test_geometry_only_gpu import _launch
from test_partial_levels_gpu import SDF_KEYS, _check, _fused_vs_chain_and_static, _install_nan_tails, _params, _run_all
from test_tc_kernels_gpu import TILE, _inputs, _sms
from util import rel_l2

pytestmark = pytest.mark.gpu

LEVELS = [17, 18, 19, 23, 24]
CASES = [(L, ml) for L in LEVELS for ml in (None, L - 3, 9)]


def _model(levels, seed, n_appear=4, radiance=True, log2_hashmap_size=16):
    from neuralsim_b200.fields.neus import LoTDNeuS
    gen = torch.Generator("cuda").manual_seed(seed)
    model = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg(log2_hashmap_size=log2_hashmap_size,
                                                                                                       num_levels=levels)),
                                      decoder_cfg=dict(W=64), max_fused_levels=24),
                     radiance_cfg=dict(W=64, n_appear_embedding=n_appear) if radiance else False, device="cuda", generator=gen)
    with torch.no_grad():
        model.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=gen)
    s = model.implicit_surface
    assert s.encoding.meta.n_pseudo_levels == levels and tuple(s.decoder.layers[0].weight.shape) == (64, 2 * levels)
    assert s._fusable() and (model._color_fusable() if radiance else model._geometry_fusable())
    return model


# ===================================================================================================================== 1. kernels
@pytest.mark.parametrize("levels,max_level", CASES, ids=[f"L{L}-ml{ml}" for L, ml in CASES])
def test_kernels_against_float64_small_sizes(levels, max_level):
    model = _model(levels, seed=levels)
    _install_nan_tails(model)
    ref = Fused64Wide.from_model(model, max_level=max_level)
    assert ref.nh == 2 * levels
    for n in (1, 127, 128, 129):
        inp = _inputs(n, 4, seed=n + levels)
        _check(_run_all(model, inp, max_level), ref, inp, full_metrics=False)


@pytest.mark.parametrize("levels,max_level", [(17, None), (17, 12), (19, None), (24, None), (24, 17)])
def test_kernels_against_float64_multi_tile(levels, max_level):
    """every CTA of every persistent grid loops over three or more tiles (4 CTAs / SM is the largest grid: k_fused_sdf_tc)"""
    model = _model(levels, seed=100 + levels)
    _install_nan_tails(model)
    n = (3 * _sms() * 4 + 1) * TILE - 51
    # the inputs of the 12-level case of tests/test_partial_levels_gpu.py: their sdf cotangents do not nearly cancel, so the b2 sum (fp32
    # atomics in an order that varies run to run) stays well inside its relative bound
    inp = _inputs(n, 4, seed=12)
    ref = Fused64Wide.from_model(model, max_level=max_level)
    _check(_run_all(model, inp, max_level), ref, inp, full_metrics=True)


def test_colour_forward_device_count_below_capacity():
    model = _model(19, seed=3)
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


# ===================================================================================================================== 2. a masked level
def test_masked_17th_level_equals_the_16_level_model():
    """17 levels at max_level = 15 vs the 16-level model with the same first 16 levels, W1 columns and radiance weights (the 17th level's
    h columns removed from R1): every output bit-equal, the gradients to the order of the fp32 atomics, and exact zeros for the 17th level's
    table rows and W1 / R1 columns"""
    m17 = _model(17, seed=21, log2_hashmap_size=14)
    m16 = _model(16, seed=22, log2_hashmap_size=14)
    s17, s16 = m17.implicit_surface, m16.implicit_surface
    n16 = s16.encoding.flattened_params.numel()
    with torch.no_grad():
        s16.encoding.flattened_params.copy_(s17.encoding.flattened_params[:n16])      # the first 16 levels lie first in the table
        for a, b in zip(s16.decoder.layers, s17.decoder.layers):
            a.bias.copy_(b.bias)
        s16.decoder.layers[0].weight.copy_(s17.decoder.layers[0].weight[:, :32])
        s16.decoder.layers[1].weight.copy_(s17.decoder.layers[1].weight)
        r16, r17 = m16.radiance_net.blocks.layers, m17.radiance_net.blocks.layers
        for a, b in zip(r16, r17):
            a.bias.copy_(b.bias)
        r16[0].weight.copy_(torch.cat([r17[0].weight[:, :22 + 32], r17[0].weight[:, 22 + 34:]], 1))
        r16[1].weight.copy_(r17[1].weight)
        r16[2].weight.copy_(r17[2].weight)
    inp = _inputs(3 * TILE + 17, 4, seed=23)
    a = _run_all(m17, inp, 15)
    b = _run_all(m16, inp, 15)
    for k in ("sdf_pts", "sdf_rays", "geo_sdf", "geo_nablas", "sdf", "nablas", "rgb"):
        assert np.array_equal(a[k], b[k]), k
    close = lambda x, y: rel_l2(torch.as_tensor(x), torch.as_tensor(y)) <= 1e-5
    for part in ("sdf_bwd", "color_bwd"):
        ga, gb = a[part], b[part]
        assert close(ga["grid"][:n16], gb["grid"]) and not ga["grid"][n16:].any(), part
        W1 = ga["W1"].reshape(64, 34)
        assert close(W1[:, :32], gb["W1"].reshape(64, 32)) and not W1[:, 32:].any(), part
        for k in ("b1", "W2", "b2") + (("R2", "rb2", "R3", "rb3", "rb1") if part == "color_bwd" else ()):
            assert close(ga[k], gb[k]), (part, k)
        if part == "color_bwd":
            R1 = ga["R1"].reshape(64, -1)
            assert close(np.concatenate([R1[:, :54], R1[:, 56:]], 1), gb["R1"].reshape(64, -1)) and not R1[:, 54:56].any()


# ===================================================================================================================== 3. up-sampling
def test_upsample_persistent_at_17_levels_equals_stage_kernels():
    from test_ray_upsample_edges_gpu import LAYOUTS, Rays, _chain, _kernel
    model = _model(17, seed=9).train()
    surf = model.implicit_surface
    _install_nan_tails(model)
    layout = next(iter(LAYOUTS))
    R = Rays(12)
    for k in range(3 * _sms() * 2):
        R.add("hit", int(R.rng.integers(8, 200)))
    rt = R.tensors()
    rows = np.arange(len(R.n))
    for ml in (None, 14, 16):
        with torch.no_grad():
            ref, _, _, _ = _chain(surf, rt, rows, layout, ml=surf._ml(ml), est=False, thre=0.0)
            got, ovf = _kernel(surf, rt, layout, ml=surf._ml(ml), est=False, thre=0.0, entry="wrapper")
        assert int(ovf.sum()) == 0 and bool(torch.isfinite(ref).all())
        assert torch.equal(got, ref), ml


# ===================================================================================================================== 4. models
def _small17(cuda, radiance=True):
    """bench_cfg3's street model at 17 levels (2 dense + 15 hashed, as the shipped camera models) with a small hashmap, fused per model"""
    model = C.build_model(cuda, max_num_levels=17, log2_hashmap_size=16, target_num_params=19 * 2 ** 17).train()
    s = model.implicit_surface
    assert s.encoding.meta.n_pseudo_levels == 17 and not s._fusable()
    s.max_fused_levels = 24
    assert s._fusable() and model._color_fusable()
    return model


def test_lidar_rays_17_levels_fused_chain_and_static_frame(cuda):
    model = _small17(cuda)
    lo, ld = C.lidar_rays(1, 4096)
    _fused_vs_chain_and_static(model, (lo.cuda(), ld.cuda()), None, False, C.loss_lidar, ("depth_volume", "normals_volume", "mask_volume"))


def test_camera_rays_with_codes_17_levels_fused_chain_and_static_frame(cuda):
    model = _small17(cuda)
    co, cd = C.camera_rays(1, 4096)
    na = model.radiance_net.blocks.layers[0].in_features - 22 - 34
    ha = torch.randn(4096, na, device=cuda, generator=torch.Generator(cuda).manual_seed(3)) * 0.1
    _fused_vs_chain_and_static(model, (co.cuda(), cd.cuda()), ha, True, C.loss_cam,
                               ("depth_volume", "normals_volume", "mask_volume", "rgb_volume"))


def test_one_capture_with_sampler_pose_perturb_across_16_levels(cuda):
    """the training step of a shipped camera model at 17 levels: StaticFrame(sampler=, pose=, perturb=True, h_appear_grad=True) under the
    hard-mask annealer, its bound moving from 12 to all 17 levels (the 48-column kernels at every bound, with the ray-gradient and
    code-gradient forms of both backward kernels).  Every replay of one capture against the host-sized sequence of tests/test_importance_gpu.py
    (sample, pose rays, perturbed render, loss, error-map update): batch, images, loss, pose and code gradients and error maps bit-equal,
    parameter gradients to the order of the fp32 atomics"""
    import gc
    import test_importance_gpu as ig
    from neuralsim_b200.fields.encoding import MultiresAnnealer
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.graphics.pose import pose_rays
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from test_lotd_anneal_gpu import KEPT_PER_RAY, _set_iter
    from util import product_grads
    I = ig._I()
    n = 4096
    model = _small17(cuda)
    enc = model.implicit_surface.encoding
    stop = 6
    enc.annealer = MultiresAnnealer(enc.lotd.level_n_feats, type="hardmask", start_it=0, start_level=12, stop_it=stop)
    cs, specs = ig._cameras()
    poses = ig._street_poses(15)
    host_maps = [I.ErrorMap(s.error_map.n_images, (32, 64), device="cuda", n_steps_init=2) for s in cs.samplers]
    for hm, s in zip(host_maps, cs.samplers):
        hm.error_map.copy_(s.error_map.error_map)
        hm.construct_cdf()
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    _set_iter(model, stop)                                # the arenas are sized at all levels
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, n, loss_fn=ig._loss, near=C.NEAR, far=C.FAR, zero_grads=True, h_appear_grad=True, pose=poses, perturb=True, sampler=cs,
                     slack=2.0, kept_cap=n * KEPT_PER_RAY)

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
        loss, err = ig._loss(out, gt)
        loss.backward()
        return dict(fidx=fidx, xy=xy, gt=gt, rendered={k: v.detach().clone() for k, v in out.items()}, loss=loss.detach(), err=err.detach(),
                    grads=product_grads(model), dq=poses.dq.grad.clone(), dt=poses.dt.grad.clone(), d_codes=codes.grad.clone())

    was = torch.are_deterministic_algorithms_enabled()
    seen = set()
    its = [stop] + list(range(stop + 2))                  # the capture at all levels, then the schedule from 12 levels on
    for step, it in enumerate(its):
        cam = step % 2
        _set_iter(model, it)
        seen.add(enc.max_level)
        s0 = gen.get_offset()
        fr.step(cam=cam)
        assert fr.counts()["overflow"] == 0 and fr.check(), (step, it)
        got = dict(fidx=fr.rays_fidx.clone(), xy=fr.rays_pix.clone(), gt={k: v.clone() for k, v in fr.ground_truth.items()},
                   rendered={k: v.clone() for k, v in fr.rendered.items()}, loss=fr.loss.clone(), grads=product_grads(model), dq=poses.dq.grad.clone(),
                   dt=poses.dt.grad.clone(), d_codes=fr.d_h_appear.clone())
        maps = [s.error_map.error_map.clone() for s in cs.samplers]
        h = host(cam, s0)
        h2 = host(cam, s0)
        torch.use_deterministic_algorithms(True)
        try:
            I.recipe_update_error_map(host_maps[cam].error_map, h["fidx"], h["xy"], h["err"])
        finally:
            torch.use_deterministic_algorithms(was)
        host_maps[cam].count_step()
        for k in ("fidx", "xy", "loss", "dq", "dt", "d_codes"):
            ig._same(got[k], h[k], f"step {step} level {it} {k}")
        for k in h["gt"]:
            ig._same(got["gt"][k], h["gt"][k], f"step {step} {k}")
        for k, v in h["rendered"].items():
            ig._same(got["rendered"][k], v, f"step {step} level {it} {k}")
        for k, v in h["grads"].items():
            if v is not None:
                e, spread = rel_l2(got["grads"][k], v), rel_l2(h2["grads"][k], v)
                assert e <= max(ig.ORDER_REL, 2 * spread), (step, k, e, spread)
        for c, hm in enumerate(host_maps):
            ig._same(maps[c], hm.error_map, f"step {step} camera {c} error map")
        assert float(h["dq"].abs().max()) > 0 and float(h["d_codes"].abs().max()) > 0
        gen.set_offset(s0 + fr.sampler_reservation + fr.rng_reservation)
    assert {12, 15, 16} <= seen and len(seen) >= 5 and fr.captures == 1, seen


# ===================================================================================================================== 5. input gradients
@pytest.mark.parametrize("leaves", [("o", "d", "v", "ha"), ("ha",), ("o", "d", "v")], ids=["rays+codes", "codes", "rays"])
@pytest.mark.parametrize("levels,max_level", [(17, None), (24, 14)], ids=["L17", "L24-ml14"])
def test_color_op_input_grads_against_module_path(levels, max_level, leaves):
    """the gradients to learnable rays, view directions and appearance codes through the 48-column colour kernels (k_color_rad_bwd<A, R, 48>
    for all three (codes, rays) forms, k_color_sdf_bwd<true, 48> and the per-ray sums) against the module path, as
    tests/test_ray_grad_gpu.py does at 16 levels; the same bits on a second run"""
    import test_ray_grad_gpu as rg
    from neuralsim_b200.fields.fused_color import fused_color
    model = _model(levels, seed=300 + levels)
    model.max_level = max_level
    c = rg._case(3000, seed=levels + 5)
    for k in ("o", "d", "v", "ha"):
        if k not in leaves:
            c[k] = c[k].detach()
    run = lambda: rg._grads(rg._loss(fused_color(model, c["ridx"], c["t"], c["o"], c["d"], c["v"], c["ha"]), c["cot"]), [c[k] for k in leaves])
    got = run()
    ref = model.forward(rg._module_x(c), v=c["v"][c["ridx"]], h_appear=c["ha"][c["ridx"]], nablas_has_grad=True)
    want = rg._grads(rg._loss(ref, c["cot"]), [c[k] for k in leaves])
    assert rg._check(f"color L={levels} ml={max_level} {'+'.join(leaves)}", got, want, c, list(leaves)) >= 1
    for a, b in zip(got, run()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("levels", [17, 24])
def test_geometry_and_sdf_op_ray_grads_against_module_path(levels):
    """k_color_sdf_bwd<true, 48> without the radiance net, and k_sdf_bwd_tc<true, true, 48> (the boundary query) with a third of the
    cotangents zero, against the module path"""
    import test_ray_grad_gpu as rg
    from neuralsim_b200.fields.fused_color import fused_color
    model = _model(levels, seed=400 + levels)
    c = rg._case(3000, seed=levels + 11)
    out = fused_color(model, c["ridx"], c["t"], c["o"], c["d"], with_rgb=False)
    got = rg._grads(rg._loss(out, c["cot"], rgb=False), [c["o"], c["d"]])
    want = rg._grads(rg._loss(model.forward_sdf_nablas(rg._module_x(c), nablas_has_grad=True), c["cot"], rgb=False), [c["o"], c["d"]])
    rg._check(f"geometry L={levels}", got, want, c, ["o", "d"])
    s = model.implicit_surface
    cot = c["cot"][0] * (torch.arange(3000, device="cuda") % 3 != 0)
    got = rg._grads((s.fused_sdf_rays_autograd(c["ridx"], c["t"], c["o"], c["d"]) * cot).sum(), [c["o"], c["d"]])
    want = rg._grads((s.forward(rg._module_x(c))["sdf"].float() * cot).sum(), [c["o"], c["d"]])
    rg._check(f"sdf L={levels}", got, want, c, ["o", "d"])


@pytest.mark.parametrize("levels", [17, 24])
@pytest.mark.parametrize("n_appear", [0, 8])
def test_radiance_column_map_on_the_kernels(levels, n_appear):
    """the wide radiance column map of the kernels (ref_col at 48 h columns: R1 staging, sR1h / sR1a and the dR1 flush) at the smallest and
    largest code widths, through the colour forward and both backward kernels against float64"""
    model = _model(levels, seed=500 + levels + n_appear, n_appear=n_appear)
    _install_nan_tails(model)
    ref = Fused64Wide.from_model(model)
    assert ref.n_appear == n_appear
    inp = _inputs(TILE + 1, n_appear, seed=levels + n_appear)
    _check(_run_all(model, inp, None), ref, inp, full_metrics=False)


def test_extract_mesh_at_17_levels_launches_the_fused_query(cuda):
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    model = _small17(cuda).eval()
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


def test_accelerate_17_level_reference_model(cuda):
    from neuralsim_b200.adapter import accelerate
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from test_geometry_only_gpu import _RefLike
    src = _small17(cuda)
    ref = _RefLike(src).train()
    ours = accelerate(ref, max_fused_levels=24)
    assert ours.implicit_surface.max_fused_levels == 24 and ours.implicit_surface._fusable()
    assert accelerate(_RefLike(src).train()).implicit_surface._fusable() is False
    lo, ld = C.lidar_rays(4, 2048)
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()
    with torch.no_grad():
        want = r.render(src, lo.cuda(), ld.cuda())["rendered"]
        got = r.render(ref, lo.cuda(), ld.cuda())["rendered"]
    assert float(want["mask_volume"].sum()) > 100
    for k in ("depth_volume", "normals_volume", "mask_volume"):
        assert torch.equal(got[k], want[k]), k
