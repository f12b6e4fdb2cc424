"""The geometry-only colour query (csrc/color_tc.cu: k_color_fwd<false>, selected by nsb_fused_color_fwd with rgb == NULL) and the
models without a radiance net it serves (`radiance_cfg=False`, the LiDAR-only StreetSurf configuration).

1. The kernel against the full instantiation, bit for bit: sdf, nablas, x, the Z tile, the h half of the X tile, the occupancy collection;
   at 1, 127, 128, 129 points and at sizes where every persistent CTA loops, with max_level, and with a device count below the capacity.
2. sdf / nablas against the float64 reference (oracle/fused64.py) per element, and against the module path.
3. The second-order backward of a geometry-only model against float64 and against forward_sdf_nablas + autograd.
4. Rendering a geometry-only cfg3 model on LiDAR rays: fused == chain, graph step == host-sized step, no colour query without normals,
   17 levels through the module path.
5. adapter.accelerate on a stand-in without a radiance net."""
import ctypes

import numpy as np
import pytest
import torch

import bench_cfg3 as C
from oracle import fused64
from test_tc_kernels_gpu import (BWD_REL, NAB_FRAC_1E5, NAB_MAX_REL, SDF_FLIP_FRAC, SDF_MAX_ULP, TILE, _fp16_metrics, _inputs, _model, _rel,
                                 _sms)
from util import rel_l2

pytestmark = pytest.mark.gpu

GEO_CTAS_PER_SM = 2          # kColorGeoCtasPerSM (csrc/color_tc.cu)
SDF_KEYS = ("grid", "W1", "b1", "W2", "b2")


def _geo_size(iters):
    """the smallest n at which every CTA of the geometry-only grid runs at least `iters` tiles, with a partial last tile"""
    return (iters * _sms() * GEO_CTAS_PER_SM + 1) * TILE - 51


def _geo_twin(col):
    """a geometry-only LoTDNeuS with the colour model's table and decoder"""
    from neuralsim_b200.fields.neus import LoTDNeuS
    from oracle import lotd as olotd
    geo = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg()),
                                    decoder_cfg=dict(W=col.implicit_surface.decoder.layers[0].out_features)),
                   radiance_cfg=False, device="cuda")
    geo.implicit_surface.load_state_dict(col.implicit_surface.state_dict())
    geo.max_level = col.max_level
    assert geo.radiance_net is None and geo._geometry_fusable() and not geo._color_fusable()
    return geo


# ===================================================================================================================== 1. kernel
def _launch(model, inp, rad, *, max_level=None, count=None, collect_res=(16, 16, 16)):
    """one nsb_fused_color_fwd with all optional outputs; rad=False: rgb / view_dirs / h_appear / act_y* NULL and a net without radiance"""
    from neuralsim_b200 import _lib as L
    lib = L.lib()
    s = model.implicit_surface
    grid16, net, _held = model._fused_color_state() if rad else model._fused_geometry_state()
    n = inp["t"].shape[0]
    ridx, t, o, d, v = (inp[k].cuda().contiguous() for k in ("ridx", "t", "o", "d", "v"))
    ha = inp["ha"].cuda().contiguous() if (rad and model.use_h_appear) else None
    nan = float("nan")
    out = dict(sdf=torch.full((n,), nan, device="cuda"), nablas=torch.full((n, 3), nan, device="cuda"), x=torch.full((n, 3), nan, device="cuda"))
    rgb = torch.full((n, 3), nan, device="cuda") if rad else None
    tb = int(lib.nsb_color_tile_bytes(L.c_i64(n)))
    acts = torch.zeros(4 if rad else 2, max(int(lib.nsb_color_act_bytes(L.c_i64(n), s.encoding.meta.n_pseudo_levels)), 1), dtype=torch.uint8,
                       device="cuda")        # a saved X tile is 20 KB at more than 16 levels
    pcl = torch.zeros(int(np.prod(collect_res)), device="cuda")
    oc = L.OccCollectC(pcl.data_ptr(), (ctypes.c_int32 * 3)(*collect_res), 256.0)
    ap = [L.ptr(acts[k]) if k < acts.shape[0] else None for k in range(4)]
    cnt = torch.tensor([count if count is not None else n], dtype=torch.int64, device="cuda")
    if count is not None:
        lib.nsb_bind_device_counts(ctypes.c_void_p(cnt.data_ptr()), ctypes.c_void_p(0))
    try:
        rc = lib.nsb_fused_color_fwd(s.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(net), None, L.ptr(o, "f32"), L.ptr(d, "f32"),
                                     L.ptr(ridx, "i64"), L.ptr(t, "f32"), L.ptr(v, "f32") if rad else None, L.ptr(ha, "f32", allow_none=True),
                                     L.c_i64(n), L.c_i32(s._ml(max_level)), L.ptr(out["sdf"]), L.ptr(out["nablas"]), L.ptr(rgb, allow_none=True),
                                     L.ptr(out["x"]), *ap, ctypes.byref(oc), L.stream_ptr())
    finally:
        if count is not None:
            lib.nsb_bind_device_counts(ctypes.c_void_p(0), ctypes.c_void_p(0))
    L.check(rc, "fused_color_fwd")
    torch.cuda.synchronize()
    out["Z"] = acts[0]
    out["Xh"] = acts[1][:tb].view(-1, 16384)[:, :8192] if tb else acts[1][:0]  # per 16 KB tile (up to 16 levels): the four h chunks
    out["collect"] = pcl
    return out


_COL = {}


def _colour_model():
    if "m" not in _COL:
        _COL["m"] = _model(64, 64, 4, seed=5)
    return _COL["m"]


@pytest.mark.parametrize("n", [1, 127, 128, 129, "loop"])
@pytest.mark.parametrize("max_level", [None, 7])
def test_geometry_kernel_equals_full_kernel(n, max_level):
    col = _colour_model()
    if n == "loop":
        n = _geo_size(3)
        assert -(-n // TILE) >= 3 * _sms() * GEO_CTAS_PER_SM and n % TILE        # every CTA of the geometry grid runs >= 3 tiles
    inp = _inputs(n, 4, seed=n % 97)
    geo = _geo_twin(col)
    a = _launch(col, inp, True, max_level=max_level)
    b = _launch(geo, inp, False, max_level=max_level)
    for k in ("sdf", "nablas", "x", "Z", "Xh", "collect"):
        assert torch.equal(a[k], b[k]), k
    assert bool(torch.isfinite(b["sdf"]).all())


def test_geometry_kernel_device_count_below_capacity():
    col = _colour_model()
    n, live = _geo_size(2), _geo_size(1) - 77
    inp = _inputs(n, 4, seed=3)
    geo = _geo_twin(col)
    a = _launch(col, inp, True, count=live)
    b = _launch(geo, inp, False, count=live)
    for k in ("sdf", "nablas", "x"):
        assert torch.equal(a[k][:live], b[k][:live]), k
        assert bool(torch.isnan(b[k][live:]).all()), k                                          # nothing written past the count
    for k in ("Z", "Xh", "collect"):
        assert torch.equal(a[k], b[k]), k
    assert bool(torch.isfinite(b["sdf"][:live]).all())
    full = _launch(geo, inp, False)
    assert torch.equal(full["sdf"][:live], b["sdf"][:live]) and torch.equal(full["nablas"][:live], b["nablas"][:live])


# ===================================================================================================================== 2. forward values
@pytest.mark.parametrize("max_level", [None, 7])
def test_geometry_forward_per_element_against_float64(max_level):
    col = _colour_model()
    col.max_level = max_level
    try:
        geo = _geo_twin(col)
        n = _geo_size(3)
        assert -(-n // TILE) // min(-(-n // TILE), _sms() * GEO_CTAS_PER_SM) >= 3 and n % TILE
        inp = _inputs(n, 4, seed=17)
        ref = fused64.Fused64.from_model(col, max_level=max_level)
        fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy())
        with torch.no_grad():
            got = geo.forward_on_rays(*(inp[k].cuda() for k in ("ridx", "t", "o", "d")), with_rgb=False)
    finally:
        col.max_level = None
    assert "rgb" not in got and torch.equal(got["x"].cpu(), inp["x"])
    sdf = _fp16_metrics(got["sdf"].cpu().numpy(), fwd["sdf"], fwd["sdf_scale"])
    nab = np.abs(got["nablas"].cpu().numpy() - fwd["nablas"]) / (fwd["nablas_scale"] + 1e-30)
    print(f"METRIC geometry_fwd ml={max_level} sdf: flips={sdf[0]:.2e} max_ulp={sdf[1]:.2f} nablas: max_rel={nab.max():.2e} "
          f"frac>1e-5={(nab > 1e-5).mean():.2e}")
    assert sdf[0] <= SDF_FLIP_FRAC and sdf[1] <= SDF_MAX_ULP, sdf
    assert float(nab.max()) <= NAB_MAX_REL and float((nab > 1e-5).mean()) <= NAB_FRAC_1E5


def test_geometry_forward_against_module_path():
    """the sphere model and points of tests/test_color_gpu.py, without its radiance net"""
    from neuralsim_b200.fields import LoTDNeuSModel
    from test_color_gpu import _points
    from util import make_pair
    P, col = make_pair("cuda")
    geo = LoTDNeuSModel(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=P.lotd_cfg)), radiance_cfg=False, device="cuda")
    geo.implicit_surface.load_state_dict(col.implicit_surface.state_dict())
    o, d, ridx, t, _ha = _points()
    x = torch.addcmul(o[ridx], d[ridx], t.unsqueeze(-1))
    with torch.no_grad():
        got = geo.forward_on_rays(ridx, t, o, d, with_rgb=False)
        ref = geo.forward(x, with_rgb=False, with_normal=True)
    assert torch.equal(got["x"], x) and "rgb" not in got
    assert (got["sdf"] - ref["sdf"].float()).abs().max() <= 2e-3 and rel_l2(got["sdf"], ref["sdf"].float()) < 2e-4
    assert rel_l2(got["nablas"], ref["nablas"].float()) < 2e-3


# ===================================================================================================================== 3. backward
def test_geometry_backward_against_float64_and_module():
    col = _colour_model()
    geo = _geo_twin(col)
    n = _geo_size(3)
    inp = _inputs(n, 4, seed=29)
    c_sdf, c_nab = inp["cot"][0], inp["cot"][1]
    ps = geo.implicit_surface
    d = ps.decoder.layers
    params = [ps.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias]
    out = geo.forward_on_rays(*(inp[k].cuda() for k in ("ridx", "t", "o", "d")), with_rgb=False)
    loss = (out["sdf"] * c_sdf.cuda()).sum() + (out["nablas"] * c_nab.cuda()).sum()
    got = dict(zip(SDF_KEYS, torch.autograd.grad(loss, params)))
    ref = fused64.Fused64.from_model(col)
    fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy(), inp["ha"].numpy())
    want = ref.color_backward(fwd, c_sdf.numpy(), c_nab.numpy(), None)                  # zero rgb cotangent
    errs = {k: _rel(got[k].detach().double().cpu().numpy(), want[k]) for k in SDF_KEYS}
    print("METRIC geometry_bwd " + " ".join(f"{k}={e:.2e}" for k, e in errs.items()))
    for k in SDF_KEYS[:4]:
        assert np.abs(want[k]).max() > 0 and errs[k] < BWD_REL[k], (k, errs[k])
    # d_b2 = sum(g_sdf): these random cotangents cancel to ~1 out of ~1e5 terms, so its error is the fp32 summation error over the terms' magnitudes
    assert abs(float(got["b2"]) - float(want["b2"][0])) <= 1e-7 * float(c_sdf.double().abs().sum()), (float(got["b2"]), float(want["b2"][0]))
    # the module path: forward_sdf_nablas + autograd (second order through nablas)
    m = geo.forward_sdf_nablas(inp["x"].cuda(), has_grad=True, nablas_has_grad=True)
    loss_m = (m["sdf"].float() * c_sdf.cuda()).sum() + (m["nablas"].float() * c_nab.cuda()).sum()
    mod = dict(zip(SDF_KEYS, torch.autograd.grad(loss_m, params)))
    for k in SDF_KEYS:
        assert rel_l2(got[k], mod[k]) < 2e-2, (k, rel_l2(got[k], mod[k]))


# ===================================================================================================================== 4. rendering
def _cfg3_geo(cuda, levels):
    """bench_cfg3.build_model's street model (small table) with radiance_cfg=False"""
    from neuralsim_b200.fields import LoTDNeuSModel
    gen = torch.Generator(device=cuda).manual_seed(42)
    model = LoTDNeuSModel(
        surface_cfg=dict(aabb=C.AABB, sdf_scale=C.SDF_SCALE,
                         encoding_cfg=dict(lotd_use_cuboid=True,
                                           lotd_auto_compute_cfg=dict(type="ngp", target_num_params=(levels + 2) * 2 ** 17, min_res=16, n_feats=2,
                                                                      log2_hashmap_size=16, max_num_levels=levels),
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
    assert model.radiance_net is None and model._geometry_fusable() == (levels == 16)
    return model.train()


def _lidar(n, k=1):
    lo, ld = C.lidar_rays(k, n)
    return lo.cuda(), ld.cuda()


def _render_grads(model, r, lo, ld, fused=True):
    import neuralsim_b200.graphics.neus as GN
    import neuralsim_b200.fields.space as SP
    from neuralsim_b200.fields.networks import LoTDSDF
    model.zero_grad(set_to_none=True)
    saved = (GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable)
    if not fused:
        GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable = False, False, (lambda self: False)
    try:
        out = r.render(model, lo, ld)["rendered"]
        assert "rgb_volume" not in out
        C.loss_lidar(out).backward()
    finally:
        GN.FUSED_STAGES, SP.FUSED_RAY_TEST, LoTDSDF._fusable = saved
    s = model.implicit_surface
    return {k: v.detach().clone() for k, v in out.items()}, s.encoding.flattened_params.grad.clone(), s.decoder.layers[0].weight.grad.clone()


@pytest.mark.parametrize("levels", [16, 17])
def test_geometry_only_lidar_render_fused_equals_chain(cuda, levels):
    """16 levels: the geometry-only fused op; 17 levels (a table _fusable() rejects): the module path.  Both against the chain with every
    fused path off"""
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from neuralsim_b200 import _lib as L
    model = _cfg3_geo(cuda, levels)
    lo, ld = _lidar(2048)
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()
    L.KERNEL_TIMER.enable()
    try:
        a, ga, wa = _render_grads(model, r, lo, ld, fused=True)
        launched = L.KERNEL_TIMER.summary()
    finally:
        L.KERNEL_TIMER.disable()
    assert ("fused_color_fwd" in launched) == (levels == 16), sorted(launched)
    b, gb, wb = _render_grads(model, r, lo, ld, fused=False)
    assert float(a["mask_volume"].sum()) > 100
    for k in ("depth_volume", "normals_volume", "mask_volume"):
        assert rel_l2(a[k], b[k]) <= 1e-4, (k, rel_l2(a[k], b[k]))
    assert rel_l2(ga, gb) <= 2e-2 and rel_l2(wa, wb) <= 2e-2, (rel_l2(ga, gb), rel_l2(wa, wb))


def test_geometry_only_static_frame_equals_host_sized(cuda):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = _cfg3_geo(cuda, 16)
    lo, ld = _lidar(4096, k=2)
    ref, g_ref, w_ref = _render_grads(model, SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False)).train(), lo, ld)
    model.zero_grad(set_to_none=True)
    fr = StaticFrame(model, 4096, loss_fn=C.loss_lidar, near=C.NEAR, far=C.FAR, with_rgb=False, slack=2.0, zero_grads=True)
    fr.step(lo, ld, None)
    assert fr.counts()["overflow"] == 0 and fr.captures == 1 and fr.h_appear is None
    assert set(fr.rendered) == set(ref)
    for k, v in ref.items():
        assert torch.equal(fr.rendered[k], v), k
    s = model.implicit_surface
    assert rel_l2(s.encoding.flattened_params.grad, g_ref) <= 2e-5 and rel_l2(s.decoder.layers[0].weight.grad, w_ref) <= 2e-5
    vb = fr.volume_buffer()
    assert "rgb" not in vb and vb["nablas"].shape[0] == vb["t"].shape[0]


def test_geometry_only_static_frame_without_normals_skips_the_query(cuda):
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = _cfg3_geo(cuda, 16)
    lo, ld = _lidar(4096, k=3)
    with torch.no_grad():
        ref = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=False)).train().render(model, lo, ld)["rendered"]
        fr = StaticFrame(model, 4096, near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=False, slack=2.0)
        fr.step(lo, ld, None)
        assert fr.counts()["overflow"] == 0
        assert set(fr.rendered) == set(ref) == {"depth_volume", "mask_volume"}
        for k, v in ref.items():
            assert torch.equal(fr.rendered[k], v), k
        eager = StaticFrame(model, 4096, near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=False, slack=2.0, use_graph=False)
        L.KERNEL_TIMER.enable()
        try:
            eager.step(lo, ld, None)
            launched = L.KERNEL_TIMER.summary()
        finally:
            L.KERNEL_TIMER.disable()
    assert "fused_color_fwd" not in launched and "fused_sdf_fwd" in launched, sorted(launched)
    for k, v in ref.items():
        assert torch.equal(eager.rendered[k], v), k


# ===================================================================================================================== 5. adapter
class _RefLike(torch.nn.Module):
    """the attributes of a reference LoTDNeuS object built with `radiance_cfg: null` (radiance_net = None)"""

    def __init__(self, m):
        super().__init__()
        self.implicit_surface, self.ctrl_var, self.accel, self.space = m.implicit_surface, m.ctrl_var, m.accel, m.space
        self.radiance_net = None
        self.ray_query_cfg = dict(m.ray_query_cfg)
        self.upsample_s_divisor, self.max_level, self.it = 1.0, None, 0


def test_accelerate_geometry_only_reference_model(cuda):
    from neuralsim_b200.adapter import accelerate
    from neuralsim_b200.renderer import SingleVolumeRenderer
    src = _cfg3_geo(cuda, 16)
    ref = _RefLike(src).train()
    ours = accelerate(ref)
    assert ours.radiance_net is None and ours.implicit_surface.encoding.flattened_params is ref.implicit_surface.encoding.flattened_params
    for a, b in zip(ours.implicit_surface.decoder.layers, ref.implicit_surface.decoder.layers):
        assert a.weight is b.weight and a.bias is b.bias
    assert ours.ctrl_var.ln_inv_s is ref.ctrl_var.ln_inv_s and ours.accel.occ.occ_grid is ref.accel.occ.occ_grid
    assert ours.implicit_surface.radius3d_original is ref.implicit_surface.radius3d_original
    assert {k for k, _ in ours.named_parameters()} == {k for k, _ in src.named_parameters()}
    lo, ld = _lidar(2048, k=4)
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()
    with torch.no_grad():
        want = r.render(src, lo, ld)["rendered"]
        got = r.render(ref, lo, ld)["rendered"]          # through the patched ray_test / ray_query of the reference-like object
    assert float(want["mask_volume"].sum()) > 100
    for k in ("depth_volume", "normals_volume", "mask_volume"):
        assert torch.equal(got[k], want[k]), k
