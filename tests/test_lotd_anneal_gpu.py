"""The LoTD level schedule on the GPU: a level bound read from device memory (nsb_bind_device_max_level) by every fused kernel, the graph
step following the schedule without re-capture, and the adapter following the reference's annealed level.

1. Entry points.  The fused SDF query (points, rays, packs), its backward (plain, indexed, rays), the colour forward (with and without the
   radiance net, saved Z / X / Y1 / Y2 tiles included) and the colour backward (plain, codes, rays) give the same bits with the level in
   device memory as with the host int, on the 12- and 16-level cfg3 tables and a cubic table, at max_level -1, 0, 1, 2, 7, L-2, L-1 and
   None, at a size where every persistent CTA runs three or more tiles and the last tile is partial.  Gradients that are sums of fp32
   atomics are compared to the order of those sums; the table gradient above the level is exactly 0.  The outputs at a level are the
   float64 reference's (oracle/fused64.py) at that level.
2. The persistent up-sampling kernel with a device level equals the stage kernels at the host level.
3. The graph step on an annealed cfg3 model through a schedule that crosses every level change: one capture, every replay's rendered
   buffers and loss bit-equal to the host-sized step at the same iteration, gradients to the order of the fp32 atomics, with the code and
   ray gradients and with the LiDAR loss inside the step, and no host read in step().
4. The adapter renders at the level the reference's encoding carries."""
import ctypes
import gc

import numpy as np
import pytest
import torch

import bench_cfg3 as C
import test_lidar_loss_gpu as ll
import test_partial_levels_gpu as pl
from fused64_levels import Fused64Levels
from test_tc_kernels_gpu import TILE, _inputs, _sms
from util import rel_l2

pytestmark = pytest.mark.gpu

ORDER_REL = ll.ORDER_REL
TABLES = ("cfg3-12", "cfg3-16", "cubic-16")
_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        if kind == "cubic-16":
            m = pl._model(16, seed=16)
        else:
            L = int(kind.split("-")[1])
            m = C.build_model(torch.device("cuda"), max_num_levels=L, log2_hashmap_size=16, target_num_params=(L + 2) * 2 ** 17)
            with torch.no_grad():
                m.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=torch.Generator("cuda").manual_seed(L))
        assert m.implicit_surface._fusable() and m._color_fusable()
        _MODELS[kind] = m
    return _MODELS[kind]


def _levels(L):
    return sorted({-1, 0, 1, 2, 7, L - 2, L - 1}) + [None]


def _dev(level):
    return torch.tensor(level, dtype=torch.int32, device="cuda")


def _color_fwd_raw(model, inp, rad, level):
    """one nsb_fused_color_fwd with every output and saved tile"""
    from neuralsim_b200 import _lib as L
    s = model.implicit_surface
    grid16, net, _held = model._fused_color_state() if rad else model._fused_geometry_state()
    n = inp["t"].shape[0]
    o, d, ridx, t, v, ha = (inp[k] for k in ("o", "d", "ridx", "t", "v", "ha"))
    out = {k: torch.full(sh, float("nan"), device="cuda") for k, sh in (("sdf", (n,)), ("nablas", (n, 3)), ("x", (n, 3)))}
    if rad:
        out["rgb"] = torch.full((n, 3), float("nan"), device="cuda")
    acts = torch.zeros(4 if rad else 2, int(L.lib().nsb_color_tile_bytes(L.c_i64(n))), dtype=torch.uint8, device="cuda")
    ap = [L.ptr(acts[k]) if k < acts.shape[0] else None for k in range(4)]
    L.call(L.lib().nsb_fused_color_fwd, "fused_color_fwd", s.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(net), None, L.ptr(o, "f32"),
           L.ptr(d, "f32"), L.ptr(ridx, "i64"), L.ptr(t, "f32"), L.ptr(v, "f32") if rad else None, L.ptr(ha, "f32") if rad else None, L.c_i64(n),
           L.c_level(level), L.ptr(out["sdf"]), L.ptr(out["nablas"]), L.ptr(out.get("rgb"), allow_none=True), L.ptr(out["x"]), *ap, None, L.stream_ptr(),
           level=level)
    for k, name in enumerate(("Z", "X", "Y1", "Y2")[:acts.shape[0]]):
        out[name] = acts[k]
    return out


def _color_grads(model, inp, level, form):
    """the colour query through its autograd op at `level`; form: 'plain' (nsb_fused_color_bwd), 'codes' (_bwd_appear), 'rays' (_bwd_grads)"""
    from neuralsim_b200.fields.fused_color import ColorQuery, _FusedColor
    s = model.implicit_surface
    d, r = s.decoder.layers, model.radiance_net.blocks.layers
    params = (s.encoding.flattened_params, d[0].weight, d[0].bias, d[1].weight, d[1].bias, r[0].weight, r[0].bias, r[1].weight, r[1].bias,
              r[2].weight, r[2].bias)
    grid16, net, held = model._fused_color_state()
    ha = inp["ha"].clone().requires_grad_(form == "codes")
    ro, rd = (inp["o"].clone().requires_grad_(True), inp["d"].clone().requires_grad_(True)) if form == "rays" else (None, None)
    q = ColorQuery(s.encoding.meta, grid16, net, held, inp["o"], inp["d"], level, None, None)
    out = _FusedColor.apply(q, inp["ridx"], inp["t"], inp["v"], ha, ro, rd, True, *params)
    c_sdf, c_nab, c_rgb = inp["cot"]
    loss = (out[0] * c_sdf).sum() + (out[1] * c_nab).sum() + (out[2] * c_rgb).sum()
    extra = {"codes": [ha], "rays": [ro, rd]}.get(form, [])
    g = torch.autograd.grad(loss, list(params) + extra)
    names = ["grid", "W1", "b1", "W2", "b2", "R1", "rb1", "R2", "rb2", "R3", "rb3"] + {"codes": ["d_ha"], "rays": ["d_ro", "d_rd"]}.get(form, [])
    return dict(zip(names, g))


def _sdf_all(model, inp, level):
    """the fused SDF query in its three modes and its backward in its three forms at `level` (host int or device scalar)"""
    from neuralsim_b200.fields.networks import sdf_bwd, sdf_fwd
    s = model.implicit_surface
    grid16, dec = s._fused_state()
    meta, n = s.encoding.meta, inp["t"].shape[0]
    out = {}
    for mode in ("x", "rays", "packs"):
        sdf = torch.full((n,), float("nan"), device="cuda")
        if mode == "x":
            sdf_fwd(meta, grid16, dec, sdf, level, x=inp["x"])
        elif mode == "rays":
            sdf_fwd(meta, grid16, dec, sdf, level, rays_o=inp["o"], rays_d=inp["d"], t=inp["t"], ridx=inp["ridx"])
        else:
            sdf_fwd(meta, grid16, dec, sdf, level, rays_o=inp["po"], rays_d=inp["pd"], t=inp["pt"], packs=(inp["pinfo"], None))
        out[f"sdf_{mode}"] = sdf
    d_sdf = inp["cot"][0]
    shapes = [p.shape for p in (s.encoding.flattened_params, *[w for l in s.decoder.layers for w in (l.weight, l.bias)])]
    for form in ("plain", "indexed", "rays"):
        grads = tuple(torch.zeros(sh, device="cuda") for sh in shapes)
        if form == "plain":
            sdf_bwd(meta, grid16, dec, d_sdf, n, level, grads, x=inp["x"])
        else:
            keep = inp["keep"]
            rays = (inp["o"], inp["d"], inp["ridx"], inp["t"])
            rg = (torch.zeros_like(inp["o"]), torch.zeros_like(inp["d"])) if form == "rays" else None
            sdf_bwd(meta, grid16, dec, d_sdf, keep.numel(), level, grads, rays=rays, keep=keep, ray_grads=rg)
            if rg is not None:
                grads = grads + rg
        out[f"bwd_{form}"] = grads
    return out


def _entry_inputs(n, seed):
    inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else tuple(c.cuda() for c in v)) for k, v in _inputs(n, 4, seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    inp["keep"] = torch.sort(torch.randperm(n, generator=g)[: n - n // 5]).values.cuda()          # most rows, ascending (ray order)
    P = n // 8 + 1                                                                                  # packs of up to 8 samples, the last partial
    cnt = torch.full((P,), 8, dtype=torch.int64)
    cnt[-1] = n - 8 * (P - 1)
    inp["pinfo"] = torch.stack([torch.arange(P) * 8, cnt], 1).cuda()
    inp["po"], inp["pd"] = inp["o"][::8].contiguous(), inp["d"][::8].contiguous()
    inp["pt"] = (torch.rand(n, generator=g) * 0.5).cuda()
    return inp


def _nonzero_above(g, model, level):
    """the table gradient at the levels above `level` is exactly zero"""
    meta = model.implicit_surface.encoding.meta
    La = meta.n_levels if level is None else min(max(level + 1, 0), meta.n_levels)
    return bool(g[meta.level_offsets[La]:].any())


@pytest.mark.parametrize("table", TABLES)
def test_device_level_equals_host_level_at_every_entry_point(table):
    model = _model(table)
    L = model.implicit_surface.encoding.meta.n_levels
    n = (3 * _sms() * 4 + 1) * TILE - 51
    assert -(-n // TILE) >= 3 * _sms() * 4 and n % TILE
    inp = _entry_inputs(n, seed=L)
    prev = None
    for ml in _levels(L):
        host_level = L if ml is None else ml                     # the kernels' argument (no `or` resolution here: 0 is level 0)
        dev_level = _dev(host_level)
        a, b = _sdf_all(model, inp, host_level), _sdf_all(model, inp, dev_level)
        for k in ("sdf_x", "sdf_rays", "sdf_packs"):
            assert torch.equal(a[k], b[k]), (table, ml, k)
            assert bool(torch.isfinite(a[k]).all()), (table, ml, k)
        assert torch.equal(a["sdf_x"], a["sdf_rays"]), (table, ml)
        for form in ("plain", "indexed", "rays"):
            for k, (ga, gb) in enumerate(zip(a[f"bwd_{form}"], b[f"bwd_{form}"])):
                assert rel_l2(gb, ga) <= ORDER_REL, (table, ml, form, k, rel_l2(gb, ga))
            assert not _nonzero_above(b[f"bwd_{form}"][0], model, ml), (table, ml, form)
        for rad in (True, False):
            fa, fb = _color_fwd_raw(model, inp, rad, host_level), _color_fwd_raw(model, inp, rad, dev_level)
            for k in fa:
                assert torch.equal(fa[k], fb[k]), (table, ml, rad, k)
        for form in ("plain", "codes", "rays"):
            ga, gb = _color_grads(model, inp, host_level, form), _color_grads(model, inp, dev_level, form)
            for k in ga:
                assert rel_l2(gb[k], ga[k]) <= ORDER_REL, (table, ml, form, k, rel_l2(gb[k], ga[k]))
            assert not _nonzero_above(gb["grid"], model, ml), (table, ml, form)
        if prev is not None and ml is not None and ml >= 0:
            assert not torch.equal(prev, a["sdf_x"]), (table, ml)            # each level changes the field
        prev = a["sdf_x"]


@pytest.mark.parametrize("max_level", [1, 7, 14])
def test_device_level_against_float64(max_level):
    """the cubic 16-level table with the level in device memory against the float64 reference at that level (the partial-level checks of
    tests/test_partial_levels_gpu.py; a model-level max_level of 0 means "the encoding's level", as in the reference, so it is not a case)"""
    model = _model("cubic-16")
    ref = Fused64Levels.from_model(model, max_level=max_level)
    inp = _inputs(129, 4, seed=max_level + 5)
    got = _run_all_dev(model, inp, max_level)
    pl._check(got, ref, inp, full_metrics=False)


def _run_all_dev(model, inp, ml):
    """test_partial_levels_gpu._run_all with the level handed to the kernels in device memory"""
    from neuralsim_b200.fields import networks
    s = model.implicit_surface
    orig = networks.LoTDSDF._ml
    networks.LoTDSDF._ml = lambda self, m: _dev(orig(self, m))                 # every fused launch of the model reads a device level
    try:
        return pl._run_all(model, inp, ml)
    finally:
        networks.LoTDSDF._ml = orig
        assert s._ml(None) == s.encoding.meta.n_levels


def test_upsample_persistent_with_device_level_equals_stage_kernels():
    from test_ray_upsample_edges_gpu import LAYOUTS, Rays, _chain, _kernel
    model = _model("cfg3-16").train()
    surf = model.implicit_surface
    layout = next(iter(LAYOUTS))
    R = Rays(16)
    for k in range(3 * _sms() * 5):
        R.add("hit", int(R.rng.integers(8, 200)))
    rt = R.tensors()
    rows = np.arange(len(R.n))
    for ml in (-1, 0, 2, 9, 15, None):
        with torch.no_grad():
            ref, _, _, _ = _chain(surf, rt, rows, layout, ml=surf._ml(ml), est=False, thre=0.0)
            got, ovf = _kernel(surf, rt, layout, ml=_dev(surf._ml(ml)), est=False, thre=0.0, entry="wrapper")
        assert int(ovf.sum()) == 0 and bool(torch.isfinite(ref).all())
        assert torch.equal(got, ref), ml


# ===================================================================================================================== graph step
STOP_IT = 13          # 16 levels from start_level 2: one level per iteration, so the replays at 0..13 cross every level change
# The surface moves with the level, and with it the number of kept samples: the kept arena is sized for every boundary sample (129 coarse
# + 48 fine per ray), so that no level overflows it (a trainer relies on StaticFrame.check() to re-size instead).
KEPT_PER_RAY = 129 + 8 + 8 + 32


def _annealed_cfg3():
    from neuralsim_b200.fields.encoding import MultiresAnnealer
    model = C.build_model(torch.device("cuda"), max_num_levels=16, log2_hashmap_size=16, target_num_params=18 * 2 ** 17).train()
    enc = model.implicit_surface.encoding
    enc.annealer = MultiresAnnealer(enc.lotd.level_n_feats, type="hardmask", start_it=0, start_level=2, stop_it=STOP_IT)
    return model


def _set_iter(model, it):
    model.implicit_surface.training_before_per_step(it)
    model.ctrl_var.set_iter(it)


def test_graph_step_follows_the_level_schedule_camera():
    """camera rays with the code and ray gradients: every replay of one capture is the host-sized step at the same iteration"""
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = _annealed_cfg3()
    co, cd = (t[:4096].cuda() for t in C.camera_rays(3, C.N_CAM))
    codes = torch.randn(4096, 4, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 0.3
    cfg = dict(near=C.NEAR, far=C.FAR)

    def host():
        for p in model.parameters():                      # in place: the captured step accumulates into these tensors
            if p.grad is not None:
                p.grad.zero_()
        o, d, h = co.clone().requires_grad_(True), cd.clone().requires_grad_(True), codes.clone().requires_grad_(True)
        r = SingleVolumeRenderer(cfg).train().render(model, o, d, rays_h_appear=h)["rendered"]
        loss = C.loss_cam(r)
        loss.backward()
        return ({k: v.detach().clone() for k, v in r.items()}, loss.detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None},
                o.grad, d.grad, h.grad)

    _set_iter(model, STOP_IT)                         # the arenas are sized at all levels
    model.zero_grad(set_to_none=True)
    gc.collect()
    fr = StaticFrame(model, 4096, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, zero_grads=True, h_appear_grad=True, ray_grad=True, slack=2.0,
                     kept_cap=4096 * KEPT_PER_RAY)
    fr.step(co, cd, codes)
    seen = set()
    for it in list(range(STOP_IT + 1)) + [STOP_IT + 5]:
        _set_iter(model, it)
        seen.add(model.implicit_surface.encoding.max_level)
        h = host()
        h2 = host()
        fr.step(co, cd, codes)
        assert fr.counts()["overflow"] == 0, it
        for k, v in h[0].items():
            assert torch.equal(fr.rendered[k], v), (it, k)
        assert torch.equal(fr.loss, h[1]), it
        for n, p in model.named_parameters():
            if n in h[2]:
                e, spread = rel_l2(p.grad, h[2][n]), rel_l2(h2[2][n], h[2][n])
                assert e <= max(ORDER_REL, 2 * spread), (it, n, e, spread)
        assert torch.equal(fr.d_rays_o, h[3]) and torch.equal(fr.d_rays_d, h[4]), it
        assert torch.equal(fr.d_h_appear, h[5]), it
    assert seen == set(range(2, 16)) and fr.captures == 1
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _set_iter(model, 4)
        fr.step(co, cd, codes)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert fr.captures == 1


def test_graph_step_follows_the_level_schedule_lidar_loss():
    """LiDAR rays with the fused LiDAR loss inside the step (loss_on_ret=True)"""
    model = _annealed_cfg3()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    _set_iter(model, STOP_IT)                         # the arenas are sized at all levels
    fr, lidar, terms, lo, ld, ranges = ll._frame_case(model, cfg)
    fr.kept_cap = 4096 * KEPT_PER_RAY
    lidar.set_step(ranges, STOP_IT)
    fr.step(lo, ld)
    for it in range(STOP_IT + 1):
        _set_iter(model, it)
        ll._compare_to_host(model, fr, lidar, terms, lo, ld, ranges, it, cfg, f"it {it}")
    assert fr.captures == 1


# ===================================================================================================================== adapter
def test_adapter_follows_the_reference_encodings_level():
    from neuralsim_b200.adapter import accelerate
    from neuralsim_b200.fields.neus import volume_integration
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from oracle import scene as oscene
    from test_adapter_gpu import _RefLike
    from util import make_pair
    _, src = make_pair(torch.device("cuda"))
    ref = _RefLike(src).train()
    accelerate(ref)
    ro, rd = oscene.pinhole_rays(30, 40, oscene.orbit_camera(1, 8))
    ro, rd, ha = ro.cuda(), rd.cuda(), torch.zeros(1200, 4, device="cuda")
    r = SingleVolumeRenderer(dict(near=0.01)).train()

    def via_ref():
        with torch.no_grad():
            raw = ref.ray_query(ray_tested=ref.ray_test(ro, rd, near=0.01, rays_h_appear=ha), config=dict(with_rgb=True, with_normal=True), return_buffer=True)
            rendered = dict(mask_volume=torch.zeros(1200, device="cuda"), depth_volume=torch.zeros(1200, device="cuda"),
                            rgb_volume=torch.zeros(1200, 3, device="cuda"), normals_volume=torch.zeros(1200, 3, device="cuda"))
            return volume_integration(raw["volume_buffer"], rendered, training=True)

    enc = src.implicit_surface.encoding                   # the reference's encoding object: its annealer sets max_level, the model's stays None
    with torch.no_grad():
        full = r.render(src, ro, rd, rays_h_appear=ha)["rendered"]
        enc.max_level = 3
        want = r.render(src, ro, rd, rays_h_appear=ha)["rendered"]
    got = via_ref()
    enc.max_level = None
    assert ref.max_level is None
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=0, atol=1e-6), k
    assert float((want["rgb_volume"] - full["rgb_volume"]).abs().max()) > 1e-3
    back = via_ref()
    for k in full:
        assert torch.allclose(back[k], full[k], rtol=0, atol=1e-6), k
