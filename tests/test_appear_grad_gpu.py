"""The appearance-code gradient of the fused colour query (k_color_rad_bwd<true> + k_appear_ray_sum, csrc/color_tc.cu;
nsb_fused_color_bwd_appear) against the float64 reference, through the host-sized render and through the one-launch graph step.

Bounds.  AP_REL is the rel-L2 bound tests/test_tc_kernels_gpu.py puts on R1's gradient against oracle/fused64.py (BWD_REL["R1"]):
the code gradient dZ1 . R1[:, h_appear] is the other contraction of the same fp16 dZ1, so a ReLU mask that flips with a one-ulp change
of its input moves it the same way.  FRAME_REL is tests/test_step_grad_frame_gpu.py's REL, the bound of the 800x600 step against its
float64 replay.  MODULE_REL is the fused-vs-module-path bound of tests/test_cfg3_gpu.py.  ORDER_REL bounds two runs that differ only
in the order of the fp32 atomics (tests/test_step_grad_frame_gpu.py's LIN_REL)."""
import ctypes
import gc
import json

import numpy as np
import pytest
import torch

import test_tc_kernels_gpu as tk
from appear64 import code_grad, ray_sum, step_code_grads
from oracle import fused64, scene as oscene, step64
from util import make_pair, product_grads, rel_l2

pytestmark = pytest.mark.gpu

AP_REL = tk.BWD_REL["R1"]           # 6e-3
FRAME_REL = 6e-4
MODULE_REL = 2e-2
ORDER_REL = 2e-5
SENT = -12345.0


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# ===================================================================================================================== 1. the entry point
def _ray_layout(n, seed, long_ray):
    """ridx [n] sorted: runs of 1..40 samples (they straddle 128-row tiles), every 7th ray without a sample, and with long_ray one ray
    of 300 samples that starts at about row 100 (it spans three tiles) -> (ridx, number of rays; the last two have no sample)"""
    rng = np.random.default_rng(seed)
    lens, total = [], 0
    while total < n:
        if long_ray and total >= 100 and 300 not in lens:
            k = 300
        else:
            k = 0 if len(lens) % 7 == 3 else int(rng.integers(1, 41))
        lens.append(k)
        total += k
    return np.repeat(np.arange(len(lens)), lens)[:n].astype(np.int64), len(lens) + 2


def _inputs(n, n_appear, seed, long_ray=False, ridx=None, R=None):
    if ridx is None:
        ridx, R = _ray_layout(n, seed, long_ray)
    g = torch.Generator().manual_seed(seed)
    o = torch.rand(R, 3, generator=g) * 1.6 - 0.8
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    t = torch.rand(n, generator=g) * 0.3
    v = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    ha = torch.randn(R, n_appear, generator=g) * 0.5
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    ridx = torch.as_tensor(ridx)
    x = (d[ridx].double() * t.double()[:, None] + o[ridx].double()).float()       # the kernels' fma(d, t, o)
    return dict(ridx=ridx, R=R, o=o, d=d, t=t, v=v, ha=ha, cot=cot, x=x)


def _direct(model, inp, *, appear=True, cap_extra=0, ray_map=None):
    """nsb_fused_color_fwd + nsb_fused_color_bwd(_appear) on inp's samples.  cap_extra > 0: the capacity is that many samples larger
    than the device-resident count; the extra samples name ray R (a ray no counted sample names) and carry NaN cotangents"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.fields.fused_color import h_tile_cols
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _call
    P = L.ptr
    n, R = inp["t"].shape[0], inp["R"]
    m = n + cap_extra
    grid16, net, _alive = model._fused_color_state()
    meta, ml = model.implicit_surface.encoding.meta, model.implicit_surface._ml(None)
    cu = lambda a: a.contiguous().cuda()
    o, d, v, ha = (cu(torch.cat([inp[k], inp[k][:1]])) for k in ("o", "d", "v", "ha"))      # row R: the extra samples' ray
    ridx = cu(torch.cat([inp["ridx"], torch.full((cap_extra,), R, dtype=torch.int64)]))
    t = cu(torch.cat([inp["t"], inp["t"][:cap_extra]]))
    cot = [cu(torch.cat([c, torch.full((cap_extra, *c.shape[1:]), float("nan"))])) for c in inp["cot"]]
    out = {k: torch.empty(m, *s, device="cuda") for k, s in (("sdf", ()), ("nab", (3,)), ("rgb", (3,)), ("x", (3,)))}
    acts = torch.empty(4, int(L.lib().nsb_color_act_bytes(L.c_i64(m), meta.n_pseudo_levels)), dtype=torch.uint8, device="cuda")
    ps = tk._params(model)
    grads = {k: torch.zeros(p.shape, dtype=torch.float32, device="cuda") for k, p in ps.items()}
    dh = torch.full((m, h_tile_cols(meta.n_pseudo_levels)), SENT, device="cuda")
    rows = torch.full((m, 8), SENT, device="cuda")
    d_ha = torch.zeros(R + 1, ha.shape[1], device="cuda")
    d_ha[R] = SENT
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[CNT_SLOTS["kept"]] = n
    fwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o, "f32"), P(d, "f32"), P(ridx, "i64"), P(t, "f32"), P(v, "f32"), P(ha, "f32"),
           L.c_i64(m), L.c_i32(ml), P(out["sdf"]), P(out["nab"]), P(out["rgb"]), P(out["x"]), *[P(acts[k]) for k in range(4)], None, L.stream_ptr())
    bwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o, "f32"), P(d, "f32"), P(ridx, "i64"), P(t, "f32"), L.c_i64(m), L.c_i32(ml),
           *[P(acts[k]) for k in range(4)], P(out["rgb"]), P(cot[0]), P(cot[1]), P(cot[2]), P(dh), *[P(grads[k]) for k in tk.BWD_REL])
    if appear:
        bwd = bwd + (P(rows), P(ray_map, "i64", allow_none=True), P(d_ha), L.stream_ptr())
        fns = ((L.lib().nsb_fused_color_fwd, "fused_color_fwd", fwd), (L.lib().nsb_fused_color_bwd_appear, "fused_color_bwd_appear", bwd))
    else:
        fns = ((L.lib().nsb_fused_color_fwd, "fused_color_fwd", fwd), (L.lib().nsb_fused_color_bwd, "fused_color_bwd", bwd + (L.stream_ptr(),)))
    for fn, what, args in fns:
        if cap_extra:
            _call(fn, what, cnt, CNT_SLOTS["kept"], None, *args)
        else:
            L.check(fn(*args), what)
    torch.cuda.synchronize()
    return dict(dh=dh, rows=rows, d_ha=d_ha, grads=grads)


_MODELS = {}


def _model(n_appear):
    if n_appear not in _MODELS:
        _MODELS[n_appear] = tk._model(64, 64, n_appear, seed=100 + n_appear)
    return _MODELS[n_appear]


def _check_against_f64(model, inp, got, what, ref=None, fwd=None):
    """ref: the float64 reference (default: Fused64 of the model), fwd: its colour forward on inp (computed when None)"""
    n, R, na = inp["t"].shape[0], inp["R"], inp["ha"].shape[1]
    ref = fused64.Fused64.from_model(model) if ref is None else ref
    ridx = inp["ridx"].numpy()
    if fwd is None:
        fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy()[ridx], inp["ha"].numpy()[ridx])
    want = code_grad(ref, fwd, inp["cot"][2].numpy())
    want_ray = ray_sum(want, ridx, R)
    rows = got["rows"].cpu().numpy()
    d_ha = got["d_ha"].cpu().numpy()[:R]
    e_rows, e_ray = _rel(rows[:n, :na], want), _rel(d_ha, want_ray)
    print(f"METRIC appear {what} n={n} rays={R} n_appear={na} rows_rel={e_rows:.2e} rays_rel={e_ray:.2e} (bound {AP_REL:.0e})")
    assert np.abs(want).max() > 0
    assert e_rows <= AP_REL and e_ray <= AP_REL, (e_rows, e_ray)
    assert (rows[:n, na:] == 0).all()                                   # columns beyond n_appear: zero
    empty = np.setdiff1d(np.arange(R), ridx)
    assert (d_ha[empty] == 0).all() and not np.signbit(d_ha[empty]).any()                    # rays without a sample: +0
    return empty.shape[0]


SIZES = [(1, 4), (127, 4), (128, 4), (129, 4), (67661, 4), (129, 1), (3000, 1), (129, 8), (3000, 8)]


@pytest.mark.parametrize("n,n_appear", SIZES, ids=[f"n{n}-a{a}" for n, a in SIZES])
def test_entry_point_against_float64(n, n_appear):
    model = _model(n_appear)
    inp = _inputs(n, n_appear, seed=n + n_appear, long_ray=n > 500)
    if n > 500:                                                          # one ray with more than 256 samples, across tiles
        assert int(torch.bincount(inp["ridx"]).max()) > 256
        ends = np.nonzero(np.diff(inp["ridx"].numpy()))[0] + 1           # runs that straddle a 128-row tile boundary
        starts = np.concatenate([[0], ends])
        stops = np.concatenate([ends, [n]])
        assert ((starts // 128) != ((stops - 1) // 128)).sum() >= 5
    got = _direct(model, inp)
    assert _check_against_f64(model, inp, got, f"n{n}") >= 2
    plain = _direct(model, inp, appear=False)
    assert torch.equal(got["dh"], plain["dh"])                          # the same radiance backward, bit for bit


def test_entry_point_device_count_and_ray_map():
    """count below the capacity: rows past the count and the ray only those rows name stay untouched; a ray map permutes the output
    rows and nothing else (the same bits)"""
    model = _model(4)
    inp = _inputs(5000, 4, seed=77, long_ray=True)
    a = _direct(model, inp)
    b = _direct(model, inp, cap_extra=700)
    n, R = 5000, inp["R"]
    assert torch.equal(b["d_ha"][:R], a["d_ha"][:R]) and bool((b["d_ha"][R] == SENT).all())
    assert torch.equal(b["rows"][:n], a["rows"][:n]) and bool((b["rows"][n:] == SENT).all())
    assert torch.equal(b["dh"][:n], a["dh"][:n]) and bool((b["dh"][n:] == SENT).all())
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(3)).cuda()
    c = _direct(model, inp, ray_map=torch.cat([perm, torch.tensor([R], device="cuda")]))
    assert torch.equal(c["d_ha"][perm], a["d_ha"][:R])


# ===================================================================================================================== 2. host-sized render
def _frame_rays(cuda):
    ro, rd = oscene.pinhole_rays(48, 64, oscene.orbit_camera(1, 8, radius=3.0, elev_deg=25.0))
    miss_o = torch.tensor([[3.0, 3.0, 3.0]]).repeat(40, 1)                # 40 rays that miss the box
    miss_d = torch.nn.functional.normalize(torch.tensor([[0.2, 0.3, 1.0]]), dim=-1).repeat(40, 1)
    ro, rd = torch.cat([ro, miss_o]), torch.cat([rd, miss_d])
    codes = torch.randn(ro.shape[0], 4, generator=torch.Generator().manual_seed(9)) * 0.3
    w = torch.tensor([-1.0, -0.5, 0.5, 1.0])[torch.randint(0, 4, (ro.shape[0], 3), generator=torch.Generator().manual_seed(10))]
    return ro.to(cuda), rd.to(cuda), codes.to(cuda), w.to(cuda)


def _loss(rendered, w):
    """rgb weighted per ray (a cotangent of order 1: the code gradient is not lost to fp16 rounding) + the other images' means"""
    return (rendered["rgb_volume"] * w).sum() + sum(rendered[k].mean() for k in ("depth_volume", "mask_volume", "normals_volume"))


def _host(model, ro, rd, codes, w):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model.zero_grad(set_to_none=True)
    out = SingleVolumeRenderer(dict(near=0.01)).train().render(model, ro, rd, rays_h_appear=codes)["rendered"]
    _loss(out, w).backward()
    return {k: v.detach().clone() for k, v in out.items()}, product_grads(model)


def _fused_only(model, monkeypatch):
    def module_path(*a, **k):
        raise AssertionError("the colour query fell back to the module path")
    monkeypatch.setattr(model, "forward", module_path)


_HOST = {}


def _host_case(cuda, monkeypatch):
    if "r" not in _HOST:
        _, model = make_pair(cuda)
        model.train()
        ro, rd, codes0, w = _frame_rays(cuda)
        kept = {}
        with monkeypatch.context() as mp:
            _fused_only(model, mp)
            fwd_on_rays = model.forward_on_rays

            def record(*a, **k):                                          # the kept samples the colour query runs on
                kept.update(ridx=a[0].detach().cpu(), t=a[1].detach().cpu(), o=a[2].detach().cpu(), d=a[3].detach().cpu(), v=a[4].detach().cpu(),
                            ha=a[5].detach().cpu())
                return fwd_on_rays(*a, **k)
            mp.setattr(model, "forward_on_rays", record)
            codes = codes0.clone().requires_grad_(True)
            r_grad, g_grad = _host(model, ro, rd, codes, w)
            r_det, g_det = _host(model, ro, rd, codes0, w)
            _, g_det2 = _host(model, ro, rd, codes0, w)
        _HOST["r"] = dict(model=model, ro=ro, rd=rd, codes0=codes0, w=w, r_grad=r_grad, g_grad=g_grad, r_det=r_det, g_det=g_det, g_det2=g_det2,
                          d_codes=codes.grad.detach().clone(), kept=kept)
    return _HOST["r"]


def test_host_sized_render_with_learnable_codes(cuda, monkeypatch):
    h = _host_case(cuda, monkeypatch)
    for k in h["r_det"]:
        assert torch.equal(h["r_grad"][k], h["r_det"][k]), k                       # the same forward, bit for bit
    rep = {}
    for k, v in h["g_det"].items():
        if v is None:
            assert h["g_grad"][k] is None, k
            continue
        rep[k] = (rel_l2(h["g_grad"][k], v), rel_l2(h["g_det2"][k], v))             # learnable vs detached codes; two detached runs
        assert rep[k][0] <= max(ORDER_REL, 2 * rep[k][1]), (k, rep[k])
    d = h["d_codes"]
    miss = d[-40:]
    assert bool((miss == 0).all()) and float(d[:-40].abs().max()) > 0
    # the module path (FUSED_STAGES off) on the same codes
    from neuralsim_b200.graphics import neus as GN
    model, codes = h["model"], h["codes0"].clone().requires_grad_(True)
    monkeypatch.setattr(GN, "FUSED_STAGES", False)
    _host(model, h["ro"], h["rd"], codes, h["w"])
    e = rel_l2(d, codes.grad)
    print("METRIC appear host-sized", json.dumps(dict(param_rel=rep, codes_vs_module=e)))
    assert e <= MODULE_REL, e


def test_entry_point_on_frame_kept_samples(cuda, monkeypatch):
    h = _host_case(cuda, monkeypatch)
    k = h["kept"]
    n, R = k["t"].shape[0], k["o"].shape[0]
    g = torch.Generator().manual_seed(12)
    cot = (torch.randn(n, generator=g), torch.randn(n, 3, generator=g) * 0.05, torch.randn(n, 3, generator=g))
    x = (k["d"][k["ridx"]].double() * k["t"].double()[:, None] + k["o"][k["ridx"]].double()).float()
    inp = dict(ridx=k["ridx"], R=R, o=k["o"], d=k["d"], t=k["t"], v=k["v"], ha=k["ha"], cot=cot, x=x)
    assert n > 10000 and int(torch.bincount(k["ridx"]).max()) > 1
    got = _direct(h["model"], inp)
    _check_against_f64(h["model"], inp, got, "frame-kept")
    assert torch.equal(got["dh"], _direct(h["model"], inp, appear=False)["dh"])


# ===================================================================================================================== 3. graph step
def test_graph_step_code_gradient(cuda, monkeypatch):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    h = _host_case(cuda, monkeypatch)
    model, ro, rd, codes0, w = h["model"], h["ro"], h["rd"], h["codes0"], h["w"]
    model.zero_grad(set_to_none=True)
    gc.collect()
    frame = StaticFrame(model, ro.shape[0], loss_fn=lambda r: _loss(r, w), near=0.01, h_appear_grad=True, zero_grads=True)
    frame.step(ro, rd, codes0)
    assert frame.counts()["overflow"] == 0
    for k in ("rgb_volume", "depth_volume", "normals_volume", "mask_volume"):
        assert torch.equal(frame.rendered[k], h["r_grad"][k]), k
    first = frame.d_h_appear.clone()
    assert torch.equal(first, h["d_codes"])                               # the host-sized codes' .grad, bit for bit
    frame.step(ro, rd, codes0)
    assert torch.equal(frame.d_h_appear, first)                           # a replay overwrites: nothing accumulates
    assert frame.captures == 1
    # a parameter update: the next replay follows it
    R1 = model.radiance_net.blocks.layers[0].weight
    saved = R1.detach().clone()
    with torch.no_grad():
        R1.mul_(1.25)
    frame.step(ro, rd, codes0)
    upd = frame.d_h_appear.clone()
    assert not torch.equal(upd, first)
    codes = codes0.clone().requires_grad_(True)
    _host(model, ro, rd, codes, w)
    assert torch.equal(upd, codes.grad)
    with torch.no_grad():
        R1.copy_(saved)


def test_graph_step_option_off_keeps_no_buffer(cuda):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    _, model = make_pair(cuda)
    assert StaticFrame(model, 16, near=0.01).d_h_appear is None
    with pytest.raises(RuntimeError, match="appearance codes"):
        StaticFrame(model, 16, near=0.01, with_rgb=False, h_appear_grad=True)


# ===================================================================================================================== 4. the 800x600 frame
_FRAME = {}


def _frame_case(cuda, monkeypatch):
    """bench.py's model and 800x600 frame (view 0) with seeded codes and an rgb loss weighted per ray; the graph step's d_h_appear and
    the float64 replay (oracle/step64.py, tests/appear64.py) of a 4096-ray subset of its hit rays on the host-sized step's own decisions"""
    if "r" in _FRAME:
        return _FRAME["r"]
    import bench
    import test_step_grad_frame_gpu as sf
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = bench.build_model(cuda).train()
    o, d = sf._rays(0, False, cuda)
    n = o.shape[0]
    g = torch.Generator().manual_seed(21)
    codes = (torch.randn(n, 4, generator=g) * 0.3).to(cuda)
    w = torch.tensor([-1.0, -0.5, 0.5, 1.0])[torch.randint(0, 4, (n, 3), generator=g)].to(cuda)
    loss = lambda r: (r["rgb_volume"] * w).sum()
    cap = sf._Capture(monkeypatch, model)
    hc = codes.clone().requires_grad_(True)
    out = SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=hc)["rendered"]
    loss(out).backward()
    r_host = {k: v.detach().clone() for k, v in out.items()}
    c = cap.host()
    del out
    monkeypatch.undo()
    model.zero_grad(set_to_none=True)
    gc.collect()
    frame = StaticFrame(model, n, loss_fn=loss, near=0.01, h_appear_grad=True)
    frame.step(o, d, codes)
    assert frame.counts()["overflow"] == 0
    for k in r_host:
        assert torch.equal(frame.rendered[k], r_host[k]), k
    assert torch.equal(frame.d_h_appear, hc.grad)
    hit = c["compact"]["rays_inds_hit"]
    solid = np.nonzero(r_host["mask_volume"].cpu().numpy()[hit] > 0.5)[0]    # as in that file: grazing rays' alphas are fp32 noise
    packs = np.sort(np.random.default_rng(5).choice(solid, sf.N_SUBSET, replace=False))
    dec = sf._decisions(c, packs)
    ref64 = fused64.Fused64.from_model(model)
    R = packs.shape[0]
    g_rgb = w[torch.from_numpy(hit[packs]).to(cuda)].double().cpu().numpy()
    cot = dict(g_mask=np.zeros(R), g_depth=np.zeros(R), g_rgb=g_rgb, g_nablas=np.zeros((R, 3)))
    ref = step_code_grads(ref64, dec, c["compact"]["inv_s"], **cot, ln_inv_s_factor=model.ctrl_var.ln_inv_s_factor)
    got = frame.d_h_appear[torch.from_numpy(hit[packs]).to(cuda)].double().cpu().numpy()
    miss = np.setdiff1d(np.arange(n), hit)
    _FRAME["r"] = dict(got=got, ref=ref, dec=dec, ref64=ref64, cot=cot, inv_s=c["compact"]["inv_s"], factor=model.ctrl_var.ln_inv_s_factor,
                       miss_zero=bool((frame.d_h_appear[torch.from_numpy(miss).to(cuda)] == 0).all()), n_miss=int(miss.shape[0]))
    return _FRAME["r"]


def test_frame_code_gradient_matches_float64_replay(cuda, monkeypatch):
    r = _frame_case(cuda, monkeypatch)
    e = _rel(r["got"], r["ref"])
    print(f"METRIC appear frame800x600 subset={r['got'].shape[0]} rel={e:.2e} (bound {FRAME_REL:.0e}) misses={r['n_miss']}")
    assert np.abs(r["ref"]).max() > 0
    assert e <= FRAME_REL, e
    assert r["miss_zero"]


def test_frame_wrong_references_fail(cuda, monkeypatch):
    """the bound can fail: two float64 references with a deliberate defect -- (1) the ReLU mask of Y1 left out of dZ1 on every 10th ray,
    (2) every 100th ray given its neighbour's code gradient -- fail the comparison the kernels pass"""
    r = _frame_case(cuda, monkeypatch)
    ref = r["ref"]
    rays = np.arange(0, ref.shape[0], 10)
    ref1 = ref.copy()
    ref1[rays] = step_code_grads(r["ref64"], step64.select(r["dec"], rays), r["inv_s"], **{k: v[rays] for k, v in r["cot"].items()},
                                 ln_inv_s_factor=r["factor"], alter=lambda fwd: dict(fwd, Y1=np.abs(fwd["Y1"]) + 1.0))
    ref2 = ref.copy()
    every = np.arange(0, ref.shape[0] - 1, 100)
    ref2[every] = ref[every + 1]
    errs = [_rel(r["got"], ref1), _rel(r["got"], ref2)]
    print(f"METRIC appear frame wrong references: rel={errs[0]:.2e}, {errs[1]:.2e} (bound {FRAME_REL:.0e})")
    assert all(e > FRAME_REL for e in errs), errs
