"""The gradient to learnable rays (pose refinement) through the fused NeuS query: k_sdf_bwd_tc<true, true> (nsb_fused_sdf_bwd_rays),
k_color_rad_bwd<., true> + k_color_sdf_bwd<true> (nsb_fused_color_bwd_grads) and their per-ray sums (k_ray_row_sum).  The entry points
are pinned to the float64 reference tests/rays64.py; the autograd ops and the host-sized render to the module path, which differentiates
the same way (the depths are constants and the encoding's input gradient is first order).

Bounds.  RAY_REL is the rel-L2 bound of the entry points against float64: AP_REL (tests/test_appear_grad_gpu.py), the bound of the other
contraction of the same fp16 dZ1.  MODULE_REL is the fused-vs-module-path bound of tests/test_cfg3_gpu.py: the module path runs the
autocast fp16 graph, the fused kernels round at the same points but sum in other orders."""
import ctypes
import json

import numpy as np
import pytest
import torch

import test_appear_grad_gpu as ag
import test_tc_kernels_gpu as tk
from fused64_levels import Fused64Levels
from oracle import lotd as olotd
from rays64 import color_rows, ray_grads, sdf_rows
from util import make_pair, product_grads, rel_l2

pytestmark = pytest.mark.gpu

RAY_REL = ag.AP_REL
MODULE_REL = 2e-2
SENT = -12345.0


# ===================================================================================================================== 1. the entry points
_LEVEL_MODELS = {}


def _level_model(n_levels, zero_table=False):
    if (n_levels, zero_table) not in _LEVEL_MODELS:
        from neuralsim_b200.fields.neus import LoTDNeuS
        gen = torch.Generator("cuda").manual_seed(400 + n_levels)
        m = LoTDNeuS(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=olotd.gen_ngp_cfg(num_levels=n_levels)), decoder_cfg=dict(W=64)),
                     radiance_cfg=dict(W=64, n_appear_embedding=4), device="cuda", generator=gen)
        with torch.no_grad():
            m.implicit_surface.encoding.flattened_params.uniform_(-0.5, 0.5, generator=gen)
            if zero_table:
                m.implicit_surface.encoding.flattened_params.zero_()
        assert m._color_fusable()
        _LEVEL_MODELS[n_levels, zero_table] = m
    return _LEVEL_MODELS[n_levels, zero_table]


def _entry(model, inp, ml, *, cap_extra=0, rgb=True, sdf=False):
    """nsb_fused_color_fwd + nsb_fused_color_bwd_grads (sdf=False) or nsb_fused_sdf_bwd_rays (sdf=True) on inp's samples, with the
    device-resident count n and a capacity cap_extra larger (the extra samples name ray R and carry NaN cotangents)"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.fields.fused_color import h_tile_cols
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _call
    P = L.ptr
    n, R = inp["t"].shape[0], inp["R"]
    m = n + cap_extra
    s = model.implicit_surface
    meta = s.encoding.meta
    cu = lambda a: a.contiguous().cuda()
    o, d, v, ha = (cu(torch.cat([inp[k], inp[k][:1]])) for k in ("o", "d", "v", "ha"))
    ridx = cu(torch.cat([inp["ridx"], torch.full((cap_extra,), R, dtype=torch.int64)]))
    t = cu(torch.cat([inp["t"], inp["t"][:cap_extra]]))
    cot = [cu(torch.cat([c, torch.full((cap_extra, *c.shape[1:]), float("nan"))])) for c in inp["cot"]]
    outs = {k: torch.zeros(R + 1, 3, device="cuda") for k in ("o", "d", "v")}
    for k in outs:
        outs[k][R] = SENT
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[CNT_SLOTS["kept"]] = n
    fns = []
    if sdf:
        grid16, dec = s._fused_state()
        ps = [s.encoding.flattened_params, *[p for l in s.decoder.layers for p in (l.weight, l.bias)]]
        grads = [torch.zeros(p.shape, dtype=torch.float32, device="cuda") for p in ps]
        rows = torch.full((m, 8), SENT, device="cuda")
        fns.append((L.lib().nsb_fused_sdf_bwd_rays, "fused_sdf_bwd_rays",
                    (meta.c_ref, P(grid16, "f16"), ctypes.byref(dec), P(o), P(d), P(ridx), P(t), P(cot[0]), None, L.c_i64(m), L.c_i32(ml),
                     *[P(g) for g in grads], P(rows), None, P(outs["o"]), P(outs["d"]), L.stream_ptr())))
    else:
        grid16, net, _alive = model._fused_color_state() if rgb else model._fused_geometry_state()
        out = {k: torch.empty(m, *sh, device="cuda") for k, sh in (("sdf", ()), ("nab", (3,)), ("rgb", (3,)), ("x", (3,)))}
        acts = torch.empty(4, int(L.lib().nsb_color_act_bytes(L.c_i64(m), meta.n_pseudo_levels)), dtype=torch.uint8, device="cuda")
        ps = tk._params(model)
        grads = {k: torch.zeros(p.shape, dtype=torch.float32, device="cuda") for k, p in ps.items()}
        dh = torch.empty(m, h_tile_cols(meta.n_pseudo_levels), device="cuda")
        rows = torch.full((m, 36), SENT, device="cuda")
        fwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o), P(d), P(ridx), P(t), P(v) if rgb else None, P(ha) if rgb else None,
               L.c_i64(m), L.c_i32(ml), P(out["sdf"]), P(out["nab"]), P(out["rgb"]) if rgb else None, P(out["x"]), P(acts[0]), P(acts[1]),
               P(acts[2]) if rgb else None, P(acts[3]) if rgb else None, None, L.stream_ptr())
        gp = [P(grads[k]) for k in tk.BWD_REL]
        gp = gp if rgb else gp[:5] + [None] * 6
        bwd = (meta.c_ref, P(grid16, "f16"), ctypes.byref(net), None, P(o), P(d), P(ridx), P(t), L.c_i64(m), L.c_i32(ml), P(acts[0]), P(acts[1]),
               *((P(acts[2]), P(acts[3]), P(out["rgb"])) if rgb else (None, None, None)), P(cot[0]), P(cot[1]), P(cot[2]) if rgb else None,
               P(dh) if rgb else None, *gp, P(v), None, None, None, P(rows), P(outs["o"]), P(outs["d"]), P(outs["v"]) if rgb else None,
               L.stream_ptr())
        fns += [(L.lib().nsb_fused_color_fwd, "fused_color_fwd", fwd), (L.lib().nsb_fused_color_bwd_grads, "fused_color_bwd_grads", bwd)]
    for fn, what, args in fns:
        if cap_extra:
            _call(fn, what, cnt, CNT_SLOTS["kept"], None, *args)
        else:
            L.check(fn(*args), what)
    torch.cuda.synchronize()
    return outs, rows


def _want(model, inp, ml, *, rgb=True, sdf=False, drop_rad_x=False):
    ref = Fused64Levels.from_model(model, max_level=ml)            # the 16-level layout with zero columns for L < 16
    ridx = inp["ridx"].numpy()
    c = [x.numpy() for x in inp["cot"]]
    if sdf:
        g_x, g_v = sdf_rows(ref, inp["x"].numpy(), c[0]), None
    else:
        fwd = ref.color_forward(inp["x"].numpy(), inp["v"].numpy()[ridx], inp["ha"].numpy()[ridx])
        g_x, g_v = color_rows(ref, fwd, inp["v"].numpy()[ridx], c[0], c[1], c[2] if rgb else None)
        if drop_rad_x:                       # a deliberately wrong reference: without the radiance input's direct dL/dx columns
            from rays64 import _radiance_dZ1
            g_x = g_x - _radiance_dZ1(ref, fwd, c[2]) @ ref.R1[:, 0:3]
    return ray_grads(g_x, inp["t"].numpy(), ridx, inp["R"], g_v if rgb and not sdf else None)


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _check_entry(what, outs, want, inp):
    R = inp["R"]
    rep = {}
    for k, w in zip(("o", "d", "v"), want):
        if w is None:
            continue
        got = outs[k][:R].cpu().numpy()
        rep[k] = _rel(got, w)
        assert np.abs(w).max() > 0, k
    print(f"METRIC raygrad entry {what}", json.dumps(rep))
    empty = np.setdiff1d(np.arange(R), inp["ridx"].numpy())
    for k in ("o", "d", "v"):
        e = outs[k][:R][torch.as_tensor(empty, device="cuda")]
        assert bool((e == 0).all()) and not bool(torch.signbit(e).any()), k          # rays without a sample: +0
    for k, e in rep.items():
        assert e <= RAY_REL, (k, e)
    return rep


ENTRY = [(1, 16, None), (127, 16, None), (128, 16, None), (129, 16, None), (3000, 16, None), (67661, 16, None), (3000, 16, 10),
         (129, 12, None), (3000, 12, None), (3000, 12, 8)]


@pytest.mark.parametrize("n,levels,max_level", ENTRY, ids=[f"n{n}-L{l}-ml{m}" for n, l, m in ENTRY])
def test_entry_points_against_float64(n, levels, max_level):
    model = _level_model(levels)
    ml = max_level if max_level is not None else model.implicit_surface._ml(None)
    inp = ag._inputs(n, 4, seed=n + levels, long_ray=n > 500)
    outs, _ = _entry(model, inp, ml)
    _check_entry(f"colour n={n} L={levels} ml={ml}", outs, _want(model, inp, ml), inp)
    outs, _ = _entry(model, inp, ml, rgb=False)
    _check_entry(f"geometry n={n} L={levels} ml={ml}", outs, _want(model, inp, ml, rgb=False), inp)
    assert bool((outs["v"][:inp["R"]] == 0).all())
    outs, _ = _entry(model, inp, ml, sdf=True)
    _check_entry(f"sdf n={n} L={levels} ml={ml}", outs, _want(model, inp, ml, sdf=True), inp)


def test_entry_point_wrong_reference_fails():
    """on a table of zeros (J = 0) g_x is the radiance input's direct dL/dx alone: the entry point matches the reference, and a reference
    without that term must fail"""
    model = _level_model(16, zero_table=True)
    ml = model.implicit_surface._ml(None)
    inp = ag._inputs(3000, 4, seed=91, long_ray=True)
    outs, _ = _entry(model, inp, ml)
    _check_entry("colour zero table", outs, _want(model, inp, ml), inp)
    wrong = _want(model, inp, ml, drop_rad_x=True)
    e = _rel(wrong[0], outs["o"][:inp["R"]].cpu().numpy())           # relative to the kernel's gradient (the wrong one is all zero here)
    print(f"METRIC raygrad entry wrong reference rel={e:.2e}")
    assert e > RAY_REL


@pytest.mark.parametrize("sdf", [False, True], ids=["colour", "sdf"])
def test_entry_point_device_count(sdf):
    """count below the capacity: rows past the count and the ray only those rows name stay untouched, and the counted rays get the bits
    of a launch of exactly the count"""
    model = _level_model(16)
    ml = model.implicit_surface._ml(None)
    inp = ag._inputs(5000, 4, seed=78, long_ray=True)
    a, ra = _entry(model, inp, ml, sdf=sdf)
    b, rb = _entry(model, inp, ml, sdf=sdf, cap_extra=700)
    R, n = inp["R"], 5000
    for k in ("o", "d") + (() if sdf else ("v",)):
        assert torch.equal(b[k][:R], a[k][:R]) and bool((b[k][R] == SENT).all()), k
    w, m = (8 if sdf else 12), n + 700                   # the per-sample ray rows: the first rows x w floats of the scratch
    fa, fb = ra.view(-1), rb.view(-1)
    assert torch.equal(fb[:n * w], fa[:n * w]) and bool((fb[n * w:m * w] == SENT).all())


# ===================================================================================================================== 2. the autograd ops

_MODELS = {}


def _model(max_level):
    if max_level not in _MODELS:
        m = tk._model(64, 64, 4, seed=300)
        m.max_level = max_level
        _MODELS[max_level] = m
    return _MODELS[max_level]


def _case(n, seed):
    inp = ag._inputs(n, 4, seed, long_ray=n > 500)
    cu = lambda a: a.cuda()
    leaf = lambda a: a.cuda().requires_grad_(True)
    return dict(R=inp["R"], ridx=cu(inp["ridx"]), t=cu(inp["t"]), o=leaf(inp["o"]), d=leaf(inp["d"]), v=leaf(inp["v"]), ha=leaf(inp["ha"]),
                cot=[cu(c) for c in inp["cot"]])


def _module_x(c):
    return torch.addcmul(c["o"][c["ridx"]], c["d"][c["ridx"]], c["t"].unsqueeze(-1))


def _loss(out, cot, rgb=True):
    return (out["sdf"].float() * cot[0]).sum() + (out["nablas"].float() * cot[1]).sum() + ((out["rgb"].float() * cot[2]).sum() if rgb else 0)


def _grads(loss, leaves):
    return torch.autograd.grad(loss, leaves, allow_unused=True)


def _check(what, got, want, c, leaves):
    rep = {}
    for k, a, b in zip(leaves, got, want):
        assert a is not None and b is not None, k
        rep[k] = rel_l2(a, b)
        assert torch.isfinite(a).all(), k
    empty = np.setdiff1d(np.arange(c["R"]), c["ridx"].cpu().numpy())
    for k, a in zip(leaves, got):
        if k != "ha":
            e = a.detach()[torch.as_tensor(empty, device=a.device)]
            assert bool((e == 0).all()) and not bool(torch.signbit(e).any()), k          # rays without a sample: +0
    print(f"METRIC raygrad {what}", json.dumps(rep))
    for k, e in rep.items():
        assert e <= MODULE_REL, (k, e)
    return len(empty)


SIZES = [1, 127, 128, 129, 3000, 67661]


@pytest.mark.parametrize("max_level", [None, 10], ids=["all-levels", "max-level-10"])
@pytest.mark.parametrize("n", SIZES)
def test_color_op_ray_grads_against_module_path(n, max_level):
    from neuralsim_b200.fields.fused_color import fused_color
    model = _model(max_level)
    c = _case(n, seed=n + 5)
    out = fused_color(model, c["ridx"], c["t"], c["o"], c["d"], c["v"], c["ha"])
    leaves = ["o", "d", "v", "ha"]
    got = _grads(_loss(out, c["cot"]), [c[k] for k in leaves])
    ref = model.forward(_module_x(c), v=c["v"][c["ridx"]], h_appear=c["ha"][c["ridx"]], nablas_has_grad=True)
    want = _grads(_loss(ref, c["cot"]), [c[k] for k in leaves])
    n_empty = _check(f"color n={n} max_level={max_level}", got, want, c, leaves)
    assert n < 8 or n_empty >= 1
    # deterministic: the same bits on a second run
    out2 = fused_color(model, c["ridx"], c["t"], c["o"], c["d"], c["v"], c["ha"])
    got2 = _grads(_loss(out2, c["cot"]), [c[k] for k in leaves])
    for a, b in zip(got, got2):
        assert torch.equal(a, b)


@pytest.mark.parametrize("n", [129, 3000])
def test_geometry_op_ray_grads_against_module_path(n):
    """the geometry-only form (LiDAR rays: sdf + nablas, no radiance net runs)"""
    from neuralsim_b200.fields.fused_color import fused_color
    model = _model(None)
    c = _case(n, seed=n + 11)
    out = fused_color(model, c["ridx"], c["t"], c["o"], c["d"], with_rgb=False)
    got = _grads(_loss(out, c["cot"], rgb=False), [c["o"], c["d"]])
    ref = model.forward_sdf_nablas(_module_x(c), nablas_has_grad=True)
    want = _grads(_loss(ref, c["cot"], rgb=False), [c["o"], c["d"]])
    _check(f"geometry n={n}", got, want, c, ["o", "d"])


@pytest.mark.parametrize("n", [1, 128, 129, 3000, 67661])
def test_sdf_op_ray_grads_against_module_path(n):
    """the boundary samples' SDF query (k_sdf_bwd_tc<true, true>), with the compaction of zero cotangents"""
    model = _model(None)
    c = _case(n, seed=n + 17)
    s = model.implicit_surface
    cot = c["cot"][0] * (torch.arange(n, device="cuda") % 3 != 0)          # a third of the samples carry no cotangent
    sdf = s.fused_sdf_rays_autograd(c["ridx"], c["t"], c["o"], c["d"])
    got = _grads((sdf * cot).sum(), [c["o"], c["d"]])
    want = _grads((s.forward(_module_x(c))["sdf"].float() * cot).sum(), [c["o"], c["d"]])
    _check(f"sdf n={n}", got, want, c, ["o", "d"])


# ===================================================================================================================== host-sized render
def _pose(params, ro, rd):
    """a learnable SE(3) correction of the rays: rotation exp(omega) (Rodrigues) and translation"""
    omega, trans = params[:3], params[3:]
    th = omega.norm().clamp_min(1e-12)
    k = omega / th
    K = torch.zeros(3, 3, device=ro.device, dtype=ro.dtype)
    K = K.index_put((torch.tensor([2, 1, 0, 2, 1, 0]), torch.tensor([1, 2, 2, 0, 0, 1])), torch.stack([k[0], -k[0], k[1], -k[1], k[2], -k[2]]))
    Rm = torch.eye(3, device=ro.device) + torch.sin(th) * K + (1 - torch.cos(th)) * (K @ K)
    return ro @ Rm.T + trans, rd @ Rm.T


def _render_loss(model, ro, rd, codes, w, params):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    o, d = _pose(params, ro, rd)
    out = SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=codes)["rendered"]
    return ag._loss(out, w), out


def _fused_only(model, mp):
    """the host-sized fused query must run (counted in the returned list), and no query may reach the module path"""
    from neuralsim_b200.graphics import neus as GN
    def module_path(*a, **k):
        raise AssertionError("a query fell back to the module path")
    mp.setattr(model, "forward", module_path)
    mp.setattr(model.implicit_surface, "forward", module_path)
    calls, orig = [], GN._query_fused

    def spy(*a, **k):
        ret = orig(*a, **k)
        calls.append(ret is not None)
        return ret
    mp.setattr(GN, "_query_fused", spy)
    return calls


def test_host_sized_render_with_learnable_pose(cuda, monkeypatch):
    """camera rays from a learnable pose (and learnable codes): the fused query runs, and the pose, code and parameter gradients match
    the module path's"""
    from neuralsim_b200.graphics import neus as GN
    _, model = make_pair(cuda)
    model.train()
    ro, rd, codes0, w = ag._frame_rays(cuda)
    p0 = torch.tensor([0.01, -0.02, 0.015, 0.01, 0.02, -0.01], device=cuda)

    def run():
        model.zero_grad(set_to_none=True)
        params, codes = p0.clone().requires_grad_(True), codes0.clone().requires_grad_(True)
        loss, out = _render_loss(model, ro, rd, codes, w, params)
        loss.backward()
        return params.grad.clone(), codes.grad.clone(), product_grads(model), {k: v.detach().clone() for k, v in out.items()}

    with monkeypatch.context() as mp:
        calls = _fused_only(model, mp)
        gp, gc_, gm, out_f = run()
    assert calls and all(calls)
    with monkeypatch.context() as mp:
        mp.setattr(GN, "FUSED_STAGES", False)
        mp_gp, mp_gc, mp_gm, out_m = run()
    rep = dict(pose=rel_l2(gp, mp_gp), codes=rel_l2(gc_, mp_gc), rgb=rel_l2(out_f["rgb_volume"], out_m["rgb_volume"]))
    rep.update({k: rel_l2(v, mp_gm[k]) for k, v in gm.items() if v is not None and k != "ln_inv_s"})
    print("METRIC raygrad host-sized", json.dumps(rep))
    assert float(gp.abs().max()) > 0
    for k, e in rep.items():
        assert e <= MODULE_REL, (k, e)


def test_adam_steps_move_pose_as_module_path(cuda, monkeypatch):
    """a few Adam steps on the pose alone (the model fixed) take it where the module path takes it"""
    from neuralsim_b200.graphics import neus as GN
    _, model = make_pair(cuda)
    model.train()
    for p in model.parameters():
        p.requires_grad_(False)
    ro, rd, codes, w = ag._frame_rays(cuda)

    def steps():
        params = torch.tensor([0.02, -0.01, 0.01, 0.03, 0.0, -0.02], device=cuda, requires_grad=True)
        opt = torch.optim.Adam([params], lr=2e-3)
        for _ in range(4):
            opt.zero_grad()
            _render_loss(model, ro, rd, codes, w, params)[0].backward()
            opt.step()
        return params.detach().clone()

    with monkeypatch.context() as mp:
        calls = _fused_only(model, mp)
        a = steps()
    assert len(calls) == 4 and all(calls)
    with monkeypatch.context() as mp:
        mp.setattr(GN, "FUSED_STAGES", False)
        b = steps()
    start = torch.tensor([0.02, -0.01, 0.01, 0.03, 0.0, -0.02], device=cuda)
    moved_f, moved_m = a - start, b - start
    print("METRIC raygrad adam", json.dumps(dict(moved_rel=rel_l2(moved_f, moved_m))))
    assert float(moved_m.abs().min()) > 0
    assert rel_l2(moved_f, moved_m) <= 0.1
