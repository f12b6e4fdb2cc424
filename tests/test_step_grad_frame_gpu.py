"""The benchmark's own training step (bench.py: the 800x600 frame, bench.build_model, near=0.01, zero appearance codes, training mode,
gradients through bench.flat_grad_views) pinned to a float64 replay of the step on its own samples (oracle/step64.py).

Masked cotangent at full size.  The loss is bench.loss_of of the rendered buffers with every ray weighted by a mask w_r: 1 on a seeded
subset of 4096 hit rays (spread over the frame) and 64 misses, 0 elsewhere.  The kernels still run every sample of the frame:
each persistent backward CTA sums its 40-85 tiles, most of them carrying a zero cotangent, the kept-sample alpha backward and the
colour backward add into one table gradient, and the 8x4 pixel blocks decide which samples share a warp's merged update.  The loss is
a sum over rays, so the float64 replay of the subset alone is the exact expected gradient.  Its decisions (boundary samples, kept
samples, early stops) are read off the host-sized step's own forward by wrapping the fused query's stage functions; the graph step's
forward is bit-equal to the host-sized one (checked here on the rendered buffers), so the same replay judges both.  The graph step takes
its mask from a tensor its loss captured, rewritten in place between replays: a replay must follow a changed cotangent.

Bounds.  oracle/fused64.py with rounding=True rounds to fp16 exactly where the kernels round, so what separates the kernels from the
replay is (a) fp32 summation order (atomics and wgmma accumulation, ~2^-24 of the summed magnitudes, far below the bounds) and (b) the
rare fp16 value that lands on the other side of a rounding boundary because of (a) or the SFU softplus of the SDF query
(tests/test_tc_kernels_gpu.py: <= 2.3e-3 of the boundary sdf values, one ulp).  A flipped boundary sdf moves x = sdf inv_s by up to
2^-11 |x|: the alpha of that interval, and through the transmittance every later weight of its ray, move by ~5e-4 relative near the
surface and up to ~5e-3 at |x| ~ 10, where the weights are small.  About one ray in five has such a flip among the ~100 boundary
samples its kept alphas read, so a gradient summed over the subset moves by ~1e-4 relative; a table entry that few samples reach moves
by up to the ray's own change.  Flips of different rays are independent, so they add in quadrature while the gradient adds
coherently: with n rays the bounds below (for N_SUBSET = 4096) grow by sqrt(4096 / n) (the random batch has a few hundred hits).
Hit rays are rays whose mask exceeds 0.5: on a grazing ray the kept alphas are differences of sigmoids near 1, which fp32 resolves
only to ~2^-24 of 1, and the normalised depth divides by the ray's tiny mask, so its gradient is fp32 noise in the kernels and in the
reference CUDA alike.  Hence:
  REL = 6e-4          rel-L2 of every tensor and of every LoTD level's slice of the table gradient (3x to 13x tighter than
                      tests/test_render_gpu.py's GRAD_TOL, 2e-3 to 8e-3)
  WORST = 2e-4        the largest entry error of a level relative to that level's norm
  exact zeros         entries the replay leaves exactly zero are cells no subset sample reaches; the kernels must leave them exactly
                      zero (a zero cotangent adds +-0): any value there leaked in from another ray
  LIN_REL = 2e-5      linearity: K = 4 disjoint masks covering every ray sum to the all-ones gradient up to fp32 atomic summation
                      order, the bound tests/test_static_gpu.py puts on two summation orders of the same step
At the 800x600 frame the rgb cotangent w_k / (3 * 480000) rounds to zero where the contract rounds it to fp16 (r16(g_rgb)), so the
radiance net's float64 gradient is exactly zero there and the kernels' must be exactly zero too; the 4096-ray batch exercises it.
Sensitivity: two deliberately wrong float64 references -- one kept sample dropped in every ~1000th ray of the subset, one level's
table contribution dropped on a tenth of the samples -- must fail the same assertions the real comparison passes.
"""
import json

import numpy as np
import pytest
import torch

import bench
from oracle import fused64, neus64, step64
from util import product_grads

pytestmark = pytest.mark.gpu

N_SUBSET, N_MISS = 4096, 64
EPS, THRE = 1e-4, 0.0                   # the query's early-stop eps and alpha threshold (graphics/neus_fused.py defaults)
REL, WORST, LIN_REL = 6e-4, 2e-4, 2e-5
DROP_LEVEL = 8                          # the level the second wrong reference loses on a tenth of the samples
KEYMAP = dict(grid="grid", W1="dec_W1", b1="dec_b1", W2="dec_W2", b2="dec_b2", R1="rad_W1", rb1="rad_b1", R2="rad_W2", rb2="rad_b2",
              R3="rad_W3", rb3="rad_b3", ln_inv_s="ln_inv_s")
CASES = {"frame-view0": (0, False), "frame-view3": (3, False), "random4096-view0": (0, True)}
_CACHE = {}


def _weigh(rendered, mask):
    return {k: v * (mask if v.dim() == 1 else mask[:, None]) for k, v in rendered.items()}


def _rays(view, random, device):
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(view, bench.N_VIEWS))
    if random:                              # bench.py --random-rays --rays 4096
        sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(1000 + view))[:4096]
        o, d = o[sel], d[sel]
    return o.contiguous().to(device), d.contiguous().to(device)


class _Capture:
    """records the host-sized query's decisions by wrapping its stage functions (nothing is added to the product)"""

    def __init__(self, monkeypatch, model):
        from neuralsim_b200.graphics import neus_fused as NF
        self.rec = {}

        def wrap(name, fn, keep):
            def w(*a, **k):
                r = fn(*a, **k)
                self.rec[name] = keep(a, k, r)
                return r
            return w
        monkeypatch.setattr(NF, "assemble_boundary", wrap("boundary", NF.assemble_boundary, lambda a, k, r: dict(d1=r[0], pinfo=r[3])))
        monkeypatch.setattr(NF, "neus_alpha_compact", wrap("compact", NF.neus_alpha_compact, lambda a, k, r: dict(
            r, alpha=r["alpha"].detach(), inv_s=float(a[1].detach()))))
        monkeypatch.setattr(model, "forward_on_rays", wrap("color", model.forward_on_rays, lambda a, k, r: dict(
            ridx=a[0], t=a[1], rays_o=a[2], rays_d=a[3], view=a[4], h_appear=a[5])))

    def host(self):
        return {k: {kk: (vv.detach().cpu().numpy() if torch.is_tensor(vv) else vv) for kk, vv in v.items()} for k, v in self.rec.items()}


def _host_step(model, o, d, mask, flat):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    flat.zero_()
    out = SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=torch.zeros(o.shape[0], 4, device=o.device))["rendered"]
    bench.loss_of(_weigh(out, mask)).backward()
    return {k: v.detach().clone() for k, v in out.items()}, product_grads(model)


def _decisions(c, rays_of_packs):
    """decisions of the kept packs `rays_of_packs` (indices into the compressed packs) from a capture"""
    comp, bnd, col = c["compact"], c["boundary"], c["color"]
    assert np.array_equal(col["ridx"], comp["ridx"]) and np.array_equal(col["t"].view(np.int32), comp["t"].view(np.int32))
    u = np.asarray(rays_of_packs, np.int64)
    tr = comp["nidx"][u]                                       # tested ray of each pack
    b, n = bnd["pinfo"][tr, 0], bnd["pinfo"][tr, 1]
    kb, kn = comp["pack_infos"][u, 0], comp["pack_infos"][u, 1]
    nb = np.cumsum(n) - n
    bidx = np.repeat(b - nb, n) + np.arange(int(n.sum()))
    kidx = np.repeat(kb - (np.cumsum(kn) - kn), kn) + np.arange(int(kn.sum()))
    kpi = np.stack([np.cumsum(kn) - kn, kn], 1)
    a32 = comp["alpha"][kidx]
    vis_f = neus64.replay(a32, kpi, EPS, THRE)["vis"]
    vis_b = neus64.replay(a32, kpi, EPS, THRE, backward=True)["vis"]
    assert vis_f.all() and vis_b.all()                          # the compression kept exactly what the compositing visits
    return dict(o=col["rays_o"][tr], d=col["rays_d"][tr], view=col["view"][tr], h_appear=col["h_appear"][tr], t1=bnd["d1"][bidx],
                pinfo=np.stack([nb, n], 1), kept=comp["pidx"][kidx] - np.repeat(b - nb, kn), kept_pinfo=kpi, t_kept=comp["t"][kidx],
                vis_fwd=vis_f, vis_bwd=vis_b)


def _cotangents(n_batch, R):
    """d loss_of / d (mask, depth, rgb, normals) of a weighted ray: fp32 1/numel of each mean"""
    a, b = float(np.float32(1) / np.float32(n_batch)), float(np.float32(1) / np.float32(3 * n_batch))
    return dict(g_mask=np.full(R, a), g_depth=np.full(R, a), g_rgb=np.full((R, 3), b), g_nablas=np.full((R, 3), b))


def _compare(got, ref, meta, n_sub):
    """-> (report, failures): per tensor rel-L2, per LoTD level rel-L2 / worst entry / leaked zeros.  The bounds hold for N_SUBSET rays;
    fewer rays average their independent flips less: sqrt(N_SUBSET / n_sub) times the bound"""
    rep, fail = {}, []
    f = max(1.0, (N_SUBSET / n_sub) ** 0.5)
    rel_b, worst_b = REL * f, WORST * f
    for k, pk in KEYMAP.items():
        g, r = got[pk].double().numpy().reshape(-1), np.asarray(ref[k], np.float64).reshape(-1)
        rel = float(np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-300))
        rep[k] = rel
        if rel > rel_b:
            fail.append(f"{k}: rel-L2 {rel:.2e} > {rel_b:.1e}")
        if k != "grid":
            continue
        for lvl in range(meta.n_levels):
            s = slice(meta.level_offsets[lvl], meta.level_offsets[lvl + 1])
            gl, rl = g[s], r[s]
            nrm = max(np.linalg.norm(rl), 1e-300)
            lrel, worst = float(np.linalg.norm(gl - rl) / nrm), float(np.abs(gl - rl).max() / nrm)
            leaked = int(((rl == 0) & (gl != 0)).sum())
            rep[f"grid.L{lvl}"] = dict(rel=lrel, worst=worst, leaked=leaked, touched=int((rl != 0).sum()))
            if lrel > rel_b:
                fail.append(f"grid level {lvl}: rel-L2 {lrel:.2e} > {rel_b:.1e}")
            if worst > worst_b:
                fail.append(f"grid level {lvl}: worst entry {worst:.2e} of the level norm > {worst_b:.1e}")
            if leaked:
                fail.append(f"grid level {lvl}: {leaked} entries nonzero where no subset sample reaches")
    return rep, fail


def _linearity(step, n, g_all, device, seed):
    """K = 4 disjoint masks covering every ray: their gradients sum to the all-ones gradient"""
    part = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).to(device) % 4
    acc = None
    for q in range(4):
        g = step((part == q).float())
        acc = {k: v.double() for k, v in g.items()} if acc is None else {k: acc[k] + g[k].double() for k in acc}
    res = {k: float((acc[k] - g_all[k].double()).norm() / g_all[k].double().norm().clamp_min(1e-300)) for k in g_all}
    return res


def _run_case(name, monkeypatch, dev):
    if name in _CACHE:
        return _CACHE[name]
    import time
    from neuralsim_b200.graphics.neus_static import StaticFrame
    view, random = CASES[name]
    model = bench.build_model(dev).train()
    flat, params = bench.flat_grad_views(model)
    views = [p.grad.data_ptr() for p in params]
    o, d = _rays(view, random, dev)
    n = o.shape[0]
    cap = _Capture(monkeypatch, model)
    ones = torch.ones(n, device=dev)
    r_all, g_all = _host_step(model, o, d, ones, flat)
    assert [p.grad.data_ptr() for p in params] == views            # gradients accumulate in the flat buffer
    c0 = cap.host()
    # the subset: seeded, spread over the frame; hit rays are rays that render the surface (mask > 0.5), misses rays without a kept sample
    hit = c0["compact"]["rays_inds_hit"]
    solid = np.nonzero(r_all["mask_volume"].cpu().numpy()[hit] > 0.5)[0]
    rng = np.random.default_rng(view * 7 + int(random))
    n_sub = N_SUBSET if solid.shape[0] >= 2 * N_SUBSET else solid.shape[0]       # the training batch: all its solid hits
    packs = np.sort(rng.choice(solid, n_sub, replace=False))
    miss = np.setdiff1d(np.arange(n), hit)
    miss = rng.choice(miss, min(N_MISS, miss.shape[0]), replace=False)
    mask = torch.zeros(n, device=dev)
    mask[torch.from_numpy(hit[packs]).to(dev)] = 1.0
    mask[torch.from_numpy(miss).to(dev)] = 1.0
    r_sub, g_host = _host_step(model, o, d, mask, flat)
    c1 = cap.host()
    # same forward, same decisions
    assert np.array_equal(c1["compact"]["pidx"], c0["compact"]["pidx"]) and np.array_equal(c1["boundary"]["d1"].view(np.int32),
                                                                                            c0["boundary"]["d1"].view(np.int32))
    for k in r_all:
        assert torch.equal(r_sub[k], r_all[k]), k
    dec = _decisions(c1, packs)
    ref64 = fused64.Fused64.from_model(model)
    t0 = time.time()
    ref = step64.step_grads(ref64, dec, c1["compact"]["inv_s"], **_cotangents(n, n_sub), ln_inv_s_factor=model.ctrl_var.ln_inv_s_factor)
    t_replay = time.time() - t0
    meta = ref64.meta

    def host_grads(m):
        return _host_step(model, o, d, m, flat)[1]
    lin_host = _linearity(host_grads, n, g_all, dev, seed=view)
    # the graph step: capture once, the mask a tensor its loss reads, rewritten between replays
    monkeypatch.undo()
    gmask = torch.ones(n, device=dev)
    frame = StaticFrame(model, n, loss_fn=lambda rendered: bench.loss_of(_weigh(rendered, gmask)), near=0.01, pre_hook=flat.zero_)

    def graph_grads(m):
        gmask.copy_(m)
        frame.step(o, d, None)
        assert frame.counts()["overflow"] == 0
        return product_grads(model)
    g_graph_all = graph_grads(ones)
    for k in r_all:
        assert torch.equal(frame.rendered[k], r_all[k]), k           # bit-equal forward: the same decisions
    g_graph = graph_grads(mask)
    lin_graph = _linearity(graph_grads, n, g_graph_all, dev, seed=view + 100)
    assert frame.captures == 1
    sel = torch.from_numpy(hit[packs]).to(dev)
    fwd = {k: float(np.linalg.norm(r_all[k + "_volume"][sel].double().cpu().numpy() - ref["out"][k]) / np.linalg.norm(ref["out"][k]))
           for k in ("mask", "depth", "rgb", "normals")}
    res = dict(fwd=fwd, n=n, n_sub=n_sub, kept=int(dec["kept"].shape[0]), boundary=int(dec["t1"].shape[0]), t_replay=t_replay, ref=ref, dec=dec,
               ref64=ref64, meta=meta, inv_s=c1["compact"]["inv_s"], factor=model.ctrl_var.ln_inv_s_factor, host=g_host, graph=g_graph,
               lin_host=lin_host, lin_graph=lin_graph)
    _CACHE[name] = res
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_step_gradients_match_float64_replay(cuda, monkeypatch, name):
    r = _run_case(name, monkeypatch, cuda)
    out = dict(case=name, rays=r["n"], subset=r["n_sub"], kept_samples=r["kept"], boundary_samples=r["boundary"],
               replay_seconds=round(r["t_replay"], 1), forward_rel_l2=r["fwd"],
               norms={k: float(np.linalg.norm(r["ref"][k])) for k in KEYMAP})
    fails = []
    for path in ("host", "graph"):
        rep, f = _compare(r[path], r["ref"], r["meta"], r["n_sub"])
        out[path] = rep
        fails += [f"{path}: {x}" for x in f]
        lin = r[f"lin_{path}"]
        out[f"linearity_{path}"] = lin
        fails += [f"{path} linearity: {k} {v:.2e} > {LIN_REL:.0e}" for k, v in lin.items() if v > LIN_REL]
    print(json.dumps(out))
    assert not fails, fails


def _drop_kept(dec, every):
    """dec with the middle kept sample of every `every`-th ray (with >= 2 kept) removed: that ray composites one sample fewer"""
    kpi = dec["kept_pinfo"]
    rays = np.nonzero(kpi[:, 1] >= 2)[0][::every]
    drop = kpi[rays, 0] + kpi[rays, 1] // 2
    keep = np.ones(dec["kept"].shape[0], bool)
    keep[drop] = False
    out = dict(dec)
    for k in ("kept", "t_kept", "vis_fwd", "vis_bwd"):
        out[k] = dec[k][keep]
    kn = kpi[:, 1].copy()
    kn[rays] -= 1
    out["kept_pinfo"] = np.stack([np.cumsum(kn) - kn, kn], 1)
    return out, rays


def test_wrong_references_fail(cuda, monkeypatch):
    """the bounds can fail: two float64 references with a deliberate, small defect fail the comparison the kernels pass"""
    r = _run_case("frame-view0", monkeypatch, cuda)
    dec, ref, ref64, n = r["dec"], r["ref"], r["ref64"], r["n"]
    R = dec["pinfo"].shape[0]
    g = _cotangents(n, R)
    kw = dict(ln_inv_s_factor=r["factor"])
    # (1) one kept sample dropped in every ~1000th ray: replay only those rays both ways (the gradient is a sum over rays)
    bad, rays = _drop_kept(dec, 1000)
    sub = lambda dd: step64.step_grads(ref64, step64.select(dd, rays), r["inv_s"], **{k: v[rays] for k, v in g.items()}, **kw)
    right, wrong = sub(dec), sub(bad)
    ref1 = {k: ref[k] - right[k] + wrong[k] for k in KEYMAP}
    # (2) level DROP_LEVEL's table contribution dropped on the samples of every 10th ray (a tenth of the samples)
    tenth = np.arange(0, R, 10)
    part = step64.step_grads(ref64, step64.select(dec, tenth), r["inv_s"], **{k: v[tenth] for k, v in g.items()}, **kw)
    meta = r["meta"]
    s = slice(meta.level_offsets[DROP_LEVEL], meta.level_offsets[DROP_LEVEL + 1])
    ref2 = dict(ref)
    ref2["grid"] = ref["grid"].copy()
    ref2["grid"][s] -= part["grid"][s]
    report = {}
    for tag, bad_ref in (("dropped kept sample", ref1), ("dropped level contribution", ref2)):
        for path in ("host", "graph"):
            _, f = _compare(r[path], bad_ref, meta, r["n_sub"])
            report[f"{tag} / {path}"] = f
            assert f, (tag, path)
    print(json.dumps(dict(rays_with_a_dropped_sample=len(rays), failures=report)))
