"""The StreetSurf training step (bench_cfg3.py: cuboid 40 x 150 x 15 m box, cuboid `ngp` LoTD with hashed levels, 128 coarse samples +
[8, 8, 32] fine, sdf_scale 25, inv_s ~ 200) pinned to a float64 replay of the step on its own samples (oracle/step64.py), on the
host-sized step and on the one-launch graph step (StaticFrame).  The method is tests/test_step_grad_frame_gpu.py's: the decisions
(boundary samples, kept samples, early stops) are read off the host-sized step's own forward by wrapping the query's stage functions, the
graph step's forward is bit-equal to it (checked on the rendered buffers), and the replay of those decisions in float64 is the expected
gradient.  What the cubic cfg2 frame cannot check and this file does: the per-axis ray normalisation d / radius3d, the per-axis nablas
scale fac = sdf_scale / radius3d_original (25/20, 25/75, 25/7.5), the cuboid level resolutions, the geometry-only query of LiDAR rays,
the LiDAR loss's line-of-sight cotangent entering the compositing adjoint as a per-sample g_vw, and the 17-level (48-column) kernels.

Cases (8192 rays each unless stated):
  camera      bench_cfg3.build_model (16 levels, 2^20 hash, 32 Mi parameters), camera_rays with random codes, loss_cam on weighted buffers
  lidar       the same model, lidar_rays, with_rgb=False, loss_lidar on weighted buffers
  lidar-loss  the same model and the 12-level LiDAR-only model (tests/test_partial_levels_gpu._cfg3_geo12), 4096 lidar_rays with the
              ranges of tests/test_lidar_loss_gpu._ranges, LidarLoss(LIDAR_CFG) (l1 depth, neus_unisim line of sight, toofar 80, median
              x 100); the graph step runs it with loss_on_ret=True.  The loss is not a sum over rays, so the whole batch is replayed:
              the cotangents g_depth [R] and g_vw [K] come from oracle/lidar64.py, given the kernels' fp32 rendered depth, the fp32 kept
              depths and the replay's float64 weights, its mask equal to LidarLoss.mask bit for bit
  camera-17   tests/test_wide_levels_gpu._small17 (17 levels, the shipped camera table count, max_fused_levels=24), camera rays with
              codes; the code gradients against tests/appear64.step_code_grads as well
The weighted cases weigh every ray by a mask w_r: n (the batch size, a power of two) on a seeded subset of <= N_SUBSET solid hits
(mask > 0.5) and N_MISS misses, 0 elsewhere; the loss is a sum over rays, so the replay of the subset is the exact expected gradient of
the whole step.  The weight n makes each mean's cotangent of order one (exactly: 1/n times n in fp32): at weight 1 the rgb cotangent
1/(3n) = 4e-5 puts the radiance backward in fp16's subnormal range (r16(g_rgb), dZ2 and dZ1 of oracle/fused64.py fall to a few ulps of
2^-24), where a one-ulp flip changes a value by 100 %: measured so, the code gradients of the camera case sat at 2.2e-3 rel-L2 and a few
table entries per level were zero on one side only.  The lidar-loss case multiplies the loss by n for the same reason (its cotangents
0.05 / n per ray and 0.1 / n_kept 2 vw per sample put the sdf backward's dz there: measured so, levels 4-8 sat at 1.7e-3 to 2.9e-3
rel-L2 with the whole table at 7.5e-5), and sets the ranges of the beams that do not see the road solidly
(rendered mask <= 0.5) beyond discard_toofar, so the loss reads solid rays only, and replays the rays in the loss's mask.

Bounds.  oracle/fused64.py rounds to fp16 exactly where the kernels round, so what separates the kernels from the replay is fp32
summation order and the rare fp16 value on the other side of a rounding boundary (test_step_grad_frame_gpu.py).  A flipped boundary sdf
moves x = sdf inv_s by up to 2^-11 |x|.  Here inv_s ~ 200 and the plane's sdf is dz / 25 (dz in metres), so x = 8 dz: the kept alphas of
a ray span |x| <~ 10 over ~1.2 m around the road, and the 32 + 8 + 8 fine samples put ~40 boundary samples there (the coarse 1.2 m
steps add one or two).  The flip argument of the 800x600 frame is the same per ray: an interval's alpha and every later weight of its ray
move by ~5e-4 relative near the surface, ~5e-3 at |x| ~ 10 where the weights are small; about one ray in five has such a flip among the
boundary samples its kept alphas read, so a gradient summed over 4096 rays moves by ~1e-4 relative, a table entry few samples reach
by up to its ray's change.  The street packs are far longer (~150 kept samples per ray: every sample before the road has a tiny positive
alpha) but their weight sits on the same few intervals around the zero crossing, so the per-ray change does not grow with them.  The per-axis fac multiplies the nablas by 1.25,
0.33 and 3.33: an fp16 flip of the nablas chain moves the z component most, by the same relative amount.  Rays that see the plane
at a grazing angle (the far LiDAR beams) have long kept packs with small weights: fp32 resolves their alphas to 2^-24 of 1, the same
noise as the frame's grazing rays, and the subset takes solid hits only.  Hence the bounds of the 800x600 frame hold per tensor:
  REL = 6e-4          rel-L2 of every tensor and of every LoTD level's slice of the table gradient
  WORST = 2e-4        the largest entry error of a level relative to that level's norm
  LEAK = 1e-5         entries the replay leaves exactly zero: at most 1e-5 of their level's norm in the kernels' gradient.  Far from
                      the road a sample's sdf cotangent dz = r16(d w2 s) falls below fp16's smallest subnormal (2^-24): one side
                      rounds it to zero, the other to 2^-24, and the cells only that sample reaches are exactly zero on one side only
                      (measured: 0 to ~3000 such entries per case, none above 3.7e-7 of its level's norm); a value leaked in from another ray is as large
                      as that ray's own entries, orders of magnitude above the bound
  LIN_REL = 2e-5      linearity: 4 disjoint masks covering every ray sum to the all-ones gradient up to fp32 atomic order
  FWD_REL = 1e-4      the replay's mask, depth and normals of the replayed rays against the rendered buffers (the replay reproduces the
                      kernels' points: a wrong ray normalisation or fac moves them by far more)
With fewer rays than N_SUBSET the bounds grow by sqrt(N_SUBSET / n) (independent flips average less), as in the frame test.
Sensitivity (test_wrong_references_fail): each deliberately wrong float64 reference fails the assertions the kernels pass -- one kept
sample dropped in every ~1000th ray, one level's contribution dropped on a tenth of the samples, fac with x and y swapped, and on
lidar-loss the line-of-sight g_vw zeroed on every 10th kept ray.

Runtime and memory: the float64 gradient of the 32 Mi-entry table is 256 MB, and the replay holds two more for the colour and sdf
backward passes.  The street packs make the replays long: measured on an H100 80GB HBM3 (700 W power limit, its host's CPUs), 40-120 s
per case over 380 k to 830 k kept samples (printed per case as replay_seconds), about 14 minutes for the file.
"""
import gc
import json
import time

import numpy as np
import pytest
import torch

import bench_cfg3 as C
from appear64 import step_code_grads
from fused64_levels import Fused64Levels
from fused64_wide import Fused64Wide
from oracle import fused64, lidar64, neus64, step64

pytestmark = pytest.mark.gpu

N_SUBSET, N_MISS = 4096, 64
EPS, THRE = 1e-4, 0.0                   # the query's early-stop eps and alpha threshold (graphics/neus_fused.py defaults)
REL, WORST, LIN_REL, FWD_REL, LEAK = 6e-4, 2e-4, 2e-5, 1e-4, 1e-5
DROP_LEVEL = 8                          # the level the second wrong reference loses on a tenth of the samples
RAD = ("R1", "rb1", "R2", "rb2", "R3", "rb3")
KEYS = ("grid", "W1", "b1", "W2", "b2") + RAD + ("ln_inv_s",)
LIDAR_IT = 100                          # the iteration of the lidar-loss case (epsilon 1.5)
CASES = {"camera": ("cfg3", "camera"), "lidar": ("cfg3", "lidar"), "lidar-loss": ("cfg3", "lidar-loss"),
         "lidar-loss-geo12": ("geo12", "lidar-loss"), "camera-17": ("small17", "camera")}
_CACHE = {}


def _model(kind, dev):
    if kind == "cfg3":
        return C.build_model(dev).train(), fused64.Fused64
    if kind == "geo12":
        import test_partial_levels_gpu as pl
        return pl._cfg3_geo12(dev), Fused64Levels
    import test_wide_levels_gpu as wl
    return wl._small17(dev), Fused64Wide


def _grads(model):
    """the parameter gradients under the oracle's names (None where a parameter has none)"""
    s = model.implicit_surface
    d = s.decoder.layers
    ps = dict(grid=s.encoding.flattened_params, W1=d[0].weight, b1=d[0].bias, W2=d[1].weight, b2=d[1].bias, ln_inv_s=model.ctrl_var.ln_inv_s)
    if model.radiance_net is not None:
        ps.update(zip(RAD, [p for l in model.radiance_net.blocks.layers for p in (l.weight, l.bias)]))
    return {k: (None if p.grad is None else p.grad.detach().float().cpu().clone()) for k, p in ps.items()}


def _zero(model):
    for p in model.parameters():                # in place: a captured step keeps accumulating into these tensors
        if p.grad is not None:
            p.grad.zero_()


def _weigh(rendered, mask):
    return {k: v * (mask if v.dim() == 1 else mask[:, None]) for k, v in rendered.items()}


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
        # camera rays: (ridx, t, o, d, view, h_appear); LiDAR rays: (ridx, t, o, d) and with_rgb=False
        monkeypatch.setattr(model, "forward_on_rays", wrap("color", model.forward_on_rays, lambda a, k, r: dict(
            ridx=a[0], t=a[1], rays_o=a[2], rays_d=a[3], view=a[4] if len(a) > 4 else None, h_appear=a[5] if len(a) > 5 else None)))

    def host(self):
        return {k: {kk: (vv.detach().cpu().numpy() if torch.is_tensor(vv) else vv) for kk, vv in v.items()} for k, v in self.rec.items()}


def _decisions(c, rays_of_packs):
    """decisions of the kept packs `rays_of_packs` (indices into the compressed packs) from a capture"""
    comp, bnd, col = c["compact"], c["boundary"], c["color"]
    assert np.array_equal(col["ridx"], comp["ridx"]) and np.array_equal(col["t"].view(np.int32), comp["t"].view(np.int32))
    u = np.asarray(rays_of_packs, np.int64)
    tr = comp["nidx"][u]                                       # tested ray of each pack
    b, n = bnd["pinfo"][tr, 0], bnd["pinfo"][tr, 1]
    kb, kn = comp["pack_infos"][u, 0], comp["pack_infos"][u, 1]
    nb = np.cumsum(n) - n
    kidx = np.repeat(kb - (np.cumsum(kn) - kn), kn) + np.arange(int(kn.sum()))
    bidx = np.repeat(b - nb, n) + np.arange(int(n.sum()))
    kpi = np.stack([np.cumsum(kn) - kn, kn], 1)
    a32 = comp["alpha"][kidx]
    vis_f = neus64.replay(a32, kpi, EPS, THRE)["vis"]
    vis_b = neus64.replay(a32, kpi, EPS, THRE, backward=True)["vis"]
    assert vis_f.all() and vis_b.all()                          # the compression kept exactly what the compositing visits
    opt = lambda v: None if v is None else v[tr]
    return dict(o=col["rays_o"][tr], d=col["rays_d"][tr], view=opt(col["view"]), h_appear=opt(col["h_appear"]), t1=bnd["d1"][bidx],
                pinfo=np.stack([nb, n], 1), kept=comp["pidx"][kidx] - np.repeat(b - nb, kn), kept_pinfo=kpi, t_kept=comp["t"][kidx],
                vis_fwd=vis_f, vis_bwd=vis_b, ray=comp["rays_inds_hit"][u])


def _cotangents(n_batch, R, kind):
    """d loss / d (mask, depth, rgb, normals) of a ray of weight n_batch for bench_cfg3.loss_cam / loss_lidar: fp32 1/numel of each
    mean (the depth mean's weight 1e-2 rounded to fp32 first) times the weight, exact for a power-of-two batch"""
    f, w = np.float32, np.float32(n_batch)
    assert n_batch & (n_batch - 1) == 0
    a, b, dep = float(f(1) / f(n_batch) * w), float(f(1) / f(3 * n_batch) * w), float(f(f(1e-2) / f(n_batch)) * w)
    g = dict(g_mask=np.full(R, a), g_depth=np.full(R, dep), g_rgb=np.full((R, 3), b), g_nablas=np.full((R, 3), b))
    if kind == "lidar":
        g["g_rgb"] = np.zeros((R, 3))
    return g


def _compare(got, ref, meta, n_sub, radiance):
    """-> (report, failures): per tensor rel-L2, per LoTD level rel-L2 / worst entry / leaked zeros; the radiance net's gradients exactly
    zero (or None) where the rays read no rgb.  The bounds hold for N_SUBSET rays: sqrt(N_SUBSET / n_sub) times them for fewer"""
    rep, fail = {}, []
    f = max(1.0, (N_SUBSET / n_sub) ** 0.5)
    rel_b, worst_b = REL * f, WORST * f
    for k in KEYS:
        if k in RAD and radiance != "rgb":
            # LiDAR rays: nothing reaches the radiance net (a model without one has no such gradient)
            nz = 0 if got.get(k) is None else int((got[k] != 0).sum())
            rep[k] = dict(nonzero=nz)
            if nz:
                fail.append(f"{k}: {nz} nonzero entries on rays without rgb")
            continue
        g, r = got[k].double().numpy().reshape(-1), np.asarray(ref[k], np.float64).reshape(-1)
        rel = float(np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-300))
        rep[k] = rel
        if not rel <= rel_b:
            fail.append(f"{k}: rel-L2 {rel:.2e} > {rel_b:.1e}")
        if k != "grid":
            continue
        for lvl in range(meta.n_levels):
            s = slice(meta.level_offsets[lvl], meta.level_offsets[lvl + 1])
            gl, rl = g[s], r[s]
            nrm = max(np.linalg.norm(rl), 1e-300)
            lrel, worst = float(np.linalg.norm(gl - rl) / nrm), float(np.abs(gl - rl).max() / nrm)
            lk = (rl == 0) & (gl != 0)
            leaked, leaked_max = int(lk.sum()), float(np.abs(gl[lk]).max() / nrm) if lk.any() else 0.0
            rep[f"grid.L{lvl}"] = dict(rel=lrel, worst=worst, leaked=leaked, leaked_max=leaked_max, touched=int((rl != 0).sum()))
            if not lrel <= rel_b:
                fail.append(f"grid level {lvl}: rel-L2 {lrel:.2e} > {rel_b:.1e}")
            if not worst <= worst_b:
                fail.append(f"grid level {lvl}: worst entry {worst:.2e} of the level norm > {worst_b:.1e}")
            if not leaked_max <= LEAK:
                fail.append(f"grid level {lvl}: {leaked} entries nonzero where the replay is zero, up to {leaked_max:.1e} of the level norm")
    return rep, fail


def _linearity(step, n, g_all, device, seed):
    """K = 4 disjoint masks covering every ray: their gradients sum to the all-ones gradient"""
    part = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).to(device) % 4
    acc = None
    for q in range(4):
        g = {k: v for k, v in step((part == q).float()).items() if v is not None}
        acc = {k: v.double() for k, v in g.items()} if acc is None else {k: acc[k] + g[k].double() for k in acc}
    return {k: float((acc[k] - g_all[k].double()).norm() / g_all[k].double().norm().clamp_min(1e-300)) for k in acc
            if float(g_all[k].abs().max()) > 0}


def _fwd_rel(rendered, dec, ref):
    sel = torch.from_numpy(dec["ray"]).to(rendered["mask_volume"].device)
    return {k: float(np.linalg.norm(rendered[k + "_volume"][sel].double().cpu().numpy() - ref["out"][k]) / np.linalg.norm(ref["out"][k]))
            for k in ("mask", "depth", "normals")}


def _weighted_case(name, monkeypatch, dev):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    kind, rays = CASES[name]
    model, ref_cls = _model(kind, dev)
    with_rgb = rays == "camera"
    seed = 2 if kind == "cfg3" else 3
    o, d = (x.to(dev) for x in (C.camera_rays(seed, C.N_CAM) if with_rgb else C.lidar_rays(seed, C.N_LIDAR)))
    n = o.shape[0]
    ha = None
    if with_rgb:
        na = model.radiance_net.blocks.layers[0].in_features - 22 - model.implicit_surface.encoding.out_features
        ha = torch.randn(n, na, device=dev, generator=torch.Generator(dev).manual_seed(11)) * 0.3
    loss = C.loss_cam if with_rgb else C.loss_lidar
    rnd = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=with_rgb, with_normal=True)).train()
    codes = [None]

    def host_step(mask):
        _zero(model)
        h = None
        if with_rgb:
            h = codes[0] = ha.clone().requires_grad_(True)
        out = rnd.render(model, o, d, rays_h_appear=h)["rendered"] if with_rgb else rnd.render(model, o, d)["rendered"]
        loss(_weigh(out, mask)).backward()
        return {k: v.detach().clone() for k, v in out.items()}, _grads(model)
    cap = _Capture(monkeypatch, model)
    ones = torch.ones(n, device=dev)
    r_all, g_all = host_step(ones * n)
    c0 = cap.host()
    hit = c0["compact"]["rays_inds_hit"]
    solid = np.nonzero(r_all["mask_volume"].cpu().numpy()[hit] > 0.5)[0]
    rng = np.random.default_rng(len(name))
    n_sub = N_SUBSET if solid.shape[0] >= 2 * N_SUBSET else solid.shape[0]
    assert n_sub >= 1000, n_sub
    packs = np.sort(rng.choice(solid, n_sub, replace=False))
    miss = np.setdiff1d(np.arange(n), hit)
    miss = rng.choice(miss, min(N_MISS, miss.shape[0]), replace=False)
    mask = torch.zeros(n, device=dev)
    mask[torch.from_numpy(hit[packs]).to(dev)] = float(n)
    mask[torch.from_numpy(miss).to(dev)] = float(n)
    r_sub, g_host = host_step(mask)
    d_codes_host = codes[0].grad.detach().clone() if with_rgb else None
    c1 = cap.host()
    assert np.array_equal(c1["compact"]["pidx"], c0["compact"]["pidx"]) and np.array_equal(c1["boundary"]["d1"].view(np.int32),
                                                                                            c0["boundary"]["d1"].view(np.int32))
    for k in r_all:
        assert torch.equal(r_sub[k], r_all[k]), k
    dec = _decisions(c1, packs)
    ref64 = ref_cls.from_model(model)
    cot = _cotangents(n, n_sub, rays)
    kw = dict(ln_inv_s_factor=model.ctrl_var.ln_inv_s_factor, with_rgb=with_rgb)
    t0 = time.time()
    ref = step64.step_grads(ref64, dec, c1["compact"]["inv_s"], **cot, **kw)
    t_replay = time.time() - t0
    lin_host = _linearity(lambda m: host_step(m * n)[1], n, g_all, dev, seed=5)
    # the graph step: captured once, the mask a tensor its loss reads, rewritten in place between replays
    monkeypatch.undo()
    gmask = torch.ones(n, device=dev)
    _zero(model)
    frame = StaticFrame(model, n, loss_fn=lambda rendered: loss(_weigh(rendered, gmask)), near=C.NEAR, far=C.FAR, with_rgb=with_rgb,
                        slack=2.0, zero_grads=True, h_appear_grad=with_rgb)

    def graph_step(m):
        gmask.copy_(m)
        frame.step(o, d, ha)
        assert frame.counts()["overflow"] == 0
        return _grads(model)
    g_graph_all = graph_step(ones * n)
    for k in r_all:
        assert torch.equal(frame.rendered[k], r_all[k]), k           # bit-equal forward: the same decisions
    g_graph = graph_step(mask)
    d_codes_graph = frame.d_h_appear.detach().clone() if with_rgb else None
    lin_graph = _linearity(lambda m: graph_step(m * n), n, g_graph_all, dev, seed=105)
    assert frame.captures == 1
    res = dict(n=n, n_sub=n_sub, kept=int(dec["kept"].shape[0]), boundary=int(dec["t1"].shape[0]), t_replay=t_replay, ref=ref, dec=dec,
               ref64=ref64, meta=ref64.meta, inv_s=c1["compact"]["inv_s"], kw=kw, cot=cot, host=g_host, graph=g_graph, lin_host=lin_host,
               lin_graph=lin_graph, fwd=_fwd_rel(r_all, dec, ref), radiance="rgb" if with_rgb else ("zero" if model.radiance_net is not None else "none"))
    if with_rgb:
        res["codes"] = dict(host=d_codes_host, graph=d_codes_graph)
    return res


def _lidar_loss_case(name, monkeypatch, dev):
    import test_lidar_loss_gpu as ll
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.loss import LidarLoss
    from neuralsim_b200.renderer import SingleVolumeRenderer
    kind, _ = CASES[name]
    model, ref_cls = _model(kind, dev)
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    n = 4096
    lo, ld = (x.to(dev) for x in C.lidar_rays(1, n))
    ranges = ll._ranges(model, lo, ld, cfg)
    with torch.no_grad():
        solid = SingleVolumeRenderer(cfg).train().render(model, lo, ld)["rendered"]["mask_volume"] > 0.5
    ranges[~solid] = 120.0                                     # beams that do not see the road return nothing within discard_toofar
    lidar = LidarLoss(**ll.LIDAR_CFG)
    cap = _Capture(monkeypatch, model)
    _zero(model)
    ret = SingleVolumeRenderer(cfg).train().render(model, lo, ld, return_buffer=True)
    terms = lidar(None, ret, None, {"ranges": ranges}, it=LIDAR_IT)
    (sum(terms.values()) * n).backward()                       # the loss times n: cotangents of order one (see the module docstring)
    rendered, terms = {k: v.detach().clone() for k, v in ret["rendered"].items()}, {k: v.detach().clone() for k, v in terms.items()}
    g_host = _grads(model)
    mask_kernel = lidar.mask.bool().cpu().numpy()
    c = cap.host()
    n_packs = c["compact"]["pack_infos"].shape[0]
    dec = _decisions(c, np.arange(n_packs))                    # the whole batch: every kept pack
    ref64 = ref_cls.from_model(model)
    inv_s = c["compact"]["inv_s"]
    t0 = time.time()
    vw = step64.kept_weights(ref64, dec, inv_s)
    eps = ll._eps(LIDAR_IT)
    gt = ranges.cpu().numpy()
    lo64 = lidar64.lidar_loss(rendered["depth_volume"].cpu().numpy(), rendered["mask_volume"].cpu().numpy(), gt, dec["t_kept"], vw,
                              dec["kept_pinfo"], dec["ray"], fn_type="l1", w_depth=0.05, w_los=0.1, epsilon=eps, discard_toofar=80.0,
                              median_factor=100.0)
    assert np.array_equal(lo64["mask"], mask_kernel)            # the validity mask, the median discard included, bit for bit
    cot = dict(g_mask=np.zeros(n_packs), g_depth=lo64["g_depth"][dec["ray"]] * n, g_rgb=None, g_nablas=np.zeros((n_packs, 3)), g_vw=lo64["g_vw"] * n)
    # the rays the loss reads (its mask): the others carry zero cotangents and add nothing
    live = np.nonzero(mask_kernel[dec["ray"]])[0]
    assert solid.cpu().numpy()[dec["ray"][live]].all()
    cot = _sub_cot(cot, live, dec)
    dec = step64.select(dec, live) | dict(ray=dec["ray"][live])
    kw = dict(ln_inv_s_factor=model.ctrl_var.ln_inv_s_factor, with_rgb=False)
    ref = step64.step_grads(ref64, dec, inv_s, **cot, **kw)
    t_replay = time.time() - t0
    # the graph step with the loss inside (loss_on_ret=True), on the same rays, ranges and iteration.  The host-sized step's autograd
    # graph goes first: its AccumulateGrad nodes, kept alive, would pin the parameters to the default stream and break the capture
    monkeypatch.undo()
    del ret
    model.zero_grad(set_to_none=True)
    gc.collect()
    fterms = {}

    def loss_fn(ret):
        fterms.update(lidar(None, ret))
        return sum(fterms.values()) * n
    fr = StaticFrame(model, n, loss_fn=loss_fn, loss_on_ret=True, near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True, zero_grads=True)
    lidar.set_step(ranges, LIDAR_IT)
    fr.step(lo, ld)
    assert fr.counts()["overflow"] == 0
    for k, v in rendered.items():
        assert torch.equal(fr.rendered[k], v), k
    for k, v in terms.items():
        assert torch.equal(fterms[k], v), k
    g_graph = _grads(model)
    return dict(n=n, n_sub=N_SUBSET, kept=int(dec["kept"].shape[0]), boundary=int(dec["t1"].shape[0]), t_replay=t_replay, ref=ref, dec=dec,
                ref64=ref64, meta=ref64.meta, inv_s=inv_s, kw=kw, cot=cot, host=g_host, graph=g_graph, fwd=_fwd_rel(rendered, dec, ref),
                radiance="zero" if model.radiance_net is not None else "none", lidar=dict(
                    kept_rays=n_packs, replayed_rays=int(live.shape[0]), masked=int(mask_kernel.sum()), los_rows=int((lo64["g_vw"] != 0).sum()),
                    terms={k: float(v) for k, v in terms.items()}, los64=lo64["los"], depth64=lo64["depth"]))


def _run_case(name, monkeypatch, dev):
    if name not in _CACHE:
        fn = _lidar_loss_case if CASES[name][1] == "lidar-loss" else _weighted_case
        _CACHE[name] = fn(name, monkeypatch, dev)
    return _CACHE[name]


@pytest.mark.parametrize("name", list(CASES))
def test_street_step_gradients_match_float64_replay(cuda, monkeypatch, name):
    r = _run_case(name, monkeypatch, cuda)
    out = dict(case=name, rays=r["n"], replayed=r["dec"]["kept_pinfo"].shape[0], kept_samples=r["kept"], boundary_samples=r["boundary"],
               replay_seconds=round(r["t_replay"], 1), forward_rel_l2=r["fwd"], lidar=r.get("lidar"),
               norms={k: float(np.linalg.norm(r["ref"][k])) for k in KEYS if r["ref"].get(k) is not None})
    fails = [f"forward {k}: rel-L2 {v:.2e} > {FWD_REL:.0e}" for k, v in r["fwd"].items() if not v <= FWD_REL]
    n_sub = r["n_sub"] if "lin_host" in r else N_SUBSET
    for path in ("host", "graph"):
        rep, f = _compare(r[path], r["ref"], r["meta"], n_sub, r["radiance"])
        out[path] = rep
        fails += [f"{path}: {x}" for x in f]
        if "lin_host" in r:
            lin = r[f"lin_{path}"]
            out[f"linearity_{path}"] = lin
            fails += [f"{path} linearity: {k} {v:.2e} > {LIN_REL:.0e}" for k, v in lin.items() if v > LIN_REL]
    if "codes" in r:
        # the appearance-code gradient of every replayed ray; the codes of the other rays carry a zero cotangent and stay exactly zero
        want = step_code_grads(r["ref64"], r["dec"], r["inv_s"], **r["cot"], **r["kw"])
        rows = torch.from_numpy(r["dec"]["ray"])
        for path in ("host", "graph"):
            g = r["codes"][path].cpu()
            rel = float(np.linalg.norm(g[rows].double().numpy() - want) / np.linalg.norm(want))
            others = torch.ones(g.shape[0], dtype=torch.bool)
            others[rows] = False
            out[f"codes_{path}"] = rel
            if not rel <= REL:
                fails.append(f"{path} codes: rel-L2 {rel:.2e} > {REL:.0e}")
            if bool(g[others].any()):
                fails.append(f"{path} codes: nonzero rows of rays outside the subset")
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


def _sub_cot(cot, rays, dec):
    """the cotangents of the rays `rays` (g_vw: of their kept samples)"""
    out = {k: (None if v is None else v[rays]) for k, v in cot.items() if k != "g_vw"}
    if cot.get("g_vw") is not None:
        kpi = dec["kept_pinfo"][rays]
        out["g_vw"] = cot["g_vw"][np.repeat(kpi[:, 0], kpi[:, 1]) + np.arange(int(kpi[:, 1].sum())) - np.repeat(np.cumsum(kpi[:, 1]) - kpi[:, 1], kpi[:, 1])]
    return out


def test_wrong_references_fail(cuda, monkeypatch):
    """the bounds can fail: float64 references with a deliberate, small defect fail the comparison the kernels pass"""
    report = {}

    def judge(tag, r, bad_ref):
        n_sub = r["n_sub"] if "lin_host" in r else N_SUBSET
        for path in ("host", "graph"):
            _, f = _compare(r[path], bad_ref, r["meta"], n_sub, r["radiance"])
            report[f"{tag} / {path}"] = f[:4]
            assert f, (tag, path)
    r = _run_case("camera", monkeypatch, cuda)
    dec, ref, ref64, cot, kw = r["dec"], r["ref"], r["ref64"], r["cot"], r["kw"]
    R = dec["pinfo"].shape[0]
    # (1) one kept sample dropped in every ~1000th ray: replay only those rays both ways (the gradient is a sum over rays)
    bad, rays = _drop_kept(dec, 1000)
    sub = lambda dd: step64.step_grads(ref64, step64.select(dd, rays), r["inv_s"], **_sub_cot(cot, rays, dec), **kw)
    right, wrong = sub(dec), sub(bad)
    judge("dropped kept sample", r, {k: ref[k] - right[k] + wrong[k] for k in KEYS})
    # (2) level DROP_LEVEL's table contribution dropped on the samples of every 10th ray (a tenth of the samples)
    tenth = np.arange(0, R, 10)
    part = step64.step_grads(ref64, step64.select(dec, tenth), r["inv_s"], **_sub_cot(cot, tenth, dec), **kw)
    s = slice(r["meta"].level_offsets[DROP_LEVEL], r["meta"].level_offsets[DROP_LEVEL + 1])
    ref2 = dict(ref, grid=ref["grid"].copy())
    ref2["grid"][s] -= part["grid"][s]
    judge("dropped level contribution", r, ref2)
    # (3) the nablas scale with x and y swapped (25/75 and 25/20): on the cubic cfg2 box this is the same reference
    ref64.fac = ref64.fac[[1, 0, 2]]
    try:
        swapped = step64.step_grads(ref64, dec, r["inv_s"], **cot, **kw)
    finally:
        ref64.fac = ref64.fac[[1, 0, 2]]
    judge("fac x and y swapped", r, swapped)
    # (4) lidar-loss: the line-of-sight g_vw zeroed on every 10th kept ray
    r = _run_case("lidar-loss", monkeypatch, cuda)
    dec, ref, cot = r["dec"], r["ref"], r["cot"]
    tenth = np.arange(0, dec["kept_pinfo"].shape[0], 10)
    only = dict(g_mask=np.zeros(tenth.shape[0]), g_depth=np.zeros(tenth.shape[0]), g_rgb=None, g_nablas=np.zeros((tenth.shape[0], 3)),
                g_vw=_sub_cot(cot, tenth, dec)["g_vw"])
    los = step64.step_grads(r["ref64"], step64.select(dec, tenth), r["inv_s"], **only, **r["kw"])
    judge("line-of-sight g_vw lost on every 10th ray", r, {k: (None if ref.get(k) is None else ref[k] - los[k]) for k in KEYS})
    print(json.dumps(dict(rays_with_a_dropped_sample=len(rays), failures=report)))
