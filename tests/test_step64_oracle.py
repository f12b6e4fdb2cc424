"""CPU: oracle/step64.py, the float64 replay of one NeuS training step on fixed decisions, against torch float64 autograd of the same
fixed-decision forward (boundary SDF -> alpha -> kept samples -> colour / normal query -> compositing -> loss) without rounding.  The
replay composes hand-written adjoints (oracle/fused64.py, oracle/neus64.py); here they must give the exact gradient of the composition,
for every parameter, before the replay judges the kernels (tests/test_step_grad_frame_gpu.py)."""
import numpy as np
import torch

from oracle import fused64, lotd as olotd, neus64, nets as onets, scene as oscene, step64

F32 = np.float32
CFG16 = olotd.gen_ngp_cfg(log2_hashmap_size=14)
EPS = 1e-4


def _case(seed=0, n_rays=24, radius3=None, sdf_scale=1.0, radiance=True):
    """a sphere model (radius 0.5) seen from 3 units, rays through it (none grazes its rim, where the
    mask is ~0 and the normalised depth amplifies float64 round-off); boundary packs of 20-60 sorted depths
    around the surface; the kept samples and the visited samples decided by the fp32 replay of the float64 alphas.
    radius3: the half-size of a cuboid box (the street model's 20 x 75 x 7.5 m): the rays are world rays of unit direction d_w, normalised
    as the ray test does (d = d_w / radius3, depths in metres), the view direction is d_w and the nablas scale is sdf_scale / radius3 per
    axis.  radiance=False: a model without a radiance net (radiance_cfg=False)."""
    P = oscene.make_sphere_params(seed=seed, lotd_cfg=CFG16, sdf_level=1, noise=2e-3)
    rng = np.random.default_rng(seed)
    with torch.no_grad():                         # decoder weights away from the sphere construction's zeros: every weight has a gradient
        for W in (P.dec_W1, P.dec_b1, P.dec_W2):
            W.add_(torch.from_numpy(rng.standard_normal(tuple(W.shape)) * 2e-3).float())
    rad = (P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3, P.rad_b3) if radiance else (None,) * 6
    r3 = np.ones(3) if radius3 is None else np.asarray(radius3, np.float64)
    ref = fused64.Fused64(P.grid, CFG16, P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, *rad, beta=100.0, fac=sdf_scale / r3, rounding=False)
    cam = np.array([3.0, 0.4, 0.8])
    aim = rng.uniform(-0.3, 0.3, (n_rays, 3)) * np.array([0.2, 1.0, 1.0])
    aim[-2:] *= 0.1
    d = aim - cam
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = np.broadcast_to(cam, d.shape).astype(F32)
    d = d.astype(F32)
    lens = rng.integers(20, 61, n_rays)
    # the last two rays' samples lie past the sphere, where the sdf rises: nothing of them is kept
    t1 = np.concatenate([np.sort(rng.uniform(2.2, 3.6, n) if r < n_rays - 2 else rng.uniform(3.7, 4.5, n)) for r, n in enumerate(lens)])
    view = d / np.linalg.norm(d.astype(np.float64), axis=1, keepdims=True)
    if radius3 is not None:
        # the same rays as world rays: d_w = d radius3 / |d radius3| and d = d_w / radius3 = d / |d radius3|, depths t |d radius3| in metres
        dw = d.astype(np.float64) * r3
        sc = np.linalg.norm(dw, axis=1)
        view = dw / sc[:, None]
        d = (d / sc[:, None]).astype(F32)
        t1 = t1 * np.repeat(sc, lens)
    t1 = t1.astype(F32)
    pinfo = np.stack([np.cumsum(lens) - lens, lens], 1)
    inv_s = float(F32(np.exp(10 * float(P.ln_inv_s))))
    ray_b = neus64.pack_of(pinfo, t1.shape[0])
    sdf = ref.sdf(step64.points(o[ray_b], d[ray_b], t1))
    alpha, _ = neus64.neus_alpha(sdf, pinfo, inv_s)
    r = neus64.replay(alpha.astype(F32), pinfo, EPS, 0.0)
    kept = np.nonzero(r["vis"])[0]
    kept_n = r["steps"]
    kpi = np.stack([np.cumsum(kept_n) - kept_n, kept_n], 1)
    t_kept = (t1[kept] + (t1[kept + 1] - t1[kept]) / F32(2)).astype(F32)
    a32 = alpha[kept].astype(F32)
    vis_f = neus64.replay(a32, kpi, EPS, 0.0)["vis"]
    vis_b = neus64.replay(a32, kpi, EPS, 0.0, backward=True)["vis"]
    assert (r["cross"] >= 0).sum() >= 3 and (kept_n == 0).sum() >= 1 and (kept_n > 5).sum() >= 10     # early stops, misses, long packs
    dec = dict(o=o, d=d, view=view.astype(F32), h_appear=rng.standard_normal((n_rays, P.n_appear)).astype(F32) * 0.3, t1=t1, pinfo=pinfo,
               kept=kept, kept_pinfo=kpi, t_kept=t_kept, vis_fwd=vis_f, vis_bwd=vis_b)
    g = dict(g_mask=rng.standard_normal(n_rays), g_depth=rng.standard_normal(n_rays), g_rgb=rng.standard_normal((n_rays, 3)),
             g_nablas=rng.standard_normal((n_rays, 3)))
    # the nablas scale the autograd restatement applies: fp32, as the model forms it from the box (not read from ref)
    ref.case_fac = (F32(sdf_scale) / r3.astype(F32)).astype(np.float64)
    return P, ref, dec, inv_s, g


def _field(ref, T, W, x32, with_color, view=None, ha=None, with_rgb=True):
    """the unrounded model in torch float64 at fp32 points x32: sdf, and with_color nablas (double backward) and, with_rgb, rgb"""
    W1, b1, W2, b2, R1, rb1, R2, rb2, R3, rb3 = W
    xs32 = ref.xs_of(x32)
    x64 = torch.from_numpy(x32.astype(np.float64)).requires_grad_(with_color)
    xs64 = x64 * 0.5 + 0.5
    cols = [torch.zeros(x32.shape[0], dtype=torch.float64)] * 32
    for psl, lvl, loff, foff, ooff in olotd._level_iter(ref.meta, ref.max_level):
        res = np.array(ref.meta.level_res_multidim[lvl], dtype=np.uint32)
        scale = (res - 2).astype(np.float32)
        cell, frac = olotd.pos_fract(xs32, scale)
        fr = torch.from_numpy(frac.astype(np.float64)) + (xs64 - xs64.detach()) * torch.from_numpy(scale.astype(np.float64))
        for c in range(8):
            off = np.array([(c >> k) & 1 for k in range(3)], dtype=np.uint32)
            idx = torch.from_numpy(olotd.grid_index(ref.meta, lvl, cell + off) * 2 + foff + loff)
            w = 1.0
            for k in range(3):
                w = w * (fr[:, k] if (c >> k) & 1 else 1.0 - fr[:, k])
            for f in range(2):
                cols[ooff + f] = cols[ooff + f] + w * T[idx + f]
    h = torch.stack(cols, -1)
    a = torch.nn.functional.softplus(h @ W1.T + b1, beta=ref.beta, threshold=20.0)
    sdf = (a @ W2.T + b2)[:, 0]
    if not with_color:
        return sdf
    nab = torch.autograd.grad(sdf.sum(), x64, create_graph=True)[0] * torch.from_numpy(ref.case_fac)
    if not with_rgb:
        return sdf, nab, None
    X = torch.cat([x64.detach(), onets.sh_encode(torch.from_numpy(view.astype(np.float64)), 4), nab.detach().clamp(-1, 1), h,
                   torch.from_numpy(ha.astype(np.float64))], -1)
    rgb = torch.sigmoid(torch.relu(torch.relu(X @ R1.T + rb1) @ R2.T + rb2) @ R3.T + rb3)
    return sdf, nab, rgb


def _autograd_step(P, ref, dec, inv_s, g, g_vw=None, with_rgb=True):
    T = torch.tensor(ref.T, requires_grad=True)
    W = [torch.tensor(p.half().double().numpy(), requires_grad=True) for p in
         (P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3, P.rad_b3)]
    with_rgb = with_rgb and ref.R1 is not None
    ln = torch.tensor(float(P.ln_inv_s), dtype=torch.float64, requires_grad=True)
    # inv_s = exp(10 ln): the value is the fp32 inv_s the kernels read, and autograd's d inv_s / d ln is 10 times that value
    inv = inv_s + 10 * inv_s * (ln - ln.detach())
    t1, pinfo, kept, kpi = dec["t1"], dec["pinfo"], dec["kept"], dec["kept_pinfo"]
    S, K, R = t1.shape[0], kept.shape[0], pinfo.shape[0]
    ray_b, ray_k = neus64.pack_of(pinfo, S), neus64.pack_of(kpi, K)
    sdf = _field(ref, T, W, step64.points(dec["o"][ray_b], dec["d"][ray_b], t1), False)
    # x = sdf inv_s carries the value of the kernels' fp32 product (a decision point) and the exact derivative
    x = sdf * inv
    x32 = (sdf.detach().numpy().astype(F32) * F32(inv_s)).astype(F32).astype(np.float64)
    x = x + (torch.from_numpy(x32) - x.detach())
    c = torch.sigmoid(x)
    alpha = ((c[kept] - c[kept + 1]) / (c[kept] + 1e-5)).clamp_min(0)
    _, nab, rgb = _field(ref, T, W, step64.points(dec["o"][ray_k], dec["d"][ray_k], dec["t_kept"]), True, dec["view"][ray_k],
                         dec["h_appear"][ray_k], with_rgb=with_rgb)
    ws = []
    for b, n in kpi.tolist():
        Tr = torch.ones((), dtype=torch.float64)
        for j in range(b, b + n):
            assert dec["vis_fwd"][j] and dec["vis_bwd"][j]
            ws.append(alpha[j] * Tr)
            Tr = Tr * (1 - alpha[j])
    w = torch.stack(ws)
    pk = torch.from_numpy(ray_k)
    tk = torch.from_numpy(dec["t_kept"].astype(np.float64))
    M = torch.zeros(R, dtype=torch.float64).index_add(0, pk, w)
    D = torch.zeros(R, dtype=torch.float64).index_add(0, pk, w * tk) / (M + 1e-10)
    N = torch.zeros(R, 3, dtype=torch.float64).index_add(0, pk, w[:, None] * nab)
    t = lambda k: torch.from_numpy(g[k])
    loss = (M * t("g_mask")).sum() + (D * t("g_depth")).sum() + (N * t("g_nablas")).sum()
    out = dict(mask=M, depth=D, normals=N, vw=w)
    if with_rgb:
        out["rgb"] = C = torch.zeros(R, 3, dtype=torch.float64).index_add(0, pk, w[:, None] * rgb)
        loss = loss + (C * t("g_rgb")).sum()
    if g_vw is not None:
        loss = loss + (w * torch.from_numpy(g_vw)).sum()
    grads = torch.autograd.grad(loss, [T, *W, ln], allow_unused=True)
    return dict(zip(step64.GRADS + ("ln_inv_s",), (None if gr is None else gr.numpy() for gr in grads))), out


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def test_unrounded_step_replay_equals_float64_autograd():
    P, ref, dec, inv_s, g = _case()
    got = step64.step_grads(ref, dec, inv_s, **g)
    want, out = _autograd_step(P, ref, dec, inv_s, g)
    for k, v in out.items():
        assert _rel(got["out"][k], v.detach().numpy()) < 1e-12, k
    for k, v in want.items():
        assert np.abs(v).max() > 0, k
        assert _rel(got[k], v) < 1e-10, (k, _rel(got[k], v))
    # an entry the replay leaves exactly zero is one no queried sample reaches (the GPU test relies on this)
    assert not (want["grid"] != 0)[got["grid"] == 0].any()


def test_replay_is_linear_in_the_rays():
    """the gradient of a sum over rays is the sum of the rays' gradients: a replay of two disjoint ray sets adds up to the replay of both
    (this is what lets the GPU test replay a subset of a frame)"""
    P, ref, dec, inv_s, g = _case(seed=1, n_rays=16)
    full = step64.step_grads(ref, dec, inv_s, **g)
    halves = []
    for part in (np.arange(16) % 2 == 0, np.arange(16) % 2 == 1):
        gp = {k: np.where(part.reshape((-1,) + (1,) * (v.ndim - 1)), v, 0.0) for k, v in g.items()}
        halves.append(step64.step_grads(ref, dec, inv_s, **gp))
    for k in step64.GRADS + ("ln_inv_s",):
        assert _rel(halves[0][k] + halves[1][k], full[k]) < 1e-12, k
    # and so does a replay of the two ray sets' own decisions (step64.select)
    parts = [np.nonzero(np.arange(16) % 2 == m)[0] for m in (0, 1)]
    sub = [step64.step_grads(ref, step64.select(dec, p), inv_s, **{k: v[p] for k, v in g.items()}) for p in parts]
    for k in step64.GRADS + ("ln_inv_s",):
        assert _rel(sub[0][k] + sub[1][k], full[k]) < 1e-12, k
    for k in ("mask", "depth", "rgb", "normals"):
        assert np.array_equal(np.concatenate([sub[0]["out"][k], sub[1]["out"][k]])[np.argsort(np.concatenate(parts))], full["out"][k]), k


def _check_against_autograd(got, want, out, zero=()):
    """every gradient of the replay equals autograd's; the keys in `zero` are exact zeros in the replay (None where autograd has none)"""
    for k, v in out.items():
        assert _rel(got["out"][k], v.detach().numpy()) < 1e-12, k
    for k, v in want.items():
        if k in zero:
            assert got[k] is None if v is None else (v == 0).all() and (got[k] == 0).all(), k
            continue
        assert np.abs(v).max() > 0, k
        assert _rel(got[k], v) < 1e-10, (k, _rel(got[k], v))
    assert not (want["grid"] != 0)[got["grid"] == 0].any()


def test_weight_cotangent_equals_float64_autograd():
    """g_vw: a cotangent of every kept sample's weight (the LiDAR loss's line of sight) enters the compositing adjoint"""
    P, ref, dec, inv_s, g = _case(seed=2)
    g_vw = np.random.default_rng(7).standard_normal(dec["kept"].shape[0])
    got = step64.step_grads(ref, dec, inv_s, **g, g_vw=g_vw)
    want, out = _autograd_step(P, ref, dec, inv_s, g, g_vw=g_vw)
    _check_against_autograd(got, want, out)
    assert np.array_equal(step64.kept_weights(ref, dec, inv_s), got["out"]["vw"])       # the weights a loss on them reads
    # with only g_vw the replay is the gradient of sum g_vw w, and it is not zero
    only = step64.step_grads(ref, dec, inv_s, **{k: np.zeros_like(v) for k, v in g.items()}, g_vw=g_vw)
    plain = step64.step_grads(ref, dec, inv_s, **g)
    for k in step64.GRADS + ("ln_inv_s",):
        assert _rel(plain[k] + only[k], got[k]) < 1e-12, k
    assert np.abs(only["grid"]).max() > 0 and np.abs(only["ln_inv_s"]).max() > 0


def test_geometry_only_query_equals_float64_autograd():
    """with_rgb=False (LiDAR rays on a colour model): sdf and nablas only, every radiance-net gradient exactly zero"""
    P, ref, dec, inv_s, g = _case(seed=3)
    g_vw = np.random.default_rng(8).standard_normal(dec["kept"].shape[0])
    got = step64.step_grads(ref, dec, inv_s, **g, g_vw=g_vw, with_rgb=False)
    want, out = _autograd_step(P, ref, dec, inv_s, g, g_vw=g_vw, with_rgb=False)
    rad = ("R1", "rb1", "R2", "rb2", "R3", "rb3")
    assert all(want[k] is None for k in rad) and got["out"]["rgb"] is None
    for k in rad:
        assert got[k].shape == getattr(ref, k).shape and not got[k].any(), k
    _check_against_autograd(got, {k: v for k, v in want.items() if k not in rad}, out)
    # the geometry gradients do not depend on g_rgb, nor on the view directions and codes
    dec2 = dict(dec, view=-dec["view"], h_appear=dec["h_appear"] + 1)
    other = step64.step_grads(ref, dec2, inv_s, **dict(g, g_rgb=g["g_rgb"] * 3), g_vw=g_vw, with_rgb=False)
    for k in ("grid", "W1", "b1", "W2", "b2", "ln_inv_s"):
        assert np.array_equal(other[k], got[k]), k


def test_model_without_radiance_net_equals_float64_autograd():
    """a reference built without a radiance net (radiance_cfg=False): the radiance-net gradients are None"""
    P, ref, dec, inv_s, g = _case(seed=4, radiance=False)
    got = step64.step_grads(ref, dec, inv_s, **g, with_rgb=False)
    want, out = _autograd_step(P, ref, dec, inv_s, g, with_rgb=False)
    rad = ("R1", "rb1", "R2", "rb2", "R3", "rb3")
    assert all(got[k] is None for k in rad)
    _check_against_autograd(got, {k: v for k, v in want.items() if k not in rad}, out)


def test_cuboid_box_equals_float64_autograd():
    """the street model's box: rays normalised per axis (d = d_w / radius3) and the nablas scaled by sdf_scale / radius3 per axis
    (25/20, 25/75, 25/7.5), with rgb and without; autograd takes its scale from the box, the replay from the reference's fac"""
    r3 = (20.0, 75.0, 7.5)
    for with_rgb in (True, False):
        P, ref, dec, inv_s, g = _case(seed=5, radius3=r3, sdf_scale=25.0)
        assert np.allclose(ref.fac, [1.25, 1 / 3, 25 / 7.5], rtol=1e-7)
        got = step64.step_grads(ref, dec, inv_s, **g, with_rgb=with_rgb)
        want, out = _autograd_step(P, ref, dec, inv_s, g, with_rgb=with_rgb)
        rad = () if with_rgb else ("R1", "rb1", "R2", "rb2", "R3", "rb3")
        _check_against_autograd(got, {k: v for k, v in want.items() if k not in rad}, out)
        # a reference with x and y of the nablas scale swapped differs in the normals and in the gradients
        bad = fused64.Fused64(P.grid, CFG16, P.dec_W1, P.dec_b1, P.dec_W2, P.dec_b2, P.rad_W1, P.rad_b1, P.rad_W2, P.rad_b2, P.rad_W3,
                              P.rad_b3, beta=100.0, fac=ref.fac[[1, 0, 2]], rounding=False)
        wrong = step64.step_grads(bad, dec, inv_s, **g, with_rgb=with_rgb)
        assert _rel(wrong["out"]["normals"], out["normals"].detach().numpy()) > 1e-2
        assert _rel(wrong["grid"], want["grid"]) > 1e-3 and _rel(wrong["W1"], want["W1"]) > 1e-3


def test_street_models_build_their_float64_references():
    """Fused64 (16 levels), tests/fused64_levels.Fused64Levels (12 levels, no radiance net) and tests/fused64_wide.Fused64Wide (17 levels)
    from bench_cfg3's street model: the per-axis nablas scale, the layouts and the table"""
    import bench_cfg3 as C
    import torch
    from fused64_levels import Fused64Levels
    from fused64_wide import Fused64Wide
    from neuralsim_b200.fields import LoTDNeuSModel
    want_fac = 25.0 / np.array([20.0, 75.0, 7.5])
    # the small-hashmap street models of the GPU tests (tests/test_cfg3_gpu.py, test_partial_levels_gpu.py, test_wide_levels_gpu.py)
    m16 = C.build_model("cpu", max_num_levels=16, log2_hashmap_size=16, target_num_params=18 * 2 ** 17)
    m17 = C.build_model("cpu", max_num_levels=17, log2_hashmap_size=16, target_num_params=19 * 2 ** 17)
    geo = LoTDNeuSModel(surface_cfg=dict(aabb=C.AABB, sdf_scale=C.SDF_SCALE, encoding_cfg=dict(
        lotd_use_cuboid=True, lotd_auto_compute_cfg=dict(type="ngp", target_num_params=14 * 2 ** 17, min_res=16, n_feats=2, log2_hashmap_size=16,
                                                         max_num_levels=12))), radiance_cfg=False, device="cpu")
    for cls, m, levels, n_appear in ((fused64.Fused64, m16, 16, 4), (Fused64Levels, geo, 12, 0), (Fused64Wide, m17, 17, 4)):
        ref = cls.from_model(m)
        assert ref.meta.n_levels == levels and ref.n_appear == n_appear, cls
        np.testing.assert_array_equal(ref.fac, np.asarray(m._nablas_fac(), F32).astype(np.float64))      # the kernels' fac
        np.testing.assert_allclose(ref.fac, want_fac, rtol=1e-6)
        assert np.array_equal(ref.table16, m.implicit_surface.encoding.flattened_params.detach().half().numpy())
        assert (ref.R1 is None) == (m.radiance_net is None)
        x = np.random.default_rng(0).uniform(-0.9, 0.9, (64, 3)).astype(F32)
        fwd = ref.color_forward(x, None, with_rgb=False)
        assert fwd["rgb"] is None and fwd["nablas"].shape == (64, 3)
        gb = ref.color_backward(fwd, g_nablas=np.ones((64, 3)))
        assert gb["W1"].shape == tuple(m.implicit_surface.decoder.layers[0].weight.shape)
        if m.radiance_net is not None:
            assert all(not gb[k].any() for k in ("R1", "rb1", "R2", "rb2", "R3", "rb3"))
            assert gb["R1"].shape == tuple(m.radiance_net.blocks.layers[0].weight.shape)
        else:
            assert "R1" not in gb
    with torch.no_grad():                            # the plane: the sdf of a point 1 m above the road is 1 / sdf_scale
        x = np.array([[0.0, 0.0, (C.ROAD_Z + 1.0) / 7.5]], F32)
        assert abs(fused64.Fused64.from_model(m16, rounding=False).sdf(x)[0] - 1.0 / 25.0) < 2e-3
