"""Float64 replay of one NeuS training step on fixed decisions.  TEST INFRASTRUCTURE.

The step of the fused query (graphics/neus.py: _query_fused) with its volume integration: boundary SDF -> alpha -> compression ->
colour / normal query of the kept samples -> compositing -> per-ray loss terms, and the backward pass of all of it to every parameter.
Every decision is taken from the kernels' own forward and held fixed:
  boundary  the samples of each ray: depth t1 (fp32), their packs; a sample's point is fl32(fma(d, t1, o)) of its ray, as the
            ray-parameterised kernels form it
  kept      the boundary samples the compression kept (their alphas are the compositing's inputs), their packs, and their depths
            t_kept (fp32, the interval mid points the kernels computed)
  vis_fwd / vis_bwd   the samples the compositing forward / backward visits (early stop and the alpha threshold)
Along them every value is float64, composed from oracle/fused64.py (the SDF and colour queries, rounding to fp16 where the kernels
round) and oracle/neus64.py (alpha, compositing and their adjoints).  A kept alpha_k reads sdf_k and sdf_{k+1} (neus64.neus_alpha),
so only those boundary samples are queried.  The gradient of a sum over rays is the sum of the rays' gradients: replaying a subset of
the rays of a step whose loss weighs only that subset gives the exact expected gradient of the whole step.
tests/test_step64_oracle.py checks the replay without rounding against torch float64 autograd of the same fixed-decision forward.
"""
from __future__ import annotations

import numpy as np

from . import neus64

F32 = np.float32
GRADS = ("grid", "W1", "b1", "W2", "b2", "R1", "rb1", "R2", "rb2", "R3", "rb3")


def points(o, d, t):
    """x = fl32(fma(d, t, o)): o, d [n, 3] fp32, t [n] fp32 -> [n, 3] fp32 (d t is exact in float64)"""
    o, d = np.asarray(o, F32).astype(np.float64), np.asarray(d, F32).astype(np.float64)
    return (d * np.asarray(t, F32).astype(np.float64)[:, None] + o).astype(F32)


def select(dec, rays):
    """the decisions of the rays `rays` (ascending local ray indices) of `dec`, re-packed"""
    rays = np.asarray(rays, np.int64)
    out = {k: np.asarray(dec[k])[rays] for k in ("o", "d", "view", "h_appear") if dec.get(k) is not None}
    for pk, per in (("pinfo", ("t1",)), ("kept_pinfo", ("t_kept", "vis_fwd", "vis_bwd", "kept"))):
        pi = np.asarray(dec[pk], np.int64).reshape(-1, 2)[rays]
        idx = np.repeat(pi[:, 0] - np.cumsum(pi[:, 1]) + pi[:, 1], pi[:, 1]) + np.arange(int(pi[:, 1].sum()))
        out[pk] = np.stack([np.cumsum(pi[:, 1]) - pi[:, 1], pi[:, 1]], 1)
        for k in per:
            out[k] = np.asarray(dec[k])[idx]
    # kept indices point into the new t1
    old_b = np.asarray(dec["pinfo"], np.int64).reshape(-1, 2)[rays, 0]
    kn = out["kept_pinfo"][:, 1]
    out["kept"] = out["kept"] - np.repeat(old_b - out["pinfo"][:, 0], kn)
    return out


def _boundary(ref, dec, inv32):
    """the boundary SDF where the kept alphas read it, and the kept alphas"""
    o, d = (np.asarray(dec[k], F32) for k in ("o", "d"))
    t1, pinfo = np.asarray(dec["t1"], F32), np.asarray(dec["pinfo"], np.int64).reshape(-1, 2)
    kept, kpi, t_kept = np.asarray(dec["kept"], np.int64), np.asarray(dec["kept_pinfo"], np.int64).reshape(-1, 2), np.asarray(dec["t_kept"], F32)
    S, K = t1.shape[0], kept.shape[0]
    ray_b, ray_k = neus64.pack_of(pinfo, S), neus64.pack_of(kpi, K)
    assert (ray_b >= 0).all() and (ray_k >= 0).all() and (ray_b[kept] == ray_k).all(), "kept samples must lie in their ray's boundary pack"
    # boundary SDF where the kept alphas read it (the last sample of a pack has alpha 0 and is never kept)
    assert (kept + 1 < S).all() and (ray_b[np.minimum(kept + 1, S - 1)] == ray_b[kept]).all()
    need = np.zeros(S, bool)
    need[kept] = True
    need[kept + 1] = True
    nb = np.nonzero(need)[0]
    sdf = np.zeros(S)
    sdf[nb] = ref.sdf(points(o[ray_b[nb]], d[ray_b[nb]], t1[nb]))
    alpha, _ = neus64.neus_alpha(sdf, pinfo, inv32)
    return o, d, t1, pinfo, kept, kpi, t_kept, S, ray_b, ray_k, need, sdf, alpha[kept]


def kept_weights(ref, dec, inv_s):
    """the float64 weights w = alpha T [K] of the kept samples of `dec` (step_grads' forward, without the colour query): what a loss
    on the weights reads, e.g. the LiDAR loss's line of sight"""
    b = _boundary(ref, dec, float(F32(inv_s)))
    kpi, a = b[5], b[-1]
    return neus64.transmittance(a, np.asarray(dec["vis_fwd"], bool), kpi)[1]


def step_grads(ref, dec, inv_s, g_mask, g_depth, g_rgb, g_nablas, *, g_vw=None, with_rgb=True, ln_inv_s_factor=10.0):
    """ref: oracle.fused64.Fused64 of the model.  dec: the decisions of R rays, a dict of
      o, d, view [R, 3] fp32   ray origin, direction (the ray test's: normalised by the box's half-size per axis) and view
                               direction (only with rgb)
      h_appear [R, n_appear]   (optional; zeros)
      t1 [S] fp32, pinfo [R, 2]                       boundary samples, ray r's pack
      kept [K] int64 (into t1, ascending), kept_pinfo [R, 2], t_kept [K] fp32
      vis_fwd, vis_bwd [K] bool
    inv_s: the fp32 inv_s of the alphas (= exp(ln_inv_s_factor ln_inv_s)).  g_*: cotangents of the per-ray mask, depth [R] and rgb,
    normals [R, 3] (training mode: the normals are the composited raw nablas; depth normalised by the mask).  g_vw [K] (optional): a
    cotangent of every kept sample's weight w = alpha T (the LiDAR loss's line of sight).  with_rgb=False: the rays' geometry-only
    query (LiDAR rays, k_color_fwd<false>): sdf and nablas, no rgb (g_rgb is ignored); the radiance net's gradients are exact zeros,
    None for a model without one.
    -> dict of float64 gradients GRADS + inv_s, ln_inv_s, and `out`: the float64 mask, depth, rgb (None without rgb), normals per ray
    and the kept samples' weights vw."""
    inv32 = float(F32(inv_s))
    view = np.asarray(dec["view"], F32) if with_rgb else None
    o, d, t1, pinfo, kept, kpi, t_kept, S, ray_b, ray_k, need, sdf, a = _boundary(ref, dec, inv32)
    # colour / normal query of the kept samples
    ha = dec.get("h_appear")
    ha = np.zeros((o.shape[0], ref.n_appear), F32) if ha is None else np.asarray(ha, F32)
    fwd = ref.color_forward(points(o[ray_k], d[ray_k], t_kept), view[ray_k] if with_rgb else None, ha[ray_k] if ref.n_appear and with_rgb else None,
                            with_rgb=with_rgb)
    g_rgb = g_rgb if fwd["rgb"] is not None else None
    # compositing and its adjoint
    _, w = neus64.transmittance(a, np.asarray(dec["vis_fwd"], bool), kpi)
    out = neus64.composite_forward(w, t_kept, kpi, rgb=fwd["rgb"], nablas=fwd["nablas"])
    vis_b = np.asarray(dec["vis_bwd"], bool)
    Tb, _ = neus64.transmittance(a, vis_b, kpi)
    cb = neus64.composite_backward(a, t_kept, kpi, w, Tb, vis_b, out["mask"], out["depth"], rgb=fwd["rgb"], nablas=fwd["nablas"],
                                   g_mask=g_mask, g_depth=g_depth, g_rgb=g_rgb, g_nablas=g_nablas, g_vw=g_vw)
    gc = ref.color_backward(fwd, g_nablas=cb["d_nablas"], g_rgb=cb.get("d_rgb"))
    # alpha -> boundary SDF -> table and decoder
    d_alpha = np.zeros(S)
    d_alpha[kept] = cb["d_alpha"]
    ab = neus64.alpha_backward(sdf, pinfo, inv32, d_alpha)
    nz = np.nonzero(ab["d_sdf"])[0]
    assert need[nz].all()
    gs = ref.sdf_backward(points(o[ray_b[nz]], d[ray_b[nz]], t1[nz]), ab["d_sdf"][nz])
    grads = {k: gc[k] + gs[k] if k in gs else gc.get(k) for k in GRADS}
    grads["inv_s"] = ab["d_inv_s"]
    grads["ln_inv_s"] = np.array([ab["d_inv_s"] * inv32 * ln_inv_s_factor])
    grads["out"] = dict(mask=out["mask"], depth=out["depth"], rgb=out.get("rgb"), normals=out["nablas"], vw=w)
    return grads
