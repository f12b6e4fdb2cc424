"""Float64 ray gradient on top of oracle/fused64.py.  TEST INFRASTRUCTURE.

The reference differentiates a sample x = o + d t of ray r with t a constant, view_dirs = d / |d| with a constant norm, and the encoding's
input gradient first order (dy_dx is not differentiated).  With Fused64's rounding points that gives, per sample,
    g_x = 0.5 J^T h_hat + dZ1 . R1[:, 0:3]          g_v = (dSH4/dv)^T (dZ1 . R1[:, 3:19])
with h_hat = dH = r16(d w2 s) . W1 for the SDF query (k_sdf_bwd_tc) and h_hat = dz . W1 + dZ1 . R1[:, h] for the colour query
(k_color_sdf_bwd: its dz has the softplus'' term of the nablas cotangent; h = ref.h_cols, 32 or 48 columns), and per ray  dL/do = sum g_x, dL/dd = sum t g_x, dL/dv = sum g_v.
"""
import numpy as np
import torch

from appear64 import ray_sum
from oracle import nets as onets


def sh_vjp(v, dsh):
    """(dSH4/dv)^T dsh per row, float64: v [N, 3], dsh [N, 16] -> [N, 3]"""
    vt = torch.tensor(np.asarray(v, np.float64), requires_grad=True)
    sh = onets.sh_encode(vt, 4)
    return torch.autograd.grad((sh * torch.from_numpy(np.asarray(dsh, np.float64))).sum(), vt)[0].numpy()


def _radiance_dZ1(ref, fwd, g_rgb):
    g = np.asarray(g_rgb, dtype=ref.f32).astype(np.float64)
    rgb, Y1, Y2 = fwd["rgb"], fwd["Y1"], fwd["Y2"]
    gy = ref.r16(ref.r16(g) * ((1.0 - rgb) * rgb))
    dZ2 = ref.r16((Y2 > 0) * (gy @ ref.R3))
    return ref.r16((Y1 > 0) * (dZ2 @ ref.R2))


def color_rows(ref, fwd, view_dirs, g_sdf=None, g_nablas=None, g_rgb=None):
    """per-sample (g_x [N, 3], g_v [N, 3]) of sum(g_sdf sdf + g_nablas nablas + g_rgb rgb) through color_forward `fwd` at the per-sample
    view directions view_dirs [N, 3]; g_rgb None: the geometry-only op (g_v = 0)"""
    N = fwd["sdf"].shape[0]
    f = lambda v, shape: np.zeros(shape) if v is None else np.asarray(v, dtype=ref.f32).astype(np.float64)
    g_sdf, g_nab = f(g_sdf, (N,)), f(g_nablas, (N, 3))
    J, lin, s, a16 = fwd["J"], fwd["lin"], fwd["s"], fwd["a16"]
    w2, dsdf = ref.W2[0], g_sdf[:, None]
    gin = g_nab * ref.fac * 0.5
    dG = ref.r16(np.einsum("nd,nfd->nf", gin, J))
    dd = ref.r16(dG @ ref.W1.T)
    curv = np.where(lin, 0.0, ref.beta * s * (1.0 - s))
    dz = ref.r16(dd * w2 * curv + dsdf * w2 * s)
    h_hat = dz @ ref.W1
    g_x, g_v = np.zeros((N, 3)), np.zeros((N, 3))
    if g_rgb is not None:
        dZ1 = _radiance_dZ1(ref, fwd, g_rgb)
        h_hat = h_hat + dZ1 @ ref.R1[:, ref.h_cols]
        g_x = dZ1 @ ref.R1[:, 0:3]
        g_v = sh_vjp(view_dirs, dZ1 @ ref.R1[:, 3:19])
    return g_x + 0.5 * np.einsum("nf,nfd->nd", h_hat, J), g_v


def sdf_rows(ref, x, d_sdf):
    """per-sample g_x [N, 3] of sum(d_sdf sdf) (k_sdf_bwd_tc's dH through the first-order input gradient)"""
    h, J = ref.features(ref.xs_of(x))
    z, lin, s, a16, sdf = ref._decoder(h)
    d = np.asarray(d_sdf, dtype=ref.f32).astype(np.float64)[:, None]
    dH = ref.r16(d * ref.W2[0] * s) @ ref.W1
    return 0.5 * np.einsum("nf,nfd->nd", dH, J)


def ray_grads(g_x, t, ridx, n_rays, g_v=None):
    """per-ray (dL/do, dL/dd, dL/dv | None) [n_rays, 3] from per-sample rows; rays without a sample: 0"""
    t = np.asarray(t, np.float64)[:, None]
    return (ray_sum(g_x, ridx, n_rays), ray_sum(t * g_x, ridx, n_rays), None if g_v is None else ray_sum(g_v, ridx, n_rays))
