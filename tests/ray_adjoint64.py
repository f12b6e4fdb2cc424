"""Float64 statement of the ray test's adjoint (nsb_gather_rays_backward).  TEST INFRASTRUCTURE.

The one-launch step normalises the caller's rays into the unit box, o' = (o - c) / r and d' = d / r (AABBSpace.normalize_rays), keeps
the rays that pass the box test, o_c = o'[idx] and d_c = d'[idx], and renders with view_dirs = d_c / clamp(|d_c|, 1e-10), the norm held
constant.  Given the loss's gradients g_o, g_d, g_vd to o_c, d_c and view_dirs (per compacted ray), the gradient to the caller's rays is
    d_rays_o[idx] = g_o / r          d_rays_d[idx] = (g_d + g_vd / |d_c|) / r
and 0 for rays that fail the test.  `adjoint32` is the same in the kernel's fp32 order: g_d first holds the colour and the boundary
contributions, the view term is added last, the sum is added onto 0 and divided by r.
"""
import numpy as np


def adjoint(idx, n_rays, radius3, g_o, g_d, g_vd=None, vnorm=None):
    """float64 (d_rays_o, d_rays_d) [n_rays, 3]; g_* [n, 3] per compacted ray j, which is caller row idx[j]"""
    r = np.asarray(radius3, np.float64)
    gd = np.asarray(g_d, np.float64)
    if g_vd is not None:
        gd = gd + np.asarray(g_vd, np.float64) / np.asarray(vnorm, np.float64)[:, None]
    d_o, d_d = np.zeros((n_rays, 3)), np.zeros((n_rays, 3))
    d_o[np.asarray(idx, np.int64)] = np.asarray(g_o, np.float64) / r
    d_d[np.asarray(idx, np.int64)] = gd / r
    return d_o, d_d


def adjoint32(idx, n_rays, radius3, g_o, g_d_colour, g_d_boundary, g_vd=None, vnorm=None):
    """the kernel's fp32 operations in its order: ((0 + colour) + boundary) accumulated, + g_vd / vnorm, onto 0, / r"""
    f = np.float32
    r = np.asarray(radius3, f)
    gd = (f(0) + np.asarray(g_d_colour, f)) + np.asarray(g_d_boundary, f)
    if g_vd is not None:
        gd = gd + np.asarray(g_vd, f) / np.asarray(vnorm, f)[:, None]
    d_o, d_d = np.zeros((n_rays, 3), f), np.zeros((n_rays, 3), f)
    d_o[np.asarray(idx, np.int64)] = (f(0) + np.asarray(g_o, f)) / r
    d_d[np.asarray(idx, np.int64)] = (f(0) + gd) / r
    return d_o, d_d
