"""Float64 appearance-code gradient on top of oracle/fused64.py and oracle/step64.py.  TEST INFRASTRUCTURE.

The codes are the last n_appear columns of the radiance input X = [x | SH4(v) | n | h | h_appear], so with the radiance backward's
rounding points of Fused64 (gy = r16(r16(g_rgb) (1-rgb) rgb);  dZ2 = r16([Y2>0] gy R3);  dZ1 = r16([Y1>0] dZ2 R2)) the gradient of a
point's code is  dZ1 . R1[:, h_cols.stop:]  (what k_color_rad_bwd<true> computes: R1[:, 54:] in the 16-level layout of Fused64, R1[:, 70:]
in the 48-column layout of tests/fused64_wide.py), and a ray's is the sum over its points (k_appear_ray_sum).
"""
import numpy as np

from oracle import neus64, step64


def code_grad(ref, fwd, g_rgb):
    """ref: oracle.fused64.Fused64 (or a subclass with its own h_cols) with n_appear >= 1; fwd: its color_forward; g_rgb [N, 3]
    -> d loss / d h_appear [N, n_appear]"""
    assert ref.n_appear >= 1
    g = np.asarray(g_rgb, dtype=ref.f32).astype(np.float64)
    rgb, Y1, Y2 = fwd["rgb"], fwd["Y1"], fwd["Y2"]
    gy = ref.r16(ref.r16(g) * ((1.0 - rgb) * rgb))
    dZ2 = ref.r16((Y2 > 0) * (gy @ ref.R3))
    dZ1 = ref.r16((Y1 > 0) * (dZ2 @ ref.R2))
    return dZ1 @ ref.R1[:, ref.h_cols.stop:]


def ray_sum(rows, ray, n_rays):
    """per-ray sums of per-sample rows [K, C] of the samples' rays ray [K] -> [n_rays, C] float64 (rays without a sample: 0)"""
    out = np.zeros((n_rays, np.asarray(rows).shape[1]))
    np.add.at(out, np.asarray(ray, np.int64), np.asarray(rows, np.float64))
    return out


def step_code_grads(ref, dec, inv_s, *, alter=None, **kw):
    """the code gradient [R, n_appear] of each ray of oracle.step64.step_grads(ref, dec, inv_s, **kw): the colour query's forward and
    rgb cotangent are read off step_grads' own call of ref.color_backward.  alter (optional): fwd -> fwd, applied before code_grad
    (a deliberately wrong reference)."""
    seen = {}
    orig = ref.color_backward

    def record(fwd, *a, **k):
        seen.update(fwd=fwd, g_rgb=k["g_rgb"])
        return orig(fwd, *a, **k)
    ref.color_backward = record
    try:
        step64.step_grads(ref, dec, inv_s, **kw)
    finally:
        del ref.color_backward
    fwd = seen["fwd"] if alter is None else alter(seen["fwd"])
    kpi = np.asarray(dec["kept_pinfo"], np.int64).reshape(-1, 2)
    ray_k = neus64.pack_of(kpi, int(kpi[:, 1].sum()))
    return ray_sum(code_grad(ref, fwd, seen["g_rgb"]), ray_k, kpi.shape[0])
