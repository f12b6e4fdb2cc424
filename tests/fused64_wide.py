"""The float64 reference of the fused kernels (oracle/fused64.py) in the 48-column layout of LoTD tables of L = 17..24 levels.

oracle/fused64.py computes with 32 h columns (the 16-level layout).  The kernels for 17..24 levels use a 48-column feature tile: h gets
48 - 2L zero columns, W1 zero columns at 2L..47, and the radiance input the internal order [x(3) | SH(16) | n(3) | h(48) | h_appear],
R1 with zero columns where the h columns 2L..47 sit.  Every added term is an exact float64 zero (and rounds to fp16 zero), so the values
are those of the L-level model; the gradients of W1 and R1 are returned at the L-level shapes.  L <= 16 embeds the same way, so a
16-level model and its 48-column embedding give the same values."""
import numpy as np
import torch

from oracle import fused64, lotd as olotd

H_WIDE = 48                     # h columns of the wide layout
H_COLS_WIDE = slice(22, 22 + H_WIDE)


def _np(p):
    return None if p is None else torch.as_tensor(p).detach().float().cpu().numpy()


def ref_col_wide(k, n_appear, nh, hc=H_WIDE):
    """csrc/color_tc.cu ref_col with an h tile of hc columns: internal radiance-input column k ([h(hc, nh used) | x | SH | n | h_appear | 0])
    -> reference column of [x(3) | SH(16) | n(3) | h(nh) | h_appear], or -1"""
    if k < hc:
        return 22 + k if k < nh else -1
    k -= hc
    if k < 22:
        return k
    if k < 22 + n_appear:
        return 22 + nh + (k - 22)
    return -1


class Fused64Wide(fused64.Fused64):
    def __init__(self, table, lotd_cfg, W1, b1, W2, b2, R1=None, rb1=None, R2=None, rb2=None, R3=None, rb3=None, **kw):
        nh = int(olotd.LoDMeta(3, **lotd_cfg).n_encoded_dims)
        assert 2 <= nh <= H_WIDE and nh % 2 == 0, nh
        W1 = _np(W1)
        W1p = np.zeros((W1.shape[0], H_WIDE), dtype=np.float32)
        W1p[:, :nh] = W1
        R1p = None
        if R1 is not None:
            R1 = _np(R1)
            n_appear = R1.shape[1] - 22 - nh
            assert n_appear >= 0, R1.shape
            R1p = np.zeros((R1.shape[0], 22 + H_WIDE + n_appear), dtype=np.float32)
            R1p[:, :22 + nh] = R1[:, :22 + nh]
            R1p[:, 22 + H_WIDE:] = R1[:, 22 + nh:]
        super().__init__(table, lotd_cfg, W1p, b1, W2, b2, R1p, rb1, R2, rb2, R3, rb3, **kw)
        self.nh = nh
        self.n_appear = 0 if R1p is None else R1p.shape[1] - 22 - H_WIDE

    def features(self, xs):
        """h [N, 48], J [N, 48, 3], zero in the columns 2L..47"""
        if self.rounding:
            h, J = super().features(xs)
        else:                                                      # the exact interpolation, as the base class states it for 32 columns
            N = xs.shape[0]
            h, J = np.zeros((N, H_WIDE)), np.zeros((N, H_WIDE, 3))
            for ooff, idx, w, dw in self.levels(xs):
                for f in range(2):
                    v = self.T[idx + f]
                    h[:, ooff + f] = (w * v).sum(0)
                    J[:, ooff + f, :] = np.einsum("gcn,cn->ng", dw, v)
        if h.shape[1] < H_WIDE:
            h = np.concatenate([h, np.zeros((h.shape[0], H_WIDE - h.shape[1]))], 1)
            J = np.concatenate([J, np.zeros((J.shape[0], H_WIDE - J.shape[1], 3))], 1)
        return h, J

    def _unpad(self, out):
        out["W1"] = out["W1"][:, :self.nh]
        if "R1" in out:
            out["R1"] = np.concatenate([out["R1"][:, :22 + self.nh], out["R1"][:, 22 + H_WIDE:]], 1)
        return out

    def sdf_backward(self, x, d_sdf):
        return self._unpad(super().sdf_backward(x, d_sdf))

    def color_backward(self, fwd, g_sdf=None, g_nablas=None, g_rgb=None):
        """Fused64.color_backward in the 48-column layout.  The base class reads the h columns of R1 through its 32-column module constant,
        so the method is restated here term for term with the 48 h columns (H_COLS_WIDE), the only difference."""
        N = fwd["sdf"].shape[0]
        f32 = lambda v, shape: np.zeros(shape) if v is None else np.asarray(v, dtype=self.f32).astype(np.float64)
        g_sdf, g_nab, g_rgb = f32(g_sdf, (N,)), f32(g_nablas, (N, 3)), f32(g_rgb, (N, 3))
        rgb, X, Y1, Y2 = fwd["rgb"], fwd["X"], fwd["Y1"], fwd["Y2"]
        out = {}
        # radiance net
        gy = self.r16(self.r16(g_rgb) * ((1.0 - rgb) * rgb))
        dZ2 = self.r16((Y2 > 0) * (gy @ self.R3))
        dZ1 = self.r16((Y1 > 0) * (dZ2 @ self.R2))
        dh_r = dZ1 @ self.R1[:, H_COLS_WIDE]
        out.update(R3=gy.T @ Y2, rb3=gy.sum(0), R2=dZ2.T @ Y1, rb2=dZ2.sum(0), R1=dZ1.T @ X, rb1=dZ1.sum(0))
        # decoder, first and second order
        h, J, lin, s, a16, u, g16 = fwd["h"], fwd["J"], fwd["lin"], fwd["s"], fwd["a16"], fwd["u"], fwd["g16"]
        w2, dsdf = self.W2[0], g_sdf[:, None]
        gin = g_nab * self.fac * 0.5
        dG = self.r16(np.einsum("nd,nfd->nf", gin, J))
        dd = self.r16(dG @ self.W1.T)
        curv = np.where(lin, 0.0, self.beta * s * (1.0 - s))
        dz = self.r16(dd * w2 * curv + dsdf * w2 * s)
        v = self.r16(dd * s + dsdf * a16)
        dhz = dz @ self.W1
        out.update(W1=dz.T @ h + u.T @ dG, b1=dz.sum(0), W2=v.sum(0)[None], b2=g_sdf.sum(0, keepdims=True))
        out["grid"] = self._scatter(fwd["xs"], row_w=dhz + dh_r, row_dw=g16, gin=gin)
        return self._unpad(out)
