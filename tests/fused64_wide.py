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
    h_cols = H_COLS_WIDE

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
        return self._unpad(super().color_backward(fwd, g_sdf, g_nablas, g_rgb))
