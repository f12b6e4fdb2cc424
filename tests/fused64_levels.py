"""The float64 reference of the fused kernels (oracle/fused64.py, written for the 16 x 2 layout) for LoTD tables of L = 1..16 levels.

An L-level model is embedded exactly in the 16-level layout the reference computes with: h gets 32 - 2L zero columns, W1 zero columns
at 2L..31, and R1 zero columns where the h columns 2L..31 sit in the reference's radiance input [x(3) | SH(16) | n(3) | h(32) | h_appear].
Every added term is an exact float64 zero (and rounds to fp16 zero), so the values are those of the L-level model; the gradients of W1
and R1 are returned at the L-level shapes.  This is the layout the kernels use (zero feature columns 2L..31 in their tiles)."""
import numpy as np
import torch

from oracle import fused64, lotd as olotd


def h_cols(nh):
    """the columns of h in the L-level radiance input [x(3) | SH(16) | n(3) | h(nh = 2L) | h_appear]"""
    return slice(22, 22 + nh)


def _np(p):
    return None if p is None else torch.as_tensor(p).detach().float().cpu().numpy()


class Fused64Levels(fused64.Fused64):
    def __init__(self, table, lotd_cfg, W1, b1, W2, b2, R1=None, rb1=None, R2=None, rb2=None, R3=None, rb3=None, **kw):
        nh = int(olotd.LoDMeta(3, **lotd_cfg).n_encoded_dims)
        assert 2 <= nh <= 32 and nh % 2 == 0, nh
        W1 = _np(W1)
        W1p = np.zeros((W1.shape[0], 32), dtype=np.float32)
        W1p[:, :nh] = W1
        R1p = None
        if R1 is not None:
            R1 = _np(R1)
            n_appear = R1.shape[1] - 22 - nh
            assert n_appear >= 0, R1.shape
            R1p = np.zeros((R1.shape[0], 54 + n_appear), dtype=np.float32)
            R1p[:, :22 + nh] = R1[:, :22 + nh]
            R1p[:, 54:] = R1[:, 22 + nh:]
        super().__init__(table, lotd_cfg, W1p, b1, W2, b2, R1p, rb1, R2, rb2, R3, rb3, **kw)
        self.nh = nh

    def features(self, xs):
        """h [N, 32], J [N, 32, 3], zero in the columns 2L..31"""
        h, J = super().features(xs)
        if h.shape[1] < 32:
            h = np.concatenate([h, np.zeros((h.shape[0], 32 - h.shape[1]))], 1)
            J = np.concatenate([J, np.zeros((J.shape[0], 32 - J.shape[1], 3))], 1)
        return h, J

    def _unpad(self, out):
        out["W1"] = out["W1"][:, :self.nh]
        if "R1" in out:
            out["R1"] = np.concatenate([out["R1"][:, :22 + self.nh], out["R1"][:, 54:]], 1)
        return out

    def sdf_backward(self, x, d_sdf):
        return self._unpad(super().sdf_backward(x, d_sdf))

    def color_backward(self, fwd, g_sdf=None, g_nablas=None, g_rgb=None):
        return self._unpad(super().color_backward(fwd, g_sdf, g_nablas, g_rgb))
