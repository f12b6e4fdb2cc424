"""Float64 restatement of the numerics contract of the fused tensor-core kernels.  TEST INFRASTRUCTURE.

Covers k_fused_sdf_tc / k_sdf_bwd_tc (neuralsim_b200/csrc/fused_tc.cu) and k_color_fwd / k_color_rad_bwd / k_color_sdf_bwd
(csrc/color_tc.cu).  Every sum is exact to float64; a value is rounded to fp16 exactly where the kernels round it and nowhere
else.  What then separates a kernel from this reference is only its fp32 accumulation order, the SFU softplus of
k_fused_sdf_tc and the rare fp16 value that lands on the other side of a rounding boundary because of them.  This is tighter
than oracle/nets.py, which restates the reference project's autocast graph and rounds every cotangent to fp16.

Rounding points (r16 = round to fp16; names as in the kernels' header comments):
  h        the fp16 LoTD gather of oracle/lotd.py:lod_fwd (bit-exact), levels above max_level contribute 0;
           xs = clamp(fma(x, .5, .5), 1e-6, 1-1e-6) in fp32; J = dh/dxs from the same lod_fwd (fp32)
  sdf      z = r16(h W1^T + b1);  a16 = r16(softplus_beta(z)) (ATen threshold: beta z > 20 -> z);  sdf = r16(a16 . w2 + b2)
  colour   u = r16(w2 * s), s = sigmoid(beta z) (1 above the threshold);  g = U W1;  nablas = 0.5 fac sum_levels J^T r16(g)
           X = r16([x | SH4(v) | clamp(nablas, +-1) | h | h_appear]);  Y1 = relu(r16(X R1^T + rb1));  Y2 = relu(r16(Y1 R2^T + rb2))
           rgb = r16(sigmoid(r16(Y2 R3^T + rb3)))
  radiance backward   gy = r16(r16(g_rgb) (1-rgb) rgb);  dZ2 = r16([Y2>0] gy R3);  dZ1 = r16([Y1>0] dZ2 R2);  dh_r = dZ1 R1[:, h]
  sdf / nablas backward   gin = g_nab fac 0.5;  dG = r16(J gin);  d = r16(dG W1^T);  dz = r16(d w2 beta s(1-s) [beta z <= 20] + dsdf w2 s)
           v = r16(d s + dsdf a16);  dW1 = dz^T H + u^T dG;  db1 = sum dz;  dW2 = sum v;  db2 = sum dsdf
           table, per corner: r16(g) wsum(gin) + (dz W1 + dh_r) w
  sdf backward (k_sdf_bwd_tc)   dz = r16(d w2 s);  da = r16(d a16);  dW1 = dz^T H;  db1 = sum dz;  dW2 = sum da;  table: (dz W1) w

With rounding=False every r16 is the identity, cotangents are taken in float64 instead of fp32, and h / J are the exact trilinear
interpolation of the (fp16-valued) table and its derivative, so the hand-written backward passes below are the exact gradients of
the unrounded model (tests/test_fused64_oracle.py checks them against torch double-backward).
"""
from __future__ import annotations

import numpy as np
import torch

from . import lotd as olotd
from . import nets as onets

H_COLS = slice(22, 54)          # columns of h in the radiance input [x(3) | SH(16) | n(3) | h(32) | h_appear]


def _sigmoid(v):
    return 0.5 * (1.0 + np.tanh(0.5 * v))


class Fused64:
    """Weights are taken as their fp16 images (what the kernels read), held in float64.

    table: fp32 master or fp16 image of the LoTD parameters [P];  lotd_cfg: the LoTD configuration (dict of LoDMeta);
    W1 [width, 32], b1 [width], W2 [1, width], b2 [1];  R1 [rw, 54 + n_appear], rb1, R2 [rw, rw], rb2, R3 [3, rw], rb3 (optional);
    beta: softplus beta of the decoder;  fac [3]: sdf_scale / radius3d_original (the nablas scale, fp32 in the kernels);
    max_level: highest LoTD level that contributes (None: all).  h_cols: the columns of h in R1's input; the codes follow them."""
    h_cols = H_COLS

    def __init__(self, table, lotd_cfg, W1, b1, W2, b2, R1=None, rb1=None, R2=None, rb2=None, R3=None, rb3=None, *, beta=100.0,
                 fac=(1.0, 1.0, 1.0), max_level=None, rounding=True):
        self.meta = olotd.LoDMeta(3, **lotd_cfg)
        self.rounding = rounding
        self.table16 = torch.as_tensor(table).detach().cpu().half().numpy()
        self.T = self.table16.astype(np.float64)
        w = lambda p: None if p is None else torch.as_tensor(p).detach().cpu().half().double().numpy()
        self.W1, self.b1, self.W2, self.b2 = w(W1), w(b1), w(W2).reshape(1, -1), w(b2).reshape(1)
        self.R1, self.rb1, self.R2, self.rb2, self.R3, self.rb3 = w(R1), w(rb1), w(R2), w(rb2), w(R3), w(rb3)
        self.beta = float(beta)
        self.fac = np.asarray(fac, dtype=np.float32).astype(np.float64)
        self.max_level = self.meta.n_levels if max_level is None else int(max_level)
        self.n_appear = 0 if R1 is None else self.R1.shape[1] - 54

    @classmethod
    def from_model(cls, model, max_level=None, rounding=True):
        """From a product LoTDNeuS (fields/neus.py): the parameters as the fused kernels see them."""
        s = model.implicit_surface
        d = s.decoder.layers
        # a geometry-only model (radiance_cfg=False) has no radiance net: sdf and nablas only
        r = [None] * 6 if model.radiance_net is None else [p for l in model.radiance_net.blocks.layers for p in (l.weight, l.bias)]
        fac = (s.sdf_scale / s.radius3d_original.detach().float().cpu()).tolist()
        return cls(s.encoding.flattened_params, s.encoding.lotd_cfg, d[0].weight, d[0].bias, d[1].weight, d[1].bias, *r,
                   beta=float(d[0].activation.beta), fac=fac, max_level=max_level, rounding=rounding)

    @property
    def f32(self):
        """the type the kernels receive cotangents in: fp32, or float64 without rounding"""
        return np.float32 if self.rounding else np.float64

    def r16(self, v):
        return v.astype(np.float16).astype(np.float64) if self.rounding else v

    # ------------------------------------------------------------------ LoTD geometry
    @staticmethod
    def xs_of(x):
        """network space [-1,1] -> table space, fp32 as the kernels evaluate it (x * 0.5 is exact, so x*.5+.5 == fma)"""
        x = np.asarray(x, dtype=np.float32)
        v = (x * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
        return np.clip(v, np.float32(1.0e-6), np.float32(1.0) - np.float32(1.0e-6)).astype(np.float32)

    def levels(self, xs):
        """per contributing pseudo level: (column offset in h, table index of feature 0 per corner [8, N], trilinear weight [8, N],
        dw [3, 8, N] = d(weight)/d(xs_gd)).  Weights are float64 products of the fp32 fractions."""
        meta, D = self.meta, 3
        for psl, lvl, loff, foff, ooff in olotd._level_iter(meta, self.max_level):
            res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
            scale = (res - 2).astype(np.float32)
            cell, frac = olotd.pos_fract(xs, scale)
            fr = frac.astype(np.float64)
            nf = meta.level_n_feats[lvl]
            idx = np.empty((8, xs.shape[0]), dtype=np.int64)
            w = np.empty((8, xs.shape[0]))
            dw = np.empty((D, 8, xs.shape[0]))
            for c in range(8):
                off = np.array([(c >> d) & 1 for d in range(D)], dtype=np.uint32)
                idx[c] = olotd.grid_index(meta, lvl, cell + off) * nf + foff + loff
                f = [fr[:, d] if (c >> d) & 1 else 1.0 - fr[:, d] for d in range(D)]
                w[c] = f[0] * f[1] * f[2]
                for gd in range(D):
                    o = [f[d] for d in range(D) if d != gd]
                    dw[gd, c] = (1.0 if (c >> gd) & 1 else -1.0) * float(scale[gd]) * o[0] * o[1]
            yield ooff, idx, w, dw

    def features(self, xs):
        """h [N, 32], J [N, 32, 3] (dh/dxs)."""
        if self.rounding:
            y, J = olotd.lod_fwd(self.meta, xs, self.table16, self.max_level, True)
            return y.astype(np.float64), J.astype(np.float64)
        N = xs.shape[0]
        h, J = np.zeros((N, 32)), np.zeros((N, 32, 3))
        for ooff, idx, w, dw in self.levels(xs):
            for f in range(2):
                v = self.T[idx + f]
                h[:, ooff + f] = (w * v).sum(0)
                J[:, ooff + f, :] = np.einsum("gcn,cn->ng", dw, v)
        return h, J

    def _scatter(self, xs, row_w=None, row_dw=None, gin=None):
        """table gradient, float64: the sum over points and corners c of row_w[:, col] w_c + row_dw[:, col] wsum_c, where
        wsum_c = sum_gd dw[gd, c] gin_gd is the derivative of gin . J wrt. the corner's table value (the second-order term)"""
        grad = np.zeros(self.T.shape[0])
        for ooff, idx, w, dw in self.levels(xs):
            ws = np.einsum("gcn,ng->cn", dw, gin) if row_dw is not None else None
            lo, hi = int(idx.min()), int(idx.max()) + 2
            for f in range(2):
                val = 0.0
                if row_w is not None:
                    val = val + w * row_w[None, :, ooff + f]
                if row_dw is not None:
                    val = val + ws * row_dw[None, :, ooff + f]
                grad[lo:hi] += np.bincount((idx + f - lo).ravel(), weights=np.broadcast_to(val, idx.shape).ravel(), minlength=hi - lo)
        return grad

    # ------------------------------------------------------------------ forward passes
    def _decoder(self, h):
        z = self.r16(h @ self.W1.T + self.b1)
        bz = self.beta * z
        lin = bz > 20.0
        s = np.where(lin, 1.0, _sigmoid(bz))
        a = np.where(lin, z, np.logaddexp(0.0, bz) / self.beta)
        a16 = self.r16(a)
        sdf = self.r16(a16 @ self.W2.T + self.b2)[:, 0]
        return z, lin, s, a16, sdf

    def sdf_scale(self, a16):
        """sum |a16 w2| + |b2| per point: the scale of the sdf's rounding error (one fp16 flip of a16_j moves sdf by <= 2^-10 of it)"""
        return np.abs(a16) @ np.abs(self.W2[0]) + np.abs(self.b2[0])

    def sdf(self, x, with_scale=False):
        """k_fused_sdf_tc: x [N, 3] fp32 network-space points -> sdf [N] (, sdf_scale [N])"""
        h, _ = self.features(self.xs_of(x))
        z, lin, s, a16, sdf = self._decoder(h)
        return (sdf, self.sdf_scale(a16)) if with_scale else sdf

    def color_forward(self, x, view_dirs, h_appear=None, with_rgb=True):
        """k_color_fwd at the points x [N, 3] with per-point view directions [N, 3] and appearance codes [N, n_appear].
        -> dict(sdf, nablas, rgb; sdf_scale (see sdf_scale); nablas_scale = 0.5 fac sum |r16(g) J| per point and axis, the
        scale of the nablas rounding error; and the intermediates the backward passes use).  with_rgb=False (or no radiance net):
        the geometry-only query k_color_fwd<false>, sdf and nablas; rgb is None and no radiance input is formed."""
        x = np.asarray(x, dtype=np.float32)
        xs = self.xs_of(x)
        h, J = self.features(xs)
        z, lin, s, a16, sdf = self._decoder(h)
        u = self.r16(self.W2[0] * s)
        g16 = self.r16(u @ self.W1)
        nab = np.einsum("nf,nfd->nd", g16, J) * 0.5 * self.fac
        nab_scale = np.einsum("nf,nfd->nd", np.abs(g16), np.abs(J)) * 0.5 * self.fac
        out = dict(sdf=sdf, nablas=nab, rgb=None, sdf_scale=self.sdf_scale(a16), nablas_scale=nab_scale, xs=xs, h=h, J=J, z=z, lin=lin,
                   s=s, a16=a16, u=u, g16=g16)
        if not with_rgb or self.R1 is None:
            return out
        v = torch.as_tensor(np.asarray(view_dirs), dtype=torch.float32 if self.rounding else torch.float64)
        sh = onets.sh_encode(v, 4).double().numpy()
        parts = [x.astype(np.float64), sh, np.clip(nab, -1.0, 1.0), h]
        if self.n_appear:
            parts.append(np.asarray(h_appear, dtype=np.float32).astype(np.float64))
        X = self.r16(np.concatenate(parts, -1))
        Y1 = np.maximum(self.r16(X @ self.R1.T + self.rb1), 0.0)
        Y2 = np.maximum(self.r16(Y1 @ self.R2.T + self.rb2), 0.0)
        rgb = self.r16(_sigmoid(self.r16(Y2 @ self.R3.T + self.rb3)))
        out.update(rgb=rgb, X=X, Y1=Y1, Y2=Y2)
        return out

    # ------------------------------------------------------------------ backward passes
    def sdf_backward(self, x, d_sdf):
        """k_sdf_bwd_tc: gradients of sum(d_sdf * sdf) -> dict(grid [P], W1, b1, W2, b2), float64"""
        xs = self.xs_of(x)
        h, _ = self.features(xs)
        z, lin, s, a16, sdf = self._decoder(h)
        d = np.asarray(d_sdf, dtype=self.f32).astype(np.float64)[:, None]
        dz = self.r16(d * self.W2[0] * s)
        da = self.r16(d * a16)
        dH = dz @ self.W1
        return dict(grid=self._scatter(xs, row_w=dH), W1=dz.T @ h, b1=dz.sum(0), W2=da.sum(0)[None], b2=d.sum(0))

    def color_backward(self, fwd, g_sdf=None, g_nablas=None, g_rgb=None):
        """k_color_rad_bwd + k_color_sdf_bwd: gradients of sum(g_sdf sdf + g_nablas nablas + g_rgb rgb) through the forward
        `fwd` (color_forward) -> dict(grid [P], W1, b1, W2, b2, R1, rb1, R2, rb2, R3, rb3), float64.  A geometry-only forward
        (rgb None) takes no g_rgb: the radiance net's gradients are exact zeros (absent without a radiance net)."""
        N = fwd["sdf"].shape[0]
        f32 = lambda v, shape: np.zeros(shape) if v is None else np.asarray(v, dtype=self.f32).astype(np.float64)
        g_sdf, g_nab = f32(g_sdf, (N,)), f32(g_nablas, (N, 3))
        out = {}
        if fwd["rgb"] is None:
            assert g_rgb is None, "a geometry-only forward has no rgb"
            dh_r = 0.0
            if self.R1 is not None:
                out.update({k: np.zeros(getattr(self, k).shape) for k in ("R1", "rb1", "R2", "rb2", "R3", "rb3")})
        else:
            g_rgb = f32(g_rgb, (N, 3))
            rgb, X, Y1, Y2 = fwd["rgb"], fwd["X"], fwd["Y1"], fwd["Y2"]
            # radiance net
            gy = self.r16(self.r16(g_rgb) * ((1.0 - rgb) * rgb))
            dZ2 = self.r16((Y2 > 0) * (gy @ self.R3))
            dZ1 = self.r16((Y1 > 0) * (dZ2 @ self.R2))
            dh_r = dZ1 @ self.R1[:, self.h_cols]
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
        return out
