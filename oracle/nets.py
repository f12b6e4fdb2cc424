"""CPU restatement of the tiny networks on the path: SH view-direction embedding, the autocast(fp16)
DenseLayer/MLP stack, the LoTD-SDF decoder with analytic nablas and the radiance net.  TEST INFRASTRUCTURE.

Follows (paths relative to nr3d_lib):
  SH basis        externals/shencoder/shencoder.cu:33-80 (real SH, degree<=4 as used by CFG `degree: 4`)
  DenseLayer/MLP  nr3d_lib/models/layers.py:228-312, nr3d_lib/models/blocks/mlp.py:26-125
  LoTDSDF         nr3d_lib/models/fields/sdf/lotd_sdf.py:176-257 (forward, forward_sdf_nablas)
  encoding        nr3d_lib/models/grid_encodings/lotd/lotd_encoding.py:150-213 (x/2+0.5, nablas/2)
                  nr3d_lib/models/grid_encodings/lotd/lotd.py:60,150,205 (clamp 1e-6, loss_scale 128)
  RadianceNet     nr3d_lib/models/fields/nerf/mlp_nerf.py:267-289
  LoTDNeuS        nr3d_lib/models/fields/neus/lotd_neus.py:141-167
  variance        nr3d_lib/models/fields/neus/variance.py:122-142

Autocast model.  The reference MLP is plain PyTorch under `torch.autocast('cuda', fp16)` with fp32 master
weights: F.linear casts x, W, b to fp16, cuBLAS accumulates in fp32 and rounds the (bias-included) result
once to fp16; Softplus is on autocast's fp32 list (input promoted to fp32, result fp32, re-rounded to fp16
by the next linear); ReLU / Sigmoid run in fp16.  `linear16` below is that contract:
    out = fp16( sum_k float(x16_k) * float(W16_jk)  [fp32]  + float(b16_j) ).
All functions here are differentiable torch so that autograd provides the oracle gradients
(incl. the second-order path through `nablas`).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import lotd as olotd


# ------------------------------------------------------------------ rounding helpers
class _RoundHalfSTE(torch.autograd.Function):
    """fp32 -> fp16 -> fp32 rounding whose backward also rounds the incoming gradient to fp16.
    This is what a `.half()` cast node does in the autocast graph (grad of a cast = cast of the grad)."""

    @staticmethod
    def forward(ctx, x):
        return x.half().float()

    @staticmethod
    def backward(ctx, g):
        return g.half().float()


def r16(x):
    return _RoundHalfSTE.apply(x)


def linear16(x, W, b):
    """autocast F.linear (layers.py:302-307): fp16 operands, fp32 accumulate, one rounding to fp16.
    x is any float tensor (rounded to fp16 on entry), W/b fp32 masters."""
    out = F.linear(r16(x), r16(W), None if b is None else r16(b))
    return r16(out)


def softplus_beta(x, beta=100.0, threshold=20.0):
    """nn.Softplus(beta) as ATen evaluates it in fp32: x if x*beta > threshold else log1p(exp(x*beta))/beta."""
    return F.softplus(x, beta=beta, threshold=threshold)


# ------------------------------------------------------------------ SH
def sh_encode(v, degree=4):
    """Real spherical-harmonics basis of a (unit) direction, fp32 [..., degree^2].  shencoder.cu:47-80."""
    assert 1 <= degree <= 4
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    out = [torch.full_like(x, 0.28209479177387814)]
    if degree > 1:
        out += [-0.48860251190291987 * y, 0.48860251190291987 * z, -0.48860251190291987 * x]
    if degree > 2:
        xy, yz, xz, x2, y2, z2 = x * y, y * z, x * z, x * x, y * y, z * z
        out += [1.0925484305920792 * xy, -1.0925484305920792 * yz,
                0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz,
                0.54627421529603959 * x2 - 0.54627421529603959 * y2]
    if degree > 3:
        out += [0.59004358992664352 * y * (-3.0 * x2 + y2), 2.8906114426405538 * xy * z,
                0.45704579946446572 * y * (1.0 - 5.0 * z2), 0.3731763325901154 * z * (5.0 * z2 - 3.0),
                0.45704579946446572 * x * (1.0 - 5.0 * z2), 1.4453057213202769 * z * (x2 - y2),
                0.59004358992664352 * x * (-x2 + 3.0 * y2)]
    return torch.stack(out, -1)


# ------------------------------------------------------------------ parameter container
def kaiming_linear(gen, fan_out, fan_in):
    """nn.Linear / DenseLayer default init (layers.py:283-296): U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for W and b."""
    bound = 1.0 / math.sqrt(fan_in)
    W = (torch.rand(fan_out, fan_in, generator=gen) * 2 - 1) * bound
    b = (torch.rand(fan_out, generator=gen) * 2 - 1) * bound
    return W, b


class LoTDNeuSParams:
    """Weights of CFG's model (SURVEY §8 header): LoTD 16 lvl x 2 feat (gen_ngp), SDF decoder 32->64->1
    Softplus(100), radiance net 58->64->64->3 ReLU/Sigmoid, ln_inv_s.  fp32 masters, as in the reference."""

    def __init__(self, seed=42, lotd_cfg=None, W=64, n_appear=4, sh_degree=4, lotd_bound=1.0e-4,
                 sphere_radius=0.5, ln_inv_s_init=0.3, radius3d_original=1.0, sdf_scale=1.0):
        g = torch.Generator().manual_seed(seed)
        cfg = lotd_cfg or olotd.gen_ngp_cfg()
        self.lotd_cfg = cfg
        self.meta = olotd.LoDMeta(3, **cfg)
        nf = self.meta.n_encoded_dims
        # lotd_encoding.py:257-271 `uniform_to_type`: U(-bound, bound)
        self.grid = ((torch.rand(self.meta.n_params, generator=g) * 2 - 1) * lotd_bound)
        self.dec_W1, self.dec_b1 = kaiming_linear(g, W, nf)
        self.dec_W2, self.dec_b2 = kaiming_linear(g, 1, W)
        self.sh_degree = sh_degree
        self.n_appear = n_appear
        in_rad = 3 + sh_degree ** 2 + 3 + nf + n_appear
        self.rad_W1, self.rad_b1 = kaiming_linear(g, W, in_rad)
        self.rad_W2, self.rad_b2 = kaiming_linear(g, W, W)
        self.rad_W3, self.rad_b3 = kaiming_linear(g, 3, W)
        self.ln_inv_s = torch.tensor([ln_inv_s_init])
        self.ln_inv_s_factor = 10.0
        self.radius3d_original = radius3d_original
        self.sdf_scale = sdf_scale
        self.sphere_radius = sphere_radius

    def tensors(self):
        return dict(grid=self.grid, dec_W1=self.dec_W1, dec_b1=self.dec_b1, dec_W2=self.dec_W2, dec_b2=self.dec_b2,
                    rad_W1=self.rad_W1, rad_b1=self.rad_b1, rad_W2=self.rad_W2, rad_b2=self.rad_b2,
                    rad_W3=self.rad_W3, rad_b3=self.rad_b3, ln_inv_s=self.ln_inv_s)

    def requires_grad_(self, flag=True):
        for k, t in self.tensors().items():
            t.requires_grad_(flag)
        return self

    def forward_inv_s(self):
        """variance.py:137-141 with w=0 (mix_linear before ctrl_start_it): exp(ln_inv_s * factor)."""
        return torch.exp(self.ln_inv_s * self.ln_inv_s_factor)


# ------------------------------------------------------------------ LoTD encoding as autograd functions
class _LoTDFwd(torch.autograd.Function):
    """LoTDFunction (lotd.py:48-119): y = lod_fwd(clamp(x)), backward -> dL_dgrid (x has no grad here)."""

    @staticmethod
    def forward(ctx, meta, x01, grid16, max_level):
        xc = x01.clamp(1.0e-6, 1 - 1.0e-6)
        y, _ = olotd.lod_fwd(meta, xc.numpy(), grid16.numpy(), max_level, False)
        ctx.meta, ctx.max_level = meta, max_level
        ctx.save_for_backward(xc, grid16)
        return torch.from_numpy(y)

    @staticmethod
    def backward(ctx, dL_dy):
        xc, grid16 = ctx.saved_tensors
        # lotd.py:94-106: (dL_dy * 128) -> kernel -> / 128 ; exact power-of-two scaling, dropped here.
        g = olotd.lod_bwd_grid(ctx.meta, dL_dy.numpy(), xc.numpy(), grid16.shape[0], ctx.max_level)
        return None, None, torch.from_numpy(g).to(grid16.dtype), None


class _LoTDFwdDydx(torch.autograd.Function):
    """LoTDFunctionFwdDydx (lotd.py:121-191)."""

    @staticmethod
    def forward(ctx, meta, x01, grid16, max_level):
        xc = x01.clamp(1.0e-6, 1 - 1.0e-6)
        y, dydx = olotd.lod_fwd(meta, xc.numpy(), grid16.numpy(), max_level, True)
        ctx.meta, ctx.max_level = meta, max_level
        ctx.save_for_backward(xc, grid16)
        dydx = torch.from_numpy(dydx)
        ctx.mark_non_differentiable(dydx)
        return torch.from_numpy(y), dydx

    @staticmethod
    def backward(ctx, dL_dy, _):
        if dL_dy is None:
            return None, None, None, None
        xc, grid16 = ctx.saved_tensors
        g = olotd.lod_bwd_grid(ctx.meta, dL_dy.numpy(), xc.numpy(), grid16.shape[0], ctx.max_level)
        return None, None, torch.from_numpy(g).to(grid16.dtype), None


class _LoTDBwdDydx(torch.autograd.Function):
    """LoTDFunctionBwdDydx (lotd.py:193-268): dL_dx = J^T dL_dy; its backward is the 2nd-order pass."""

    @staticmethod
    def forward(ctx, meta, dL_dy, x01, grid16, dy_dx, max_level):
        xc = x01.clamp(1.0e-6, 1 - 1.0e-6)
        ctx.meta, ctx.max_level = meta, max_level
        ctx.save_for_backward(dL_dy, xc, grid16, dy_dx)
        return torch.from_numpy(olotd.lod_bwd_input(dL_dy.numpy(), dy_dx.numpy()))

    @staticmethod
    def backward(ctx, dL_ddLdx):
        dL_dy, xc, grid16, dy_dx = ctx.saved_tensors
        a, b, _ = olotd.lod_bwd_bwd_input(ctx.meta, dL_ddLdx.numpy(), dL_dy.numpy(), xc.numpy(), grid16.numpy(),
                                          dy_dx.numpy(), ctx.max_level, ctx.needs_input_grad[1], ctx.needs_input_grad[3])
        a = None if a is None else torch.from_numpy(a).to(dL_dy.dtype)
        b = None if b is None else torch.from_numpy(b).to(grid16.dtype)
        return None, a, None, b, None, None


class _Grid16(torch.autograd.Function):
    """`params.to(torch.half)` (lotd.py:432): fp32 master -> fp16 view; the gradient comes back as fp16
    in the reference (and is then accumulated into the fp32 .grad)."""

    @staticmethod
    def forward(ctx, g32):
        return g32.half()

    @staticmethod
    def backward(ctx, g):
        return g.float()


# ------------------------------------------------------------------ model forward passes
def forward_sdf(P: LoTDNeuSParams, x, max_level=None):
    """LoTDSDF.forward (lotd_sdf.py:176-200).  x in [-1,1]^3 fp32 -> dict(sdf fp32-valued-fp16, h)."""
    grid16 = _Grid16.apply(P.grid)
    h = _LoTDFwd.apply(P.meta, x.detach() / 2. + 0.5, grid16, max_level).float()   # fp16 values
    z = linear16(h, P.dec_W1, P.dec_b1)
    a = softplus_beta(z)                       # fp32
    out = linear16(a, P.dec_W2, P.dec_b2)
    return dict(sdf=out[..., 0], h=h)


def forward_sdf_nablas(P: LoTDNeuSParams, x, nablas_has_grad=True, max_level=None):
    """LoTDSDF.forward_sdf_nablas (lotd_sdf.py:201-257)."""
    grid16 = _Grid16.apply(P.grid)
    x01 = x.detach() / 2. + 0.5
    with torch.enable_grad():
        h16, dy_dx = _LoTDFwdDydx.apply(P.meta, x01, grid16, max_level)
        h = h16.float()
        if not h.requires_grad:
            h.requires_grad_(True)
        z = linear16(h, P.dec_W1, P.dec_b1)
        a = softplus_beta(z)
        sdf = linear16(a, P.dec_W2, P.dec_b2)[..., 0]
        dL_dh = torch.autograd.grad(sdf, h, torch.ones_like(sdf), retain_graph=True,
                                    create_graph=nablas_has_grad)[0]
    dL_dh = r16(dL_dh)                         # the gradient wrt. the fp16 tensor h is an fp16 tensor
    nablas = _LoTDBwdDydx.apply(P.meta, dL_dh, x01, grid16, dy_dx, max_level) / 2.
    if not nablas_has_grad:
        nablas = nablas.detach()
    return dict(sdf=sdf, h=h, nablas=nablas * (P.sdf_scale / P.radius3d_original))


def radiance(P: LoTDNeuSParams, x, v, n, h, h_appear):
    """RadianceNet.forward (mlp_nerf.py:267-289) with [x, SH(v), n, h_extra, h_appear] -> sigmoid rgb (fp16 values)."""
    feats = [x, sh_encode(v, P.sh_degree), n, h]
    if P.n_appear > 0:
        feats.append(h_appear)
    inp = torch.cat(feats, -1)
    y = torch.relu(linear16(inp, P.rad_W1, P.rad_b1))
    y = torch.relu(linear16(y, P.rad_W2, P.rad_b2))
    y = linear16(y, P.rad_W3, P.rad_b3)
    return r16(torch.sigmoid(y))


def forward(P: LoTDNeuSParams, x, v, h_appear, nablas_has_grad=True):
    """LoTDNeuS.forward (lotd_neus.py:141-167)."""
    ret = forward_sdf_nablas(P, x, nablas_has_grad=nablas_has_grad)
    ha = None if h_appear is None else h_appear.expand(*x.shape[:-1], -1)
    ret["rgb"] = radiance(P, x, v, ret["nablas"].detach().clamp(-1, 1), ret["h"], ha)
    return ret


