"""Fused colour / normal query (csrc/color_tc.cu: three wgmma kernels) against the module path it replaces
(LoTDNeuS.forward = LoTDFunctionFwdDydx -> autocast decoder -> autograd.grad -> LoTDFunctionBwdDydx -> RadianceNet, which the
render tests pin against the CPU oracle) and against the CPU oracle directly."""
import numpy as np
import pytest
import torch

from oracle import nets as onets
from util import make_pair, product_grads, rel_l2

pytestmark = pytest.mark.gpu


def _points(n_rays=300, per_ray=23, seed=0):
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g), dim=-1) * 2.5
    d = torch.nn.functional.normalize(-o + 0.3 * torch.randn(n_rays, 3, generator=g), dim=-1) * (0.8 + 0.4 * torch.rand(n_rays, 1, generator=g))
    ridx = torch.arange(n_rays).repeat_interleave(per_ray)
    t = (1.6 + 1.9 * torch.rand(n_rays * per_ray, generator=g))
    ha = 0.1 * torch.randn(n_rays, 4, generator=g)
    return o.cuda(), d.cuda(), ridx.cuda(), t.cuda(), ha.cuda()


def _unfused(model, o, d, ridx, t, v, ha, nablas_has_grad=True):
    x = torch.addcmul(o[ridx], d[ridx], t.unsqueeze(-1))
    return model.forward(x, v=v[ridx], h_appear=ha[ridx], nablas_has_grad=nablas_has_grad, with_rgb=True, with_normal=True)


def test_fused_color_forward_matches_module_and_oracle():
    P, model = make_pair("cuda")
    o, d, ridx, t, ha = _points()
    v = d / d.norm(dim=-1, keepdim=True)
    with torch.no_grad():
        ref = _unfused(model, o, d, ridx, t, v, ha)
        got = model.forward_on_rays(ridx, t, o, d, v, ha)
    x = torch.addcmul(o[ridx], d[ridx], t.unsqueeze(-1))
    assert torch.equal(got["x"], x)
    # sdf / rgb are fp16-valued: the tensor-core accumulation order may flip a last fp16 bit on a few samples
    assert (got["sdf"] - ref["sdf"].float()).abs().max() <= 2e-3 and rel_l2(got["sdf"], ref["sdf"].float()) < 2e-4
    assert rel_l2(got["nablas"], ref["nablas"].float()) < 2e-3
    assert (got["rgb"] - ref["rgb"].float()).abs().max() <= 4e-3 and rel_l2(got["rgb"], ref["rgb"].float()) < 5e-4
    # CPU oracle on a subset
    sel = torch.arange(0, x.shape[0], 7)
    with torch.no_grad():
        oref = onets.forward(P, x[sel].cpu(), v[ridx][sel].cpu(), ha[ridx][sel].cpu(), nablas_has_grad=False)
    assert rel_l2(got["sdf"][sel], oref["sdf"]) < 2e-4
    assert rel_l2(got["nablas"][sel], oref["nablas"]) < 2e-3
    assert rel_l2(got["rgb"][sel], oref["rgb"]) < 5e-4


@pytest.mark.parametrize("which", ["rgb", "nablas", "all"])
def test_fused_color_backward_matches_module(which):
    P, model = make_pair("cuda")
    o, d, ridx, t, ha = _points(seed=1)
    v = d / d.norm(dim=-1, keepdim=True)
    n = t.numel()
    g = torch.Generator("cuda").manual_seed(3)
    c_rgb, c_nab, c_sdf = (torch.randn(n, 3, device="cuda", generator=g), torch.randn(n, 3, device="cuda", generator=g),
                           torch.randn(n, device="cuda", generator=g))

    def loss(out):
        l = 0
        if which in ("rgb", "all"):
            l = l + (out["rgb"].float() * c_rgb).sum()
        if which in ("nablas", "all"):
            l = l + (out["nablas"].float() * c_nab).sum() * 0.05
        if which == "all":
            l = l + (out["sdf"].float() * c_sdf).sum() * 0.1
        return l

    model.zero_grad(set_to_none=True)
    loss(_unfused(model, o, d, ridx, t, v, ha)).backward()
    ref = product_grads(model)
    model.zero_grad(set_to_none=True)
    loss(model.forward_on_rays(ridx, t, o, d, v, ha)).backward()
    got = product_grads(model)
    for k, r in ref.items():
        if r is None or k == "ln_inv_s":
            assert got[k] is None or float(got[k].abs().max()) == 0 or k == "ln_inv_s"
            continue
        assert got[k] is not None, k
        if float(r.abs().max()) == 0:
            assert float(got[k].abs().max()) < 1e-6, k
            continue
        assert rel_l2(got[k], r) < 2e-2, (k, rel_l2(got[k], r))


def test_fused_color_ragged_tile_and_no_grad():
    P, model = make_pair("cuda")
    o, d, ridx, t, ha = _points(n_rays=37, per_ray=5, seed=2)       # 185 points: one full + one partial tile
    v = d / d.norm(dim=-1, keepdim=True)
    with torch.no_grad():
        a = model.forward_on_rays(ridx, t, o, d, v, ha)
        b = model.forward_on_rays(ridx[:100], t[:100], o, d, v, ha)
    for k in ("sdf", "nablas", "rgb"):
        assert torch.equal(a[k][:100], b[k])
    e = model.forward_on_rays(ridx[:0], t[:0], o, d, v, ha)
    assert e["rgb"].shape == (0, 3)
