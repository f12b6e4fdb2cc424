"""Fused forward_sdf kernel (csrc/fused.cu) against (i) the CPU oracle and (ii) the reference's actual code path on the
GPU: LoTD feature kernel + torch.autocast(fp16) MLP (what nr3d_lib's DenseLayer executes)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nets as onets
from util import make_pair

pytestmark = pytest.mark.gpu


def _ulp16_mismatch(a, b):
    """fraction of elements that differ, and the largest difference in fp16 ulps of the reference value."""
    a16, b16 = a.half(), b.half()
    diff = (a16.float() - b16.float()).abs()
    ulp = torch.maximum(b16.float().abs(), torch.tensor(6.1e-5, device=b.device)) * 2 ** -10
    return float((diff > 0).float().mean()), float((diff / ulp).max())


def test_fused_sdf_vs_oracle_and_autocast(cuda):
    P, model = make_pair(cuda)
    model.eval()
    g = torch.Generator().manual_seed(7)
    x = torch.rand(40000, 3, generator=g) * 2 - 1
    x[:4] = torch.tensor([[-1., -1, -1], [1, 1, 1], [0, 0, 0], [0.5, -0.5, 0.25]])
    with torch.no_grad():
        sdf_fused = model.implicit_surface.fused_sdf(x.to(cuda))
        sdf_torch = model.implicit_surface.forward(x.to(cuda))["sdf"]         # LoTD kernel + autocast cuBLAS MLP (reference path)
        sdf_oracle = onets.forward_sdf(P, x)["sdf"]
    assert sdf_torch.dtype == torch.float16
    # sdf is an fp16 number; both implementations round at the same points, so they agree except for rare 1-ulp flips
    frac, worst = _ulp16_mismatch(sdf_fused, sdf_torch.float())
    assert frac < 2e-2 and worst <= 2.0, (frac, worst)
    frac, worst = _ulp16_mismatch(sdf_fused.cpu(), sdf_oracle)
    assert frac < 2e-2 and worst <= 2.0, (frac, worst)
    assert float((sdf_fused.cpu() - (x.norm(dim=-1) - 0.5)).abs().max()) < 0.05   # the synthetic scene is a sphere


def test_fused_sdf_rays_matches_points(cuda):
    P, model = make_pair(cuda)
    g = torch.Generator().manual_seed(8)
    o = (torch.rand(500, 3, generator=g) * 2 - 1).to(cuda); d = torch.nn.functional.normalize(torch.randn(500, 3, generator=g), dim=-1).to(cuda)
    ridx = torch.randint(0, 500, (20000,), generator=g).to(cuda); t = (torch.rand(20000, generator=g) * 0.5).to(cuda)
    with torch.no_grad():
        a = model.implicit_surface.fused_sdf_rays(ridx, t, o, d)
        b = model.implicit_surface.fused_sdf(torch.addcmul(o[ridx], d[ridx], t.unsqueeze(-1)))
        t2 = t[:19500].view(500, 39)
        c = model.implicit_surface.fused_sdf_rays(torch.arange(500, device=cuda), t2, o, d)
        e = model.implicit_surface.fused_sdf(torch.addcmul(o.unsqueeze(1), d.unsqueeze(1), t2.unsqueeze(-1)))
    assert torch.equal(a, b) and torch.equal(c, e)


def test_tensor_core_kernel_matches_cuda_core_kernel(cuda):
    """csrc/fused_tc.cu (wgmma, what LoTDSDF.fused_sdf runs) against csrc/fused.cu's k_fused_sdf (CUDA cores): same rounding points, fp32
    accumulation order differs.  The reference comes from nsb_fused_sdf with sdf_simt = 1 and the feature output h_out_half, which only
    k_fused_sdf writes: its sentinels must be gone."""
    from neuralsim_b200 import _lib
    P, model = make_pair(cuda)
    s = model.implicit_surface
    grid16, dec = s._fused_state()
    g = torch.Generator().manual_seed(11)
    for n in (1, 127, 128, 129, 5000, 200001):
        x = (torch.rand(n, 3, generator=g) * 2 - 1).to(cuda)
        ref = torch.empty(n, device=cuda)
        h = torch.full((n, 32), float("nan"), dtype=torch.half, device=cuda)
        _lib.check(_lib.lib().nsb_set_option(b"sdf_simt", 1))
        try:
            _lib.check(_lib.lib().nsb_fused_sdf(s.encoding.meta.c_ref, _lib.ptr(grid16, "f16"), ctypes.byref(dec), _lib.ptr(x, "f32"), _lib.c_i64(n),
                                                _lib.c_i32(s._ml(None)), _lib.ptr(ref), _lib.ptr(h), _lib.stream_ptr()), "fused_sdf")
        finally:
            _lib.check(_lib.lib().nsb_set_option(b"sdf_simt", 0))
        assert not bool(torch.isnan(h).any()), n                     # k_fused_sdf ran
        with torch.no_grad():
            got = s.fused_sdf(x)
        frac, worst = _ulp16_mismatch(got, ref)
        assert frac < 2e-2 and worst <= 2.0, (n, frac, worst)


def test_fused_backward_matches_autograd_chain(cuda):
    """nsb_fused_sdf_bwd (one wgmma kernel) against the unfused chain LoTDFunction + autocast MLP differentiated by torch."""
    P, model = make_pair(cuda)
    surf = model.implicit_surface
    g = torch.Generator().manual_seed(12)
    for n in (77, 128, 4000, 150001):
        x = (torch.rand(n, 3, generator=g) * 2 - 1).to(cuda)
        w = torch.randn(n, generator=g).to(cuda)
        params = [surf.encoding.flattened_params, *surf.decoder.parameters()]
        sdf_a = surf.forward(x)["sdf"].float()                          # reference chain
        ga = torch.autograd.grad((sdf_a * w).sum(), params)
        sdf_b = surf.fused_sdf_autograd(x)
        gb = torch.autograd.grad((sdf_b * w).sum(), params)
        frac, worst = _ulp16_mismatch(sdf_b, sdf_a)
        assert frac < 2e-2 and worst <= 2.0
        names = ["grid", "W1", "b1", "W2", "b2"]
        for k, a, b in zip(names, ga, gb):
            err = float((a.float() - b.float()).norm() / a.float().norm().clamp_min(1e-20))
            # the autocast chain rounds every cotangent to fp16 (and the table gradient twice); ours keeps fp32 except dz
            assert err < 1e-2, (n, k, err)
        # rays variant == points variant
        o = (torch.rand(50, 3, generator=g) * 2 - 1).to(cuda); d = torch.nn.functional.normalize(torch.randn(50, 3, generator=g), dim=-1).to(cuda)
        ridx = torch.randint(0, 50, (n,), generator=g).to(cuda); t = (torch.rand(n, generator=g) * 0.3).to(cuda)
        s1 = surf.fused_sdf_rays_autograd(ridx, t, o, d)
        g1 = torch.autograd.grad((s1 * w).sum(), params)
        s2 = surf.fused_sdf_autograd(torch.addcmul(o[ridx], d[ridx], t.unsqueeze(-1)))
        g2 = torch.autograd.grad((s2 * w).sum(), params)
        assert torch.equal(s1, s2)
        for a, b in zip(g1, g2):
            assert float((a - b).norm() / a.norm().clamp_min(1e-20)) < 1e-4     # atomics: order only
