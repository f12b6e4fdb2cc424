"""CPU: the adjoint of the one-launch step's ray test (tests/ray_adjoint64.py, what nsb_gather_rays_backward computes) against torch
autograd of the chain it differentiates -- AABBSpace.normalize_rays, the index of the rays that pass, view_dirs with a detached norm.
In float64 against the statement; in fp32 bit for bit against the kernel's order, with the gradient to d_c arriving as torch's engine
delivers it on the host-sized path: two per-ray ops created after view_dirs (the colour and the boundary query), then the view term."""
import numpy as np
import pytest
import torch

from neuralsim_b200.fields.space import AABBSpace
from ray_adjoint64 import adjoint, adjoint32


def _case(dtype, seed, n_rays=200):
    g = torch.Generator().manual_seed(seed)
    space = AABBSpace(aabb=[[-3.0, -1.5, -0.5], [5.0, 2.5, 1.5]], dtype=dtype)
    o = (torch.rand(n_rays, 3, generator=g, dtype=dtype) * 8 - 4).requires_grad_(True)
    d = (torch.randn(n_rays, 3, generator=g, dtype=dtype) * 2).requires_grad_(True)
    idx = torch.sort(torch.randperm(n_rays, generator=g)[: n_rays * 3 // 4]).values      # the rays that pass, ascending
    n = idx.shape[0]
    cot = [torch.randn(n, 3, generator=g, dtype=dtype) for _ in range(5)]                   # colour / boundary to o_c and d_c, view term
    for c in cot:
        c[torch.rand(n, generator=g) < 0.1] = 0                                             # rays that keep no sample
    return space, o, d, idx, cot


def _torch_chain(space, o, d, idx, cot, with_view=True):
    """-> (o.grad, d.grad, |d_c|): the host-sized path's autograd graph of the ray test and view directions"""
    on, dn = space.normalize_rays(o, d)
    o_c, d_c = on[idx], dn[idx]
    vn = d_c.detach().norm(dim=-1).clamp_min(1.0e-10)
    vd = d_c / vn.unsqueeze(-1)                               # created before the queries, as in neus_ray_query_march_occ_multi_upsample_compressed
    col = (o_c * cot[0]).sum() + (d_c * cot[2]).sum()         # the colour query's [o | d] terms
    bnd = (o_c * cot[1]).sum() + (d_c * cot[3]).sum()         # the boundary query's
    loss = bnd + col + ((vd * cot[4]).sum() if with_view else 0)
    loss.backward()
    return o.grad, d.grad, vn


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("with_view", [True, False], ids=["rgb", "no-rgb"])
def test_adjoint_float64_matches_autograd(seed, with_view):
    space, o, d, idx, cot = _case(torch.float64, seed)
    go, gd, vn = _torch_chain(space, o, d, idx, cot, with_view)
    want_o, want_d = adjoint(idx.numpy(), o.shape[0], space.radius3d.numpy(), (cot[0] + cot[1]).numpy(), (cot[2] + cot[3]).numpy(),
                             cot[4].numpy() if with_view else None, vn.numpy())
    np.testing.assert_allclose(go.numpy(), want_o, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(gd.numpy(), want_d, rtol=1e-13, atol=1e-15)
    miss = np.setdiff1d(np.arange(o.shape[0]), idx.numpy())
    assert (go.numpy()[miss] == 0).all() and (gd.numpy()[miss] == 0).all()


def test_wrong_adjoints_fail():
    """the comparison can fail: the statement without the view term, or without the division by the box's half-size"""
    space, o, d, idx, cot = _case(torch.float64, 3)
    _, gd, vn = _torch_chain(space, o, d, idx, cot)
    args = (idx.numpy(), o.shape[0])
    r = space.radius3d.numpy()
    no_view = adjoint(*args, r, (cot[0] + cot[1]).numpy(), (cot[2] + cot[3]).numpy())[1]
    no_div = adjoint(*args, np.ones(3), (cot[0] + cot[1]).numpy(), (cot[2] + cot[3]).numpy(), cot[4].numpy(), vn.numpy())[1]
    for wrong in (no_view, no_div):
        assert not np.allclose(gd.numpy(), wrong, rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_adjoint_fp32_order_is_autograds(seed):
    """fp32: the kernel's order of additions and divisions gives torch autograd's bits"""
    space, o, d, idx, cot = _case(torch.float32, seed, n_rays=4000)
    go, gd, vn = _torch_chain(space, o, d, idx, cot)
    c = [x.numpy() for x in cot]
    g_o = (np.float32(0) + c[0]) + c[1]                       # as the accumulator holds it: (0 + colour) + boundary
    want_o, want_d = adjoint32(idx.numpy(), o.shape[0], space.radius3d.numpy(), g_o, c[2], c[3], c[4], vn.numpy())
    assert np.array_equal(go.numpy().view(np.int32), want_o.view(np.int32))
    assert np.array_equal(gd.numpy().view(np.int32), want_d.view(np.int32))
