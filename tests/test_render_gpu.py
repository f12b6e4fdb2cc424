"""End-to-end parity of the rendering path: neuralsim_b200 (CUDA) vs the CPU oracle on identical rays, weights and grid.
Tolerance from BASELINE.json north_star: rendered RGB / depth / normals within 1e-4 relative L2."""
import numpy as np
import pytest
import torch

from oracle import render as orender
from oracle import scene as oscene
from util import make_pair, product_grads, rel_l2

pytestmark = pytest.mark.gpu
TOL = 1.0e-4
# bounds = ~3 x the measured errors; grid, dec_W1 and ln_inv_s carry the largest (round 1 accepted 2e-2 for all of them)
GRAD_TOL_DEFAULT = 2e-3
GRAD_TOL = dict(grid=4e-3, dec_W1=8e-3, ln_inv_s=3e-3)


def _rays(H=30, W=40, k=1):
    return oscene.pinhole_rays(H, W, oscene.orbit_camera(k, 8, radius=3.0, elev_deg=25.0))


def _oracle_render(P, ro, rd, training=True, perturb=False):
    rt = orender.ray_test(ro, rd, near=0.01)
    vb, det = orender.neus_ray_query(P, oscene.make_occ_grid(), rt, rays_h_appear=torch.zeros(rt["num_rays"], P.n_appear), perturb=perturb)
    return orender.volume_integration(vb, ro.shape[0], training=training), vb, det, rt


def _product_render(model, ro, rd, cuda, training=True):
    from neuralsim_b200.renderer import SingleVolumeRenderer
    r = SingleVolumeRenderer(dict(near=0.01)).train(training)
    model.train(training)
    return r.render(model, ro.to(cuda), rd.to(cuda), rays_h_appear=torch.zeros(ro.shape[0], 4, device=cuda), return_buffer=True, return_details=True)


@pytest.mark.parametrize("ln_inv_s", [0.2996, 0.5298, 0.7601])      # inv_s = 20, 200, 2000
def test_forward_parity(cuda, ln_inv_s):
    P, model = make_pair(cuda, ln_inv_s_init=ln_inv_s)
    ro, rd = _rays()
    with torch.no_grad():
        ref, vb_ref, det_ref, rt = _oracle_render(P, ro, rd)
        out = _product_render(model, ro, rd, cuda)
    got, vb = out["rendered"], out["volume_buffer"]
    # integer structure: hit rays, marched sample counts
    assert torch.equal(out["ray_tested"]["rays_inds"].cpu(), rt["rays_inds"])
    assert torch.equal(out["details"]["march.num_per_ray"].cpu(), det_ref["march.num_per_ray"])
    for k in ("rgb_volume", "depth_volume", "normals_volume", "mask_volume"):
        assert rel_l2(got[k], ref[k]) <= TOL, (k, rel_l2(got[k], ref[k]))
    assert float(got["mask_volume"].sum()) > 50.0                      # the sphere is actually rendered


def test_backward_parity(cuda):
    P, model = make_pair(cuda)
    ro, rd = _rays(24, 32, 3)
    P.requires_grad_(True)
    ref, *_ = _oracle_render(P, ro, rd)
    loss_ref = sum(v.mean() for v in ref.values())
    loss_ref.backward()
    out = _product_render(model, ro, rd, cuda)["rendered"]
    loss = sum(v.mean() for v in out.values())
    loss.backward()
    assert abs(float(loss) - float(loss_ref)) <= 1e-4 * abs(float(loss_ref))
    g = product_grads(model)
    errs = {k: rel_l2(g[k], t.grad) for k, t in P.tensors().items() if g[k] is not None}
    import json, os
    if os.path.isdir("gpurun_out"):                         # achieved per-tensor errors, kept as evidence (profiles/)
        json.dump(errs, open("gpurun_out/grad_parity_errors.json", "w"), indent=1)
    print("gradient rel-L2 vs the oracle:", {k: f"{v:.2e}" for k, v in errs.items()})
    for k, t in P.tensors().items():
        assert g[k] is not None, k
        # Both sides round the cotangents where the autocast graph rounds them; what remains is accumulation order (fp32 atomics here,
        # fp64-free serial sums in the oracle) and cuBLAS-vs-CPU GEMM order.  Per-tensor bounds = ~3 x the measured errors;
        # a missing or wrong term in the second-order path shows up as O(1).
        assert errs[k] <= GRAD_TOL.get(k, GRAD_TOL_DEFAULT), (k, errs[k])


def test_eval_mode_and_chunking(cuda):
    P, model = make_pair(cuda)
    ro, rd = _rays(20, 28, 5)
    from neuralsim_b200.renderer import SingleVolumeRenderer
    r = SingleVolumeRenderer(dict(near=0.01)).eval()
    model.eval()
    with torch.no_grad():
        ref, *_ = _oracle_render(P, ro, rd, training=False)
        a = r.render(model, ro.to(cuda), rd.to(cuda), rays_h_appear=torch.zeros(ro.shape[0], 4, device=cuda))["rendered"]
        b = r.render(model, ro.to(cuda), rd.to(cuda), rays_h_appear=torch.zeros(ro.shape[0], 4, device=cuda), rayschunk=137)["rendered"]
    for k in a:
        assert rel_l2(a[k], ref[k]) <= TOL, k
        assert torch.allclose(a[k], b[k], rtol=1e-5, atol=1e-6), k       # rays are independent: chunking changes nothing


def test_no_hit_and_empty_inputs(cuda):
    P, model = make_pair(cuda)
    from neuralsim_b200.renderer import SingleVolumeRenderer
    r = SingleVolumeRenderer(dict(near=0.01))
    o = torch.tensor([[5., 5, 5], [0., 0, -3]], device=cuda); d = torch.tensor([[0., 0, 1], [0.9, 0.1, 0.3]], device=cuda)
    d = torch.nn.functional.normalize(d, dim=-1)
    out = r.render(model, o, d, rays_h_appear=torch.zeros(2, 4, device=cuda))["rendered"]          # rays that miss the box
    assert float(out["mask_volume"].abs().sum()) == 0.0
    model.accel.occ.set_occ_grid(torch.zeros(64, 64, 64, dtype=torch.bool))                         # nothing occupied: coarse-only branch
    ro, rd = _rays(8, 8, 0)
    out = r.render(model, ro.to(cuda), rd.to(cuda), rays_h_appear=torch.zeros(64, 4, device=cuda))["rendered"]
    assert torch.isfinite(out["rgb_volume"]).all()
    out = r.render(model, ro[:0].to(cuda), rd[:0].to(cuda), rays_h_appear=torch.zeros(0, 4, device=cuda))["rendered"]
    assert out["rgb_volume"].shape == (0, 3)


def test_full_frame_size_independent_properties(cuda):
    """BASELINE.json's full size (one 800x600 frame, 480 000 rays, ~30 M SDF queries; far beyond what the CPU oracle finishes): properties that
    need no oracle -- (1) rays are independent: the frame rendered in one call (image-ordered rays -> ray-tiled kernels), in chunks, and as a
    random permutation of its rays (incoherent rays -> ray-major kernels) is the same image; (2) so are the parameter gradients;
    (3) the mask is a transmittance complement in [0, 1]; depth lies inside the ray's box interval; pixels that miss the sphere render 0."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model = bench.build_model(cuda).train()
    ro, rd = bench.pinhole_rays(bench.H, bench.W, bench.orbit(1, 8))
    ro, rd = ro.to(cuda), rd.to(cuda)
    ha = torch.zeros(ro.shape[0], 4, device=cuda)
    ren = SingleVolumeRenderer(dict(near=0.01)).train()

    def run(o, d, chunk):
        model.zero_grad(set_to_none=True)
        outs, n = [], o.shape[0]
        for s in range(0, n, chunk):
            out = ren.render(model, o[s:s + chunk], d[s:s + chunk], rays_h_appear=ha[:min(chunk, n - s)])["rendered"]
            loss = sum(v.sum() for v in out.values()) / n
            if loss.requires_grad:
                loss.backward()
            outs.append({k: v.detach() for k, v in out.items()})
        g = model.implicit_surface.encoding.flattened_params.grad.clone()
        gw = model.radiance_net.blocks.layers[0].weight.grad.clone()
        return {k: torch.cat([o_[k] for o_ in outs], 0) for k in outs[0]}, g, gw

    full, g_full, gw_full = run(ro, rd, ro.shape[0])
    chunked, g_ch, gw_ch = run(ro, rd, 100_000)
    perm = torch.randperm(ro.shape[0], device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))
    shuf, g_sh, gw_sh = run(ro[perm].contiguous(), rd[perm].contiguous(), ro.shape[0])
    for k in full:
        assert rel_l2(chunked[k], full[k]) <= 1e-6, k
        assert rel_l2(shuf[k], full[k][perm]) <= 1e-6, k
    for a, b in ((g_ch, g_full), (g_sh, g_full), (gw_ch, gw_full), (gw_sh, gw_full)):
        assert rel_l2(a, b) <= 2e-3                       # fp32 atomics: summation order
    m = full["mask_volume"]
    assert float(m.min()) >= 0.0 and float(m.max()) <= 1.0 + 1e-5
    hit = m > 0.5
    assert 0.05 < float(hit.float().mean()) < 0.2          # the sphere of radius 0.5 seen from 3 units covers ~9 % of the frame
    dep = full["depth_volume"][hit]
    assert float(dep.min()) > 2.0 and float(dep.max()) < 3.2
    assert float(full["rgb_volume"][~(m > 0)].abs().max()) == 0.0
