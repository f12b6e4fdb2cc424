"""Glue kernels of the per-ray query (csrc/neus_glue.cu): agreement with the chains of reference-API calls they replace (the pack_ops /
raymarch / raysample wrappers of this package, themselves pinned against the reference's kernels and the oracle), at one small shape per
kernel.  The kernels against a serial oracle of their own, at the sizes where they loop and at their edges: tests/test_glue_edges_gpu.py."""
import numpy as np
import pytest
import torch

from util import random_packs, rel_l2

pytestmark = pytest.mark.gpu


def test_scan_counts():
    from neuralsim_b200.graphics import neus_fused as NF
    g = torch.Generator().manual_seed(0)
    for n in (0, 1, 31, 1024, 1025, 50_000):
        c = (torch.randint(0, 7, (n,), generator=g) * (torch.rand(n, generator=g) < 0.4)).int().cuda()
        src = torch.arange(n, device="cuda") * 3 + 1
        sc = NF.scan_counts(c, want_first=True, want_info2=True, want_index=True, want_pack=True, src=src)
        cum = c.long().cumsum(0)
        first = cum - c.long()
        nz = c.nonzero()[:, 0]
        assert sc["total"] == int(c.sum()) and sc["n_nonzero"] == nz.numel()
        assert torch.equal(sc["first"].long(), first)
        assert torch.equal(sc["info2"].long(), torch.stack([first, c.long()], 1)) if n else True
        assert torch.equal(sc["index"], nz) and torch.equal(sc["src"], src[nz])
        assert torch.equal(sc["pack"], torch.stack([first[nz], c.long()[nz]], 1))


def test_merge_sorted_vals_equals_aligned_merge():
    from neuralsim_b200.graphics import neus_fused as NF
    from neuralsim_b200.graphics.pack_ops import get_pack_infos_from_batch, merge_two_packs_sorted_aligned
    rng = np.random.default_rng(1)
    pi = random_packs(rng, 900, 1, 200, "cuda")
    S = int(pi[-1].sum())
    g = torch.Generator().manual_seed(1)
    dep = torch.empty(S)
    for b, n in pi.cpu().tolist():
        dep[b:b + n] = (torch.rand(n, generator=g) * 3).sort().values
    dep = dep.cuda()
    dep[5:9] = dep[5]                                      # ties inside a pack
    sdf = torch.randn(S, device="cuda")
    for nb in (9, 33):
        fine = (torch.rand(pi.shape[0], nb, generator=g) * 3).sort(-1).values.cuda()
        fine[0, :3] = dep[pi[0, 0]]                        # ties across a and b
        sdf_f = torch.randn(pi.shape[0], nb, device="cuda")
        pa, pb, pim_ref = merge_two_packs_sorted_aligned(dep, pi, fine.flatten(), get_pack_infos_from_batch(pi.shape[0], nb, device="cuda"), b_sorted=True)
        dep_ref, sdf_ref = dep.new_empty(S + fine.numel()), dep.new_empty(S + fine.numel())
        dep_ref[pa], dep_ref[pb] = dep, fine.flatten()
        sdf_ref[pa], sdf_ref[pb] = sdf, sdf_f.flatten()
        dep_m, sdf_m, pim = NF.merge_sorted_vals(dep, sdf, pi, fine, sdf_f)
        assert torch.equal(pim, pim_ref) and torch.equal(dep_m, dep_ref) and torch.equal(sdf_m, sdf_ref)
        dep_m2, none, _ = NF.merge_sorted_vals(dep, None, pi, fine, None)
        assert none is None and torch.equal(dep_m2, dep_ref)


def test_assemble_boundary_equals_reference_chain():
    from neuralsim_b200.graphics import neus_fused as NF
    from neuralsim_b200.graphics.pack_ops import merge_two_batch_a_includes_b, packed_diff
    g = torch.Generator().manual_seed(2)
    R, nc = 701, 65
    near = torch.rand(R, generator=g) + 0.5
    coarse = (near[:, None] + torch.linspace(0, 1, nc)[None, :] * (1 + torch.rand(R, 1, generator=g))).cuda().contiguous()
    ridx_hit = torch.randperm(R, generator=g)[:260].sort().values.cuda()
    stages = [(coarse[ridx_hit, :1] + torch.rand(260, n, generator=g).sort(-1).values.cuda() * 1.5) for n in (9, 9, 33)]
    stages[0][:, 0] = coarse[ridx_hit, 7]                  # a fine sample equal to a coarse one
    stages[0] = stages[0].sort(-1).values                  # (every stage's row stays a sorted run)
    stages[1][:, 3] = stages[0][:, 2]                      # equal samples in two stages
    stages[1] = stages[1].sort(-1).values
    fine_all = torch.cat(stages, -1).contiguous()
    depths_1 = fine_all.sort(-1).values
    ridx_c = torch.arange(R, device="cuda")
    pidx0, pidx1, pi_ref = merge_two_batch_a_includes_b(coarse, ridx_c, depths_1, ridx_hit, a_sorted=True)
    S = coarse.numel() + depths_1.numel()
    d_ref, r_ref = coarse.new_zeros(S), ridx_hit.new_zeros(S)
    r_ref[pidx0], r_ref[pidx1] = ridx_c.unsqueeze(-1), ridx_hit.unsqueeze(-1)
    d_ref[pidx0], d_ref[pidx1] = coarse, depths_1
    mid_ref = d_ref + packed_diff(d_ref, pi_ref) / 2.
    d1, mid, ridx_all, pi = NF.assemble_boundary(coarse, ridx_hit, fine_all, run_len=[9, 9, 33])
    assert torch.equal(pi, pi_ref) and torch.equal(d1, d_ref) and torch.equal(ridx_all, r_ref) and torch.equal(mid, mid_ref)
    # no ray carries fine samples
    d1s, _, _, _ = NF.assemble_boundary(coarse, ridx_hit, depths_1)            # one sorted run per row
    assert torch.equal(d1s, d_ref)
    d1, mid, ridx_all, pi = NF.assemble_boundary(coarse, ridx_hit[:0], fine_all[:0])
    assert torch.equal(d1, coarse.flatten()) and torch.equal(pi[:, 1], torch.full((R,), nc, device="cuda"))
    # every ray carries fine samples (runs of listed rays longer than a chunk), and only the last one does
    fa = (coarse[:, :1] + torch.rand(R, 20, generator=g).sort(-1).values.cuda() * 1.5).contiguous()
    d1, _, ridx_all, pi = NF.assemble_boundary(coarse, ridx_c, fa)
    assert torch.equal(d1.view(R, nc + 20), torch.cat([coarse, fa], -1).sort(-1).values) and torch.equal(pi[:, 0], ridx_c * (nc + 20))
    d1, _, ridx_all, pi = NF.assemble_boundary(coarse, ridx_c[-1:], fa[-1:].contiguous())
    assert torch.equal(d1[:(R - 1) * nc], coarse[:-1].flatten()) and torch.equal(d1[(R - 1) * nc:], torch.cat([coarse[-1], fa[-1]]).sort().values)
    assert int(pi[-1, 1]) == nc + 20 and bool((ridx_all[(R - 1) * nc:] == R - 1).all())


def test_neus_alpha_compact_equals_compress_and_gathers():
    from neuralsim_b200.graphics import neus_fused as NF
    rng = np.random.default_rng(3)
    pi = random_packs(rng, 600, 1, 150, "cuda")
    S = int(pi[-1].sum())
    g = torch.Generator().manual_seed(3)
    t = torch.empty(S)
    sdf = torch.empty(S)
    for b, n in pi.cpu().tolist():
        tt = torch.rand(n, generator=g).sort().values * 2 + 0.5
        t[b:b + n] = tt
        sdf[b:b + n] = (1.4 - tt) * (0.5 + torch.rand(1, generator=g)) + 0.02 * torch.randn(n, generator=g)
    sdf[pi[3, 0]:pi[3, 0] + pi[3, 1]] = 1.0                # a pack that keeps nothing
    t, sdf = t.cuda(), sdf.cuda()
    ridx_all = torch.repeat_interleave(torch.arange(pi.shape[0], device="cuda"), pi[:, 1])
    rays_inds = torch.arange(pi.shape[0], device="cuda") * 2 + 5
    inv_s = torch.tensor(60.0, device="cuda", requires_grad=True)
    s1 = sdf.clone().requires_grad_(True)
    a_ref, nidx, pinf, pidx = NF.neus_alpha_compress(s1, inv_s, pi)
    s2 = sdf.clone().requires_grad_(True)
    inv2 = inv_s.detach().clone().requires_grad_(True)
    c = NF.neus_alpha_compact(s2, inv2, pi, ridx_all, t, rays_inds)
    assert torch.equal(c["pidx"], pidx) and torch.equal(c["nidx"], nidx) and torch.equal(c["pack_infos"], pinf)
    assert torch.equal(c["rays_inds_hit"], rays_inds[nidx]) and torch.equal(c["ridx"], ridx_all[pidx]) and torch.equal(c["t"], t[pidx])
    assert torch.equal(c["alpha"], a_ref[pidx])
    w = torch.randn(pidx.numel(), device="cuda")
    (a_ref[pidx] * w).sum().backward()
    (c["alpha"] * w).sum().backward()
    assert torch.equal(s2.grad, s1.grad)
    assert torch.allclose(inv2.grad, inv_s.grad, rtol=1e-4, atol=1e-7)     # atomics: summation order
    # nothing kept at all
    assert NF.neus_alpha_compact(torch.ones(S, device="cuda"), inv2.detach(), pi, ridx_all, t, rays_inds) is None


def test_march_lean_equals_occgrid_raymarch():
    from neuralsim_b200.graphics import neus_fused as NF
    from neuralsim_b200.graphics.raymarch import occgrid_raymarch
    from oracle import scene as oscene
    occ = oscene.make_occ_grid().cuda()
    ro, rd = oscene.pinhole_rays(40, 56, oscene.orbit_camera(2, 8))
    ro, rd = ro.cuda(), rd.cuda()
    near, far = torch.full((ro.shape[0],), 1.5, device="cuda"), torch.full((ro.shape[0],), 4.5, device="cuda")
    ref = occgrid_raymarch(occ, ro, rd, near, far, step_size=0.005, max_steps=4096)
    ridx_hit, pinfo, t0, ridx = NF.march_lean(occ, ro, rd, near, far, step_size=0.005, max_steps=4096)
    assert torch.equal(ridx_hit, ref.ridx_hit) and torch.equal(pinfo, ref.pack_infos) and torch.equal(t0, ref.depth_samples) and torch.equal(ridx, ref.ridx)
    assert NF.march_lean(torch.zeros_like(occ), ro, rd, near, far, step_size=0.005, max_steps=4096) is None


@pytest.mark.parametrize("near,far", [(None, None), (0.01, None), (0.5, 3.2)])
def test_ray_test_fused_equals_torch_chain(near, far):
    from neuralsim_b200.fields.space import AABBSpace
    sp = AABBSpace(aabb=[[-1.0, -0.7, -1.2], [0.9, 1.1, 0.8]], device="cuda")
    g = torch.Generator().manual_seed(4)
    o = (torch.randn(5000, 3, generator=g) * 2).cuda()
    d = torch.nn.functional.normalize(torch.randn(5000, 3, generator=g), dim=-1).cuda()
    d[7, 1] = 0.                                            # an axis-parallel ray
    o[8] = torch.tensor([0.2, 0.1, -0.1])                   # origin inside the box
    extra = torch.arange(5000, device="cuda").float().view(-1, 1).repeat(1, 4)
    got = sp.ray_test(o, d, near=near, far=far, rays_h_appear=extra)
    ref = sp.ray_test(o.clone().requires_grad_(True), d, near=near, far=far, rays_h_appear=extra)   # requires_grad -> the torch chain
    assert got["num_rays"] == ref["num_rays"] > 0
    for k in ("rays_inds", "near", "far", "rays_o", "rays_d", "rays_h_appear"):
        assert torch.equal(got[k], ref[k].detach()), k


def test_composite_into_image_buffers():
    from neuralsim_b200.graphics import neus_fused as NF
    rng = np.random.default_rng(5)
    pi = random_packs(rng, 300, 1, 60, "cuda")
    K = int(pi[-1].sum())
    g = torch.Generator("cuda").manual_seed(5)
    alpha0 = (torch.rand(K, device="cuda", generator=g) ** 3).clamp(0, 0.9)
    t = torch.rand(K, device="cuda", generator=g) + 1
    rgb0, nab0 = torch.rand(K, 3, device="cuda", generator=g), torch.randn(K, 3, device="cuda", generator=g)
    n_rays = 1000
    hit = torch.randperm(n_rays, device="cuda")[:300].sort().values
    cot = [torch.randn(s, device="cuda", generator=g) for s in ((n_rays,), (n_rays,), (n_rays, 3), (n_rays, 3))]

    def run(direct):
        a, r, nb = (x.clone().requires_grad_(True) for x in (alpha0, rgb0, nab0))
        if direct:
            _, m, d, c, n_ = NF.composite(a, t, pi, rgb=r, nablas=nb, ray_index=hit, n_rays=n_rays)
        else:
            _, m_, d_, c_, n__ = NF.composite(a, t, pi, rgb=r, nablas=nb)
            z = lambda *s: torch.zeros(*s, device="cuda")
            m, d = z(n_rays).index_put((hit,), m_), z(n_rays).index_put((hit,), d_)
            c, n_ = z(n_rays, 3).index_put((hit,), c_), z(n_rays, 3).index_put((hit,), n__)
        ((m * cot[0]).sum() + (d * cot[1]).sum() + (c * cot[2]).sum() + (n_ * cot[3]).sum()).backward()
        return (m, d, c, n_), (a.grad, r.grad, nb.grad)

    out, grads = run(True)
    out_r, grads_r = run(False)
    for x, y in zip(out + grads, out_r + grads_r):
        assert torch.equal(x, y)


def test_ray_tiled_sdf_query_equals_ray_major(cuda):
    """nsb_fused_sdf_packs (32 rays x 4 samples per tile) returns exactly what nsb_fused_sdf_rays returns, forward and backward."""
    from util import make_pair
    P, model = make_pair(cuda)
    rng = np.random.default_rng(11)
    pi = random_packs(rng, 333, 0, 130, "cuda")            # ragged, includes empty packs, not a multiple of 32 packs
    S = int(pi[-1].sum())
    g = torch.Generator().manual_seed(11)
    R = 500
    ro = (torch.rand(R, 3, generator=g) * 0.2 - 0.1 + torch.tensor([-2.5, 0., 0.])).cuda()
    rd = torch.nn.functional.normalize(torch.tensor([1., 0., 0.]) + 0.3 * torch.randn(R, 3, generator=g), dim=-1).cuda()
    pack_ray = torch.randperm(R, generator=g)[:pi.shape[0]].cuda()
    t = (1.5 + 2.0 * torch.rand(S, generator=g)).cuda()
    ridx = torch.repeat_interleave(pack_ray, pi[:, 1])
    surf = model.implicit_surface
    a = surf.fused_sdf_rays(ridx, t, ro, rd)
    b = surf.fused_sdf_rays(ridx, t, ro, rd, packs=(pi, pack_ray))
    assert torch.equal(a, b)
    ident = torch.arange(pi.shape[0], device="cuda")
    c = surf.fused_sdf_rays(torch.repeat_interleave(ident, pi[:, 1]), t, ro, rd, packs=(pi, None))
    assert torch.equal(c, surf.fused_sdf_rays(torch.repeat_interleave(ident, pi[:, 1]), t, ro, rd))
    w = torch.randn(S, device="cuda") * (torch.rand(S, device="cuda") < 0.3)
    grads = []
    for packs in (None, (pi, pack_ray)):
        model.zero_grad(set_to_none=True)
        s = surf.fused_sdf_rays_autograd(ridx, t, ro, rd, packs=packs)
        (s * w).sum().backward()
        grads.append(surf.encoding.flattened_params.grad.clone())
    assert rel_l2(grads[1], grads[0]) < 1e-6


def test_ray_test_flags_image_ordered_rays(cuda):
    from neuralsim_b200.fields.space import AABBSpace
    from oracle import scene as oscene
    sp = AABBSpace(2.0, device="cuda")
    ro, rd = oscene.pinhole_rays(60, 80, oscene.orbit_camera(1, 8))
    assert sp.ray_test(ro.cuda(), rd.cuda(), near=0.01)["rays_coherent"] is True
    perm = torch.randperm(ro.shape[0])
    assert sp.ray_test(ro[perm].cuda(), rd[perm].cuda(), near=0.01)["rays_coherent"] is False


def test_in_kernel_sample_collection_equals_collect_samples(cuda):
    """nsb_occ_collect: the occupancy evidence the query kernels accumulate == OccGridEma.collect_samples(x, sdf) on the same sdf."""
    from util import make_pair
    from neuralsim_b200.fields import LoTDNeuSModel
    P, model0 = make_pair(cuda)
    model = LoTDNeuSModel(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=P.lotd_cfg)), radiance_cfg=dict(n_appear_embedding=P.n_appear),
                          accel_cfg=dict(resolution=[64, 64, 64], update_from_samples_cfg=dict()), device=cuda)
    model.load_state_dict(model0.state_dict(), strict=False)
    model.train()
    occ = model.accel.occ
    assert occ.should_collect_samples and occ.collect_struct() is not None
    g = torch.Generator().manual_seed(21)
    x = (torch.rand(200_000, 3, generator=g) * 2 - 1).cuda()
    x[:1000] = (torch.rand(1000, 3, generator=g).cuda() - 0.5) * 1.02        # a cluster around the sphere-like surface region
    x[0] = torch.tensor([1.0, -1.0, 1.0])                                   # corners of the box: index clamping
    with torch.no_grad():
        sdf = model.forward_sdf(x)["sdf"]                                    # fused query, collects in-kernel
    got = occ._occ_val_grid_pcl.clone()
    occ._occ_val_grid_pcl.zero_()
    occ.collect_samples(x, val=sdf)                                          # the torch restatement of the reference (accel.py)
    ref = occ._occ_val_grid_pcl.clone()
    assert float(ref.max()) > 0.5 and torch.equal(got, ref)
    # ray-parameterised queries (ray-major and ray-tiled) collect the same evidence as their materialised points
    R = 300
    ro = (torch.tensor([-2.5, 0., 0.]) + 0.1 * torch.randn(R, 3, generator=g)).cuda()
    rd = torch.nn.functional.normalize(torch.tensor([1., 0., 0.]) + 0.2 * torch.randn(R, 3, generator=g), dim=-1).cuda()
    t = (1.6 + 1.8 * torch.rand(R, 40, generator=g)).sort(-1).values.cuda()
    ridx = torch.arange(R, device=cuda)
    pts = torch.addcmul(ro[:, None, :], rd[:, None, :], t[..., None]).reshape(-1, 3)
    grids = []
    for packs in (None, (torch.stack([ridx * 40, torch.full_like(ridx, 40)], 1).contiguous(), None)):
        occ._occ_val_grid_pcl.zero_()
        with torch.no_grad():
            s = model.forward_sdf_on_rays(ridx, t, ro, rd, packs=packs)["sdf"]
        grids.append(occ._occ_val_grid_pcl.clone())
    occ._occ_val_grid_pcl.zero_()
    occ.collect_samples(pts, val=s.reshape(-1))
    assert torch.equal(grids[0], grids[1]) and torch.equal(grids[0], occ._occ_val_grid_pcl)
    model.eval()
    assert occ.collect_struct() is None
