"""The persistent per-ray kernel (csrc/ray_upsample.cu): the no-grad up-sampling half of the NeuS query in ONE launch must give, bit for bit,
the samples the stage kernels give, including rays whose samples do not fit shared memory.  tests/test_ray_upsample_edges_gpu.py pins
it, with its group-to-group state, at its capacity, group and tie edges."""
import pytest
import torch

from oracle import scene as oscene
from util import make_pair

pytestmark = pytest.mark.gpu
NUM_FINE, FACTORS, INV_S = [9, 9, 33], [1, 4, 16], 64.0


def _stage_path(surf, o, d, ridx, ridx_hit, pinfo, t0):
    from neuralsim_b200.graphics import neus_fused as NF
    sdf = surf.fused_sdf_rays(ridx, t0, o, d)
    depth, pi, stages = t0, pinfo, []
    for i, f in enumerate(FACTORS):
        cdf = NF.upsample_cdf(sdf, depth, pi, INV_S * f, True)
        fine = NF.sample_cdf_uniform(depth, cdf, pi, NUM_FINE[i])
        stages.append(fine)
        if i < 2:
            sdf_f = surf.fused_sdf_rays(ridx_hit, fine, o, d).contiguous()
            depth, sdf, pi = NF.merge_sorted_vals(depth, sdf, pi, fine, sdf_f)
    return torch.cat(stages, -1)


@pytest.mark.parametrize("step_size,expect_long", [(0.005, False), (0.0008, True)])
def test_persistent_upsampling_equals_the_stage_kernels(cuda, step_size, expect_long):
    from neuralsim_b200.graphics import neus_fused as NF
    _, model = make_pair(cuda)
    ro, rd = oscene.pinhole_rays(60, 80, oscene.orbit_camera(1, 8))
    rt = model.ray_test(ro.to(cuda), rd.to(cuda), near=0.01)
    o, d = rt["rays_o"].contiguous(), rt["rays_d"].contiguous()
    ridx_hit, pinfo, t0, ridx = NF.march_lean(model.accel.occ.occ_grid, o, d, rt["near"].contiguous(), rt["far"].contiguous(), step_size=step_size, max_steps=4096)
    assert bool((pinfo[:, 1] > 174).any()) == expect_long           # 192 - 18: rays beyond it work in the global scratch
    surf = model.implicit_surface
    with torch.no_grad():
        ref = _stage_path(surf, o, d, ridx, ridx_hit, pinfo, t0)
        grid16, dec = surf._fused_state()
        got, overflow = NF.upsample_rays(surf.encoding.meta, grid16, dec, ridx_hit, pinfo, t0, o, d, [INV_S * f for f in FACTORS], NUM_FINE,
                                         max_level=surf._ml(None), max_steps=4096, use_estimate_alpha=True)
        assert int(overflow.sum()) == 0
        assert torch.equal(got, ref)
        # the shared-memory-only entry point of round 1: long rays are flagged, the others equal
        got0, ov0 = NF.upsample_persistent(surf, ridx_hit, pinfo, t0, o, d, [INV_S * f for f in FACTORS], NUM_FINE, use_estimate_alpha=True)
        ok = ov0 == 0
        assert bool((~ok).any()) == expect_long and torch.equal(got0[ok], ref[ok])


def test_query_with_and_without_the_persistent_kernel(cuda):
    """the whole fused query, persistent kernel on / off: same buffers, same images, same gradients (training mode, sample collection on)"""
    import neuralsim_b200.graphics.neus as GN
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from util import product_grads, rel_l2
    _, model = make_pair(cuda)
    model.accel.occ.should_collect_samples = True
    model.accel.occ.register_buffer("_occ_val_grid_pcl", torch.zeros_like(model.accel.occ.occ_val_grid), persistent=False)
    ro, rd = oscene.pinhole_rays(36, 48, oscene.orbit_camera(2, 8))
    ro, rd, ha = ro.to(cuda), rd.to(cuda), torch.zeros(36 * 48, 4, device=cuda)
    r = SingleVolumeRenderer(dict(near=0.01)).train()
    model.train()
    res = []
    for on in (True, False):
        GN.PERSISTENT_UPSAMPLE = on
        try:
            model.zero_grad(set_to_none=True)
            model.accel.occ._occ_val_grid_pcl.zero_()
            out = r.render(model, ro, rd, rays_h_appear=ha, return_buffer=True)
            sum(v.mean() for v in out["rendered"].values()).backward()
            res.append((out, product_grads(model), model.accel.occ._occ_val_grid_pcl.clone()))
        finally:
            GN.PERSISTENT_UPSAMPLE = "auto"
    (a, ga, pa), (b, gb, pb) = res
    for k in ("t", "opacity_alpha", "rgb", "nablas", "rays_inds_hit", "pack_infos_hit"):
        assert torch.equal(a["volume_buffer"][k], b["volume_buffer"][k]), k
    for k in a["rendered"]:
        assert torch.equal(a["rendered"][k], b["rendered"][k]), k
    assert torch.equal(pa, pb) and float(pa.sum()) > 0                  # the same evidence was collected in-kernel
    for k, v in gb.items():
        if v is not None:
            assert rel_l2(ga[k], v) <= 2e-5, (k, rel_l2(ga[k], v))
