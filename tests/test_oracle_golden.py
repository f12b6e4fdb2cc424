"""CPU: the oracle against (i) vectors produced by the reference's own Python (tests/golden/ref_python.npz, generator:
tests/golden/make_golden.py), (ii) the reference tests' known-answer vectors, (iii) maths properties of the LoTD restatement."""
import os

import numpy as np
import pytest
import torch

from oracle import lotd as olotd
from oracle import pack_ops as opk
from oracle import render as orender

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_python.npz"))
T = lambda k: torch.from_numpy(G[k])


def test_pack_infos_builders():
    n = T("pi")[:, 1]
    assert torch.equal(orender.get_pack_infos_from_n(n), T("pi"))
    assert torch.equal(orender.get_pack_infos_from_batch(5, 7), T("pi_from_batch"))
    assert torch.equal(T("pi_from_first"), T("pi")) and torch.equal(T("pi_from_boundary"), T("pi"))


@pytest.mark.parametrize("inv_s", [20, 64, 256, 2000])
def test_neus_alpha_matches_reference_python(inv_s):
    pi, sdf, depth = T("pi"), T("neus.sdf"), T("neus.depth")
    assert torch.allclose(orender.neus_packed_sdf_to_alpha(sdf, float(inv_s), pi), T(f"neus.packed_alpha.{inv_s}"), rtol=1e-6, atol=1e-7)
    assert torch.allclose(orender.neus_packed_sdf_to_upsample_alpha(sdf, depth, float(inv_s), pi), T(f"neus.upsample_alpha.{inv_s}"), rtol=1e-6, atol=1e-7)


def test_alpha_to_vw_and_compression_match_reference():
    a = T("vw.alpha_b")
    pi = orender.get_pack_infos_from_batch(*a.shape)
    assert torch.allclose(orender.packed_alpha_to_vw(a.flatten(), pi), T("vw.packed_default"), rtol=1e-6, atol=1e-8)
    # batched reference formula == packed kernel without early stop / threshold (nerf_utils.py:225-277)
    w = opk.packed_alpha_to_vw_forward(a.flatten(), pi, 0.0, -1.0, False)[0]
    assert torch.allclose(w.view(a.shape), T("vw.ray_alpha_to_vw"), rtol=1e-5, atol=1e-7)
    nidx, cpi, pidx = orender.packed_volume_render_compression(a.flatten(), pi)
    assert torch.equal(nidx, T("vw.compress.nidx")) and torch.equal(cpi, T("vw.compress.pack_infos")) and torch.equal(pidx, T("vw.compress.pidx"))


def test_samplers_match_reference():
    t, dt = orender.batch_sample_step_linear(T("rs.near"), T("rs.far"), 65)
    assert torch.equal(t, T("rs.linear_t")) and torch.allclose(dt, T("rs.linear_dt"))
    s, i = opk.packed_invert_cdf(T("rs.kat_bins"), T("rs.kat_cdfs"), torch.linspace(0., 1., 42)[1:-1].expand(3, 40).contiguous(), T("rs.kat_pi"))
    assert torch.equal(s, T("rs.kat_samples")) and torch.equal(i, T("rs.kat_idx"))
    assert torch.equal(orender.packed_sample_cdf(T("rs.kat_bins"), T("rs.kat_cdfs"), T("rs.kat_pi"), 9)[0], T("rs.kat_sample_cdf9"))
    # expected behaviour spelled out in raysample.py:592-596
    assert float(((s[0] > 0.1) & (s[0] < 0.2)).float().mean()) > 0.4 and float((s[2] < 0.1).float().sum()) == 0


def test_reference_known_answer_vectors():
    """pack_ops/unit_test.py:956-965 and :533-564 (exclusive-scan semantics)."""
    from_n = lambda n: orender.get_pack_infos_from_n(torch.tensor(n))
    a, b, p = opk.try_merge_two_packs_sorted_aligned(torch.tensor([0.1, 0.2, 0.3, 0.4, 0.5, 0.2, 0.8]), from_n([5, 2]),
                                                     torch.tensor([0.0, 0.25, 0.26, 0.6, 0.1, 0.15, 0.3, 0.4]), from_n([4, 4]), True)
    assert a.tolist() == [1, 2, 5, 6, 7, 11, 14] and b.tolist() == [0, 3, 4, 8, 9, 10, 12, 13] and p.tolist() == [[0, 9], [9, 6]]
    f = torch.tensor([0.8750, 0.0581, 0.9378, 0.9638, 0.9859, 0.4652, 0.9105, 0.5071, 0.0173, 0.6071, 0.7123, 0.7371, 0.8094])
    pi = from_n([4, 7, 2])
    inc = torch.tensor([0.8750, 0.9331, 1.8709, 2.8347, 0.9859, 1.4512, 2.3617, 2.8688, 2.8860, 3.4931, 4.2054, 0.7371, 1.5465])
    exc = torch.tensor([0.0, 0.8750, 0.9331, 1.8709, 0.0, 0.9859, 1.4512, 2.3617, 2.8688, 2.8860, 3.4931, 0.0, 0.7371])
    assert torch.allclose(opk.packed_cumsum(f, pi, False, False), inc, atol=2e-4)
    assert torch.allclose(opk.packed_cumsum(f, pi, True, False), exc, atol=2e-4)
    assert float(opk.packed_cumprod(f, pi, True, False).abs().sum()) == 0.0       # reference quirk (SURVEY §8a note)


def test_merges_match_reference_python():
    pa, pb, pinf = orender.merge_two_batch_a_includes_b(T("merge_batch.A"), T("merge_batch.nA"), T("merge_batch.B"), T("merge_batch.nB"))
    assert torch.equal(pa, T("merge_batch.pa")) and torch.equal(pb, T("merge_batch.pb")) and torch.equal(pinf, T("merge_batch.pinf"))


def test_reference_autograd_rules_are_the_true_adjoints():
    """The oracle uses plain differentiable torch for sum / cumsum / diff / div; the reference hand-writes the adjoints."""
    pi, f, w = T("pi"), T("grad.f"), T("grad.w")
    pidx = torch.repeat_interleave(torch.arange(pi.shape[0]), pi[:, 1])
    x = f.clone().requires_grad_(True)
    y = orender.packed_sum(x, pi)
    g, = torch.autograd.grad((y * w[:y.shape[0]]).sum(), x)
    assert torch.allclose(y, T("grad.sum.y"), rtol=1e-5, atol=1e-5) and torch.allclose(g, T("grad.sum.g"))
    x1 = f[:, 0].clone().requires_grad_(True)
    y = orender.packed_diff(x1, pi)
    g, = torch.autograd.grad((y * w[:, 0]).sum(), x1)
    assert torch.equal(y, T("grad.diff.y")) and torch.allclose(g, T("grad.diff.g"), atol=1e-6)
    al = T("grad.a2vw.alpha").clone().requires_grad_(True)
    vw = orender.packed_alpha_to_vw(al, pi)
    g, = torch.autograd.grad((vw * w[:, 0]).sum(), al)
    assert torch.allclose(vw, T("grad.a2vw.vw")) and torch.allclose(g, T("grad.a2vw.g"), rtol=1e-5, atol=1e-6)


def test_lotd_meta_and_index_math():
    cfg = olotd.gen_ngp_cfg()
    assert cfg["lod_res"] == [16, 22, 30, 42, 58, 80, 111, 154, 212, 294, 406, 561, 776, 1073, 1483, 2049]     # SURVEY §8 header
    assert cfg["lod_types"] == ["Dense"] * 6 + ["Hash"] * 10
    m = olotd.LoDMeta(3, **cfg)
    assert m.n_params == 12131648 and m.n_encoded_dims == 32
    cell = np.array([[1, 2, 3]], dtype=np.uint32)
    assert olotd.grid_index(m, 0, cell)[0] == (1 * 16 + 2) * 16 + 3                                          # z fastest
    assert olotd.grid_index(m, 15, cell)[0] == ((1 * 1) ^ (2 * 2654435761 % 2**32) ^ (3 * 805459861 % 2**32)) % 2**19


def test_lotd_gradcheck_style_properties():
    """The recipes of lotd/tests/math_test.py:99-171 (gradcheck of y wrt x and grid, of dL_dx wrt dL_dy and grid) as
    finite-difference / adjoint identities on a small fp32 table."""
    from util import small_lotd_cfg
    m = olotd.LoDMeta(3, **small_lotd_cfg())
    rng = np.random.default_rng(0)
    p = rng.uniform(-0.1, 0.1, m.n_params).astype(np.float32)
    x = rng.uniform(0.05, 0.95, (400, 3)).astype(np.float32)
    y, J = olotd.lod_fwd(m, x, p, need_input_grad=True)
    eps = 1e-4
    for d in range(3):                                            # dy/dx by central differences (away from cell borders in the median)
        xp, xm = x.copy(), x.copy(); xp[:, d] += eps; xm[:, d] -= eps
        fd = (olotd.lod_fwd(m, xp, p)[0].astype(np.float64) - olotd.lod_fwd(m, xm, p)[0]) / (xp[:, d] - xm[:, d])[:, None].astype(np.float64)
        assert np.median(np.abs(fd - J[:, :, d])) < 2e-3
    g = rng.normal(size=y.shape).astype(np.float32)
    gp = olotd.lod_bwd_grid(m, g, x, m.n_params)                  # y is linear in the table: <g, y(p)> == <dL_dp, p>
    assert abs((gp * p).sum() - (g.astype(np.float64) * y).sum()) < 1e-6 * np.abs(gp * p).sum() + 1e-6
    gin = rng.normal(size=x.shape).astype(np.float32)
    a, b, _ = olotd.lod_bwd_bwd_input(m, gin, g, x, p, J)         # dL_dx = J^T g is bilinear in (g, p)
    dLdx = olotd.lod_bwd_input(g, J)
    lhs = (gin.astype(np.float64) * dLdx).sum()
    assert abs(lhs - (b * p).sum()) < 1e-5 * abs(lhs) and abs(lhs - (a.astype(np.float64) * g).sum()) < 1e-5 * abs(lhs)
    z, _ = olotd.lod_fwd(m, x, p, max_level=-1)
    assert np.abs(z).sum() == 0                                   # lotd_torch_api.cu:294-297


_CUBOID_3D = dict(lod_res=[[6, 11, 4], [10, 17, 6], [17, 29, 9], [29, 49, 15]], lod_n_feats=[2, 4, 2, 2], lod_types=["Dense"] * 2 + ["Hash"] * 2,
                  hashmap_size=3001)
_TABLE_4D = dict(lod_res=[[6, 6, 6, 4], [9, 9, 9, 6], [13, 13, 13, 8], [20, 20, 20, 12], [7, 11, 5, 4]], lod_n_feats=[2] * 5,
                 lod_types=["Dense", "Dense", "Hash", "Hash", "Dense"], hashmap_size=2 ** 12)


@pytest.mark.parametrize("D, cfg", [(3, _CUBOID_3D), (4, _TABLE_4D)], ids=["cuboid3d", "4d"])
def test_lotd_adjoint_identities_cuboid_and_4d(D, cfg):
    """The adjoint identities of test_lotd_gradcheck_style_properties on a cuboid 3-D table (with a 4-wide level and a hash size that is
    not a power of two) and on the 4-D table of the distant model with a level that is cuboid in x / y / z.  A dense level also has to
    address every cell of its [rx, ry, rz(, rw)] box exactly once."""
    m = olotd.LoDMeta(D, **cfg)
    rng = np.random.default_rng(1)
    p = rng.uniform(-0.1, 0.1, m.n_params).astype(np.float32)
    x = rng.uniform(1e-6, 1 - 1e-6, (3000, D)).astype(np.float32)
    y, J = olotd.lod_fwd(m, x, p, need_input_grad=True)
    g = rng.normal(size=y.shape).astype(np.float32)
    gp = olotd.lod_bwd_grid(m, g, x, m.n_params)                  # <g, y(p)> == <dL_dp, p>
    assert abs((gp * p).sum() - (g.astype(np.float64) * y).sum()) < 1e-6 * np.abs(gp * p).sum() + 1e-6
    gin = rng.normal(size=x.shape).astype(np.float32)
    a, b, _ = olotd.lod_bwd_bwd_input(m, gin, g, x, p, J)         # dL_dx = J^T g is bilinear in (g, p)
    lhs = (gin.astype(np.float64) * olotd.lod_bwd_input(g, J)).sum()
    assert abs(lhs - (b * p).sum()) < 1e-5 * abs(lhs) and abs(lhs - (a.astype(np.float64) * g).sum()) < 1e-5 * abs(lhs)
    eps = 1e-4
    for d in range(D):                                            # dy/dx along each axis by central differences
        xp, xm = x.copy(), x.copy(); xp[:, d] += eps; xm[:, d] -= eps
        fd = (olotd.lod_fwd(m, xp, p)[0].astype(np.float64) - olotd.lod_fwd(m, xm, p)[0]) / (xp[:, d] - xm[:, d])[:, None].astype(np.float64)
        assert np.median(np.abs(fd - J[:, :, d])) < 2e-3, d
    for lvl, res in enumerate(m.level_res_multidim):
        if m.level_types[lvl] == olotd.DENSE:
            cells = np.stack(np.meshgrid(*[np.arange(r, dtype=np.uint32) for r in res], indexing="ij"), -1).reshape(-1, D)
            assert np.array_equal(np.sort(olotd.grid_index(m, lvl, cells)), np.arange(m.level_sizes[lvl]))


def test_cfg1_sphere_pure_torch_cpu():
    """BASELINE.json configs[0]: analytic sphere, 64x64 rays, 32 samples -- the reference's pure-PyTorch CPU path."""
    from oracle import scene
    out, loss, n = scene.sphere_cfg1_forward_backward()
    assert 1000 < n <= 64 * 64 and torch.isfinite(loss)            # rays of the 64x64 image that cross the [-1,1]^3 box
    hit = out["mask_volume"] > 0.5
    assert 0.02 < float(hit.float().mean()) < 0.5                 # the r=0.5 sphere seen from 4 units away
    assert abs(float(out["depth_volume"][hit].min()) - 3.5) < 0.1


def test_threaded_level_walk_equals_serial():
    """oracle/lotd.py walks the independent levels on a thread pool for large inputs: same bits as the serial walk."""
    from oracle import lotd as olotd
    cfg = dict(lod_res=[8, 12, 18, 24, 40, 64, 100, 160], lod_n_feats=[2] * 8, lod_types=["Dense"] * 4 + ["Hash"] * 4, hashmap_size=2 ** 14)
    meta = olotd.LoDMeta(3, **cfg)
    rng = np.random.default_rng(5)
    p = rng.uniform(-0.1, 0.1, meta.n_params).astype(np.float16)
    x = rng.uniform(1e-6, 1 - 1e-6, (6000, 3)).astype(np.float32)
    g = rng.standard_normal((6000, meta.n_encoded_dims)).astype(np.float32)
    out = {}
    for nt in (1, 8):
        olotd.THREADS[0] = nt
        try:
            y, d = olotd.lod_fwd(meta, x, p, None, True)
            gr = olotd.lod_bwd_grid(meta, g, x, meta.n_params)
        finally:
            olotd.THREADS[0] = None
        out[nt] = (y, d, gr)
    for a, b in zip(out[1], out[8]):
        assert np.array_equal(a, b)
