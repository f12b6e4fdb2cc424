"""GPU: our kernels AND the CPU oracle against the REFERENCE'S OWN CUDA kernels (oracle/_ref, compiled by oracle/build_ref.py), whose
outputs on these inputs are stored under tests/golden/ref_*.npz (tests/refgold.py: digests for the bit-exact checks, values for the others).
This is what pins the oracle for the parts the reference ships no fixtures for: LoTD, marching, alpha compositing."""
import numpy as np
import pytest
import torch

from refgold import Golden

pytestmark = pytest.mark.gpu


def _rows(t, n):
    return t.detach().reshape(t.shape[0], -1)[:n].cpu()


def _support_sample(t, n, seed):
    """a fixed sample of the non-zero entries of a large gradient (indices chosen from the reference's support)"""
    nz = torch.nonzero(t.detach().reshape(-1).float() != 0).squeeze(-1).cpu()
    g = torch.Generator().manual_seed(seed)
    return nz[torch.randperm(nz.numel(), generator=g)[:n]].sort().values


def test_lotd_against_reference_kernels(cuda):
    from oracle import lotd as olotd
    from neuralsim_b200.bindings import _lotd as ours
    G = Golden("_lotd")
    cfg = olotd.gen_ngp_cfg()
    rmeta = lambda ref: ref.LoDMeta(3, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"], False)
    om = ours.LoDMeta(3, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"])
    cm = olotd.LoDMeta(3, **cfg)
    sizes = G.value("meta", lambda ref: torch.tensor([rmeta(ref).n_params] + list(rmeta(ref).level_offsets) + list(rmeta(ref).level_sizes)))
    assert sizes.tolist() == [om.n_params] + list(om.level_offsets) + list(om.level_sizes)
    rng = np.random.default_rng(0)
    p = torch.from_numpy(rng.uniform(-0.1, 0.1, om.n_params).astype(np.float16)).to(cuda)
    x = torch.from_numpy(rng.uniform(1e-6, 1 - 1e-6, (60000, 3)).astype(np.float32)).to(cuda)
    g = torch.from_numpy((rng.normal(size=(60000, 32)) * 0.05).astype(np.float16)).to(cuda)
    gin = torch.from_numpy(rng.normal(size=(60000, 3)).astype(np.float32)).to(cuda)
    ref_fwd = lambda ref: ref.lod_fwd(rmeta(ref), x, p, None, None, None, None, True)
    y_o, d_o = ours.lod_fwd(om, x, p, None, None, None, None, True)
    G.equal("y", y_o.view(torch.int16), lambda ref: ref_fwd(ref)[0].contiguous().view(torch.int16))       # features: bit-exact
    d_r = G.value("d_rows", lambda ref: _rows(ref_fwd(ref)[1].reshape(d_o.shape), 600))
    assert torch.allclose(d_r, _rows(d_o, 600), rtol=1e-6, atol=1e-7)
    y_c, d_c = olotd.lod_fwd(cm, x[:5000].cpu().numpy(), p.cpu().numpy(), need_input_grad=True)   # the CPU oracle, same check
    G.equal("y5000", torch.from_numpy(np.ascontiguousarray(y_c)).reshape(5000, -1).view(torch.int16),
            lambda ref: ref_fwd(ref)[0].contiguous()[:5000].reshape(5000, -1).view(torch.int16))
    assert np.allclose(d_c.reshape(5000, -1)[:600], d_r.reshape(600, -1).numpy(), rtol=1e-6, atol=1e-7)
    for ml in (7, 0):
        b, _ = ours.lod_fwd(om, x, p, None, None, None, ml, False)
        G.equal(f"y_max_level{ml}", b.view(torch.int16), lambda ref: ref.lod_fwd(rmeta(ref), x, p, None, None, None, ml, False)[0].contiguous().view(torch.int16))
    # gradients: the reference accumulates with fp16 atomics (order dependent, saturating); ours in fp32 -> tolerance
    ref_bwd = lambda ref: ref.lod_bwd(rmeta(ref), g, x, p, ref_fwd(ref)[1], None, None, None, None, True, True)
    gx_o, gp_o = ours.lod_bwd(om, g, x, p, d_o, None, None, None, None, True, True)
    gx_r = G.value("gx_rows", lambda ref: _rows(ref_bwd(ref)[0], 8000))
    assert torch.allclose(gx_r, _rows(gx_o, 8000), rtol=1e-4, atol=1e-4)
    idx = G.value("gp_idx", lambda ref: _support_sample(ref_bwd(ref)[1], 20000, 1))
    gp_r = G.value("gp_sample", lambda ref: ref_bwd(ref)[1].reshape(-1)[idx.to(cuda)])
    gp_s = gp_o.reshape(-1)[idx.to(cuda)].float().cpu()
    err = float((gp_r.float() - gp_s).norm() / gp_s.norm())
    assert err < 2e-2, err
    ref_bb = lambda ref: ref.lod_bwd_bwd_input(rmeta(ref), gin, g, x, p, ref_fwd(ref)[1].contiguous(), None, None, None, None, True, True, False)
    a_o, b_o, _ = ours.lod_bwd_bwd_input(om, gin, g, x, p, d_o, None, None, None, None, True, True, False)
    a_r = G.value("a_rows", lambda ref: _rows(ref_bb(ref)[0], 4000))
    a_s = _rows(a_o, 4000)
    assert float((a_r.float() - a_s.float()).norm() / a_s.float().norm()) < 5e-3
    bidx = G.value("b_idx", lambda ref: _support_sample(ref_bb(ref)[1], 20000, 2))
    b_r = G.value("b_sample", lambda ref: ref_bb(ref)[1].reshape(-1)[bidx.to(cuda)])
    b_s = b_o.reshape(-1)[bidx.to(cuda)].float().cpu()
    assert float((b_r.float() - b_s).norm() / b_s.norm()) < 5e-2
    G.save()


@pytest.mark.parametrize("dt_gamma", [0.0, 0.01])
def test_marching_against_reference_kernels(cuda, dt_gamma):
    from oracle import march as omarch, render as orender, scene as oscene
    from neuralsim_b200.bindings import _occ_grid as ours
    G = Golden(f"_occ_grid_dt{dt_gamma}", "_occ_grid")
    os_, ds_ = [], []
    for k in range(4):
        o, d = oscene.pinhole_rays(60, 80, oscene.orbit_camera(k, 4, radius=2.5 + 0.3 * k, elev_deg=10 + 15 * k))
        os_.append(o); ds_.append(d)
    rt = orender.ray_test(torch.cat(os_), torch.cat(ds_), near=0.01)
    o, d, near, far = (rt[k].contiguous() for k in ("rays_o", "rays_d", "near", "far"))
    rng = np.random.default_rng(1)
    for gi, grid in enumerate((oscene.make_occ_grid(64), torch.from_numpy(rng.random((48, 32, 40)) < 0.1))):
        roi = torch.tensor([-1., -1, -1, 1, 1, 1])
        args = (o.to(cuda), d.to(cuda), near.to(cuda), far.to(cuda), roi.to(cuda), grid.to(cuda))
        ref_march = lambda ref: ref.ray_marching(*args, ref.ContractionType.AABB, 0.005, 0.1, dt_gamma, 1024, True)
        g = ours.ray_marching(*args, ours.ContractionType.AABB, 0.005, 0.1, dt_gamma, 1024, True)
        for k, b in enumerate(g):                                      # counts, t_starts, t_ends, ridx, gidx: bit-exact
            G.equal(f"grid{gi}.out{k}", b, lambda ref: ref_march(ref)[k])
        c = omarch.ray_marching(o, d, near, far, roi, grid, 0.005, 0.1, dt_gamma, 1024)            # and the C oracle
        G.equal(f"grid{gi}.out0", c[0], lambda ref: ref_march(ref)[0])
        G.equal(f"grid{gi}.t_starts_flat", c[1], lambda ref: ref_march(ref)[1].squeeze(-1))
        G.equal(f"grid{gi}.out4", c[4], lambda ref: ref_march(ref)[4])
        assert int(g[0][:, 1].sum()) > 1000
    G.save()


def test_pack_ops_against_reference_kernels(cuda):
    from oracle import pack_ops as opk
    from neuralsim_b200.bindings import _pack_ops as ours
    from util import random_packs
    G = Golden("_pack_ops")
    rng = np.random.default_rng(2)
    tg = torch.Generator().manual_seed(2)
    pi = random_packs(rng, 500, 1, 140).to(cuda)
    S = int(pi[:, 1].sum())
    f = torch.from_numpy(rng.normal(size=(S, 3)).astype(np.float32)).to(cuda)
    assert torch.allclose(G.value("sum", lambda ref: ref.packed_sum(f, pi)), ours.packed_sum(f, pi).cpu(), rtol=1e-5, atol=1e-5)
    for ex in (False, True):
        for rev in (False, True):
            r = G.value(f"cumsum{int(ex)}{int(rev)}_rows", lambda ref: _rows(ref.packed_cumsum(f, pi, ex, rev), 4000))
            assert torch.allclose(r, _rows(ours.packed_cumsum(f, pi, ex, rev), 4000), rtol=1e-5, atol=2e-5)
    G.equal("diff", ours.packed_diff(f, pi, None, None), lambda ref: ref.packed_diff(f, pi, None, None))
    G.equal("backward_diff", ours.packed_backward_diff(f, pi, None, None), lambda ref: ref.packed_backward_diff(f, pi, None, None))
    o = torch.from_numpy((rng.random((500, 3)) + 1).astype(np.float32)).to(cuda)
    G.equal("div", ours.packed_div(f, o, pi), lambda ref: ref.packed_div(f, o, pi))
    G.equal("add", ours.packed_add(f, o, pi), lambda ref: ref.packed_add(f, o, pi))
    a = torch.from_numpy((rng.random(S) ** 3).astype(np.float32))
    a[torch.rand(S, generator=tg) < 0.3] = 0
    a[torch.rand(S, generator=tg) < 0.02] = 0.999
    a = a.to(cuda)
    w_o = ours.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, False)[0]
    G.equal("vw", w_o, lambda ref: ref.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, False)[0])          # the serial recurrence: bit-exact
    G.equal("vw", opk.packed_alpha_to_vw_forward(a.cpu(), pi.cpu(), 1e-4, 0.0, False)[0], lambda ref: ref.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, False)[0])
    _, info_o, sel_o = ours.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, True)
    G.equal("vw_info", info_o, lambda ref: ref.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, True)[1].long())
    G.equal("vw_sel", sel_o, lambda ref: ref.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, True)[2])
    gw = torch.randn(S, generator=tg).to(cuda)
    ga_r = G.value("vw_backward", lambda ref: ref.packed_alpha_to_vw_backward(ref.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, False)[0], gw, a, pi, 1e-4, 0.0))
    ga_o = ours.packed_alpha_to_vw_backward(w_o, gw, a, pi, 1e-4, 0.0).cpu()
    assert float((ga_r - ga_o).norm() / ga_r.norm()) < 1e-4
    cdf = ours.packed_cumsum(a, pi, True, False)
    cdf = ours.packed_div(cdf, cdf[pi[:, 0] + pi[:, 1] - 1].clamp_min(1e-5).contiguous(), pi)
    bins = ours.packed_cumsum(torch.rand(S, generator=tg).to(cuda), pi, False, False)
    u = torch.linspace(0, 1, 35, device=cuda)[1:-1].expand(500, 33).contiguous()
    s_o, i_o = ours.packed_invert_cdf(bins, cdf, u, pi)
    G.equal("invert_cdf_idx", i_o, lambda ref: ref.packed_invert_cdf(bins, cdf, u, pi)[1])
    G.equal("invert_cdf_samples", s_o, lambda ref: ref.packed_invert_cdf(bins, cdf, u, pi)[0])
    G.equal("searchsorted", ours.packed_searchsorted(cdf, u, pi), lambda ref: ref.packed_searchsorted(cdf, u, pi))
    pib = random_packs(rng, 500, 1, 40).to(cuda)
    vb = ours.packed_cumsum(torch.rand(int(pib[:, 1].sum()), generator=tg).to(cuda), pib, False, False)
    for b_sorted in (True, False):
        g = ours.try_merge_two_packs_sorted_aligned(bins, pi, vb, pib, b_sorted)
        for k, y in enumerate(g):
            G.equal(f"merge{int(b_sorted)}.{k}", y, lambda ref: ref.try_merge_two_packs_sorted_aligned(bins, pi, vb, pib, b_sorted)[k])
    n = pi[:, 1].contiguous()
    for k, y in enumerate(ours.interleave_arange(n, True)):
        G.equal(f"interleave_arange.{k}", y, lambda ref: ref.interleave_arange(n, True)[k])
    st, step = torch.randn(500, generator=tg).to(cuda), torch.rand(500, generator=tg).to(cuda)
    for k, y in enumerate(ours.interleave_linstep(st, n, step, True)):
        G.equal(f"interleave_linstep.{k}", y, lambda ref: ref.interleave_linstep(st, n, step, True)[k])
    v = torch.randn(S, generator=tg).to(cuda)
    v2 = v.clone()
    i2 = ours.packed_sort_qsort(v2, pi, True)

    def ref_sort(ref):
        v1 = v.clone()
        return v1, ref.packed_sort_qsort(v1, pi, True)
    G.equal("qsort_values", v2, lambda ref: ref_sort(ref)[0])
    G.equal("qsort_gathered", v[i2], lambda ref: v[ref_sort(ref)[1]])                   # quicksort is unstable: compare values
    ids = torch.repeat_interleave(torch.arange(500, device=cuda), n)
    G.equal("pack_boundaries", ours.mark_pack_boundaries_cuda(ids), lambda ref: ref.mark_pack_boundaries_cuda(ids))
    G.save()


def test_shencoder_against_reference_kernel(cuda):
    from neuralsim_b200.bindings import _shencoder as ours
    G = Golden("_shencoder")
    tg = torch.Generator().manual_seed(4)
    N = 2000
    v = torch.nn.functional.normalize(torch.randn(N, 3, generator=tg), dim=-1).to(cuda)

    def ref_fwd(ref, C):
        out_r, j_r = torch.empty(N, C * C, device=cuda), torch.empty(N, 3 * C * C, device=cuda)
        ref.sh_encode_forward(v, out_r, N, 3, C, True, j_r)
        torch.cuda.synchronize()                                         # the reference launches on the default stream
        return out_r, j_r

    def ref_bwd(ref, C, g):
        gi_r = torch.zeros(N, 3, device=cuda)
        ref.sh_encode_backward(g, v, N, 3, C, ref_fwd(ref, C)[1], gi_r)
        torch.cuda.synchronize()
        return gi_r
    for C in (1, 2, 3, 4):
        out_o, j_o = torch.empty(N, C * C, device=cuda), torch.empty(N, 3 * C * C, device=cuda)
        ours.sh_encode_forward(v, out_o, N, 3, C, True, j_o)
        out_r = G.value(f"out{C}", lambda ref: ref_fwd(ref, C)[0])
        j_r = G.value(f"jac{C}_rows", lambda ref: _rows(ref_fwd(ref, C)[1], 800))
        assert torch.allclose(out_r, out_o.cpu(), rtol=1e-6, atol=1e-7) and torch.allclose(j_r, _rows(j_o, 800), rtol=1e-5, atol=1e-6)
        g = torch.randn(N, C * C, generator=tg).to(cuda)
        gi_o = torch.zeros(N, 3, device=cuda)
        ours.sh_encode_backward(g, v, N, 3, C, j_o, gi_o)
        gi_r = G.value(f"grad{C}", lambda ref: ref_bwd(ref, C, g))
        assert torch.allclose(gi_r, gi_o.cpu(), rtol=1e-4, atol=1e-5)
    G.save()
