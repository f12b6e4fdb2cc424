"""Generates tests/golden/ref_python.npz by IMPORTING THE REFERENCE'S OWN PYTHON (pure-PyTorch layer of nr3d_lib)
where a checkout of the reference project is found (oracle/build_ref.py: reference_root).  The reference is not part of this repository, so the vectors are committed.

    python tests/golden/make_golden.py

How the reference is imported without its CUDA extensions and without its uninstallable dependencies
(addict, kornia, imageio ... -- SURVEY.md §8c): the packages `nr3d_lib`, `nr3d_lib.graphics`, `.graphics.neus`,
`.graphics.nerf`, `.graphics.pack_ops` are registered as *empty* packages whose __path__ points at the reference tree,
so `import nr3d_lib.graphics.neus.neus_utils` executes the reference FILE but none of the package __init__.py files;
`nr3d_lib.bindings._pack_ops` is served by the CPU oracle backend (oracle/pack_ops.py), `nr3d_lib.maths` by a two-function
stub.  What the vectors therefore pin:
  * reference PyTorch maths executed verbatim: neus_utils.py, nerf_utils.py (ray_*), raysample.py, and the Python side of
    pack_ops.py (autograd rules, merge_* / get_pack_infos_* index algebra);
  * the oracle's kernel restatements only through the reference's own known-answer checks (merge KAT, invert-cdf /
    searchsorted equality, packed-vs-batched vw equality) -- those asserts run here, at generation time.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_root  # noqa: E402

if reference_root() is None:
    raise SystemExit("make_golden.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
REF = os.path.join(reference_root(), "nr3d_lib", "nr3d_lib")


def _pkg(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    sys.modules[name] = m
    return m


def import_reference():
    from oracle import pack_ops as opk
    _pkg("nr3d_lib", REF)
    _pkg("nr3d_lib.graphics", f"{REF}/graphics")
    _pkg("nr3d_lib.graphics.neus", f"{REF}/graphics/neus")
    nerf = _pkg("nr3d_lib.graphics.nerf", f"{REF}/graphics/nerf")
    pko = _pkg("nr3d_lib.graphics.pack_ops", f"{REF}/graphics/pack_ops")
    b = _pkg("nr3d_lib.bindings", "/nonexistent")
    back = types.ModuleType("nr3d_lib.bindings._pack_ops")
    for k in dir(opk.backend):
        if not k.startswith("_"):
            setattr(back, k, getattr(opk.backend, k))
    sys.modules["nr3d_lib.bindings._pack_ops"] = back
    b._pack_ops = back
    maths = types.ModuleType("nr3d_lib.maths")
    maths.logistic_density = lambda x, inv_s: inv_s * torch.sigmoid(x * inv_s) * (1 - torch.sigmoid(x * inv_s))
    sys.modules["nr3d_lib.maths"] = maths
    ref_pack = importlib.import_module("nr3d_lib.graphics.pack_ops.pack_ops")
    for k in ref_pack.__all__:
        setattr(pko, k, getattr(ref_pack, k))
    ref_nerf = importlib.import_module("nr3d_lib.graphics.nerf.nerf_utils")
    for k in ref_nerf.__all__:
        setattr(nerf, k, getattr(ref_nerf, k))
    ref_neus = importlib.import_module("nr3d_lib.graphics.neus.neus_utils")
    ref_rs = importlib.import_module("nr3d_lib.graphics.raysample")
    return ref_pack, ref_nerf, ref_neus, ref_rs


def main():
    P, NF, NU, RS = import_reference()
    rng = np.random.default_rng(1234)
    out = {}
    put = lambda k, v: out.__setitem__(k, v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))

    # ---------------- packs
    n = torch.from_numpy(rng.integers(1, 40, 23)).long()
    pi = P.get_pack_infos_from_n(n)
    S = int(n.sum())
    put("pi", pi)
    put("pi_from_batch", P.get_pack_infos_from_batch(5, 7))
    put("pi_from_first", P.get_pack_infos_from_first(pi[:, 0].contiguous(), S))
    ids = torch.repeat_interleave(torch.arange(23), n)
    put("pi_from_boundary", P.get_pack_infos_from_boundary(P.mark_pack_boundaries(ids)))

    # ---------------- NeuS maths (reference torch code, verbatim)
    depth = P.packed_cumsum(torch.from_numpy(rng.random(S).astype(np.float32)) * 0.02 + 1e-3, pi)
    sdf = torch.from_numpy((0.3 - rng.random(S) * 0.6).astype(np.float32))
    sdf = torch.sort(sdf.view(-1), descending=True).values[torch.argsort(torch.argsort(ids * 1000 - torch.arange(S)))]  # decreasing-ish
    put("neus.depth", depth); put("neus.sdf", sdf)
    for inv_s in (20.0, 64.0, 256.0, 2000.0):
        put(f"neus.packed_alpha.{int(inv_s)}", NU.neus_packed_sdf_to_alpha(sdf, inv_s, pi))
        put(f"neus.upsample_alpha.{int(inv_s)}", NU.neus_packed_sdf_to_upsample_alpha(sdf, depth, inv_s, pi))
    sdf_b = torch.from_numpy((0.2 - rng.random((9, 33)) * 0.4).astype(np.float32))
    t_b = torch.cumsum(torch.from_numpy(rng.random((9, 33)).astype(np.float32)) * 0.03, -1)
    put("neus.sdf_b", sdf_b); put("neus.t_b", t_b)
    put("neus.ray_alpha", NU.neus_ray_sdf_to_alpha(sdf_b, 64.0))
    put("neus.ray_alpha_app1", NU.neus_ray_sdf_to_alpha(sdf_b, 64.0, append_cdf_1=True))
    put("neus.ray_upsample_alpha", NU.neus_ray_sdf_to_upsample_alpha(sdf_b, t_b, 64.0))
    put("neus.ray_vw", NU.neus_ray_sdf_to_vw(sdf_b, 64.0))

    # ---------------- alpha -> weights: packed (oracle kernel) equals batched reference formula (nerf_utils.py:225-277)
    alpha_b = torch.from_numpy((rng.random((11, 29)) ** 2 * 0.5).astype(np.float32))
    vw_b = NF.ray_alpha_to_vw(alpha_b)
    pi_b = P.get_pack_infos_from_batch(11, 29)
    vw_p = NF.packed_alpha_to_vw_v2(alpha_b.flatten(), pi_b, early_stop_eps=0.0, alpha_thre=-1.0)
    assert torch.allclose(vw_p.view(11, 29), vw_b, rtol=1e-5, atol=1e-7), "packed vs batched volume weights"
    put("vw.alpha_b", alpha_b); put("vw.ray_alpha_to_vw", vw_b)
    put("vw.packed_default", NF.packed_alpha_to_vw_v2(alpha_b.flatten(), pi_b))
    nidx, cpi, pidx = P.packed_volume_render_compression(alpha_b.flatten(), pi_b)
    put("vw.compress.nidx", nidx); put("vw.compress.pack_infos", cpi); put("vw.compress.pidx", pidx)

    # ---------------- samplers
    near = torch.from_numpy(rng.random(7).astype(np.float32)); far = near + 1 + torch.from_numpy(rng.random(7).astype(np.float32))
    t, dt = RS.batch_sample_step_linear(near, far, 65, return_dt=True)
    put("rs.near", near); put("rs.far", far); put("rs.linear_t", t); put("rs.linear_dt", dt)
    # reference known-answer example (raysample.py:588-599)
    cdfs = torch.tensor([0.0, 0.1, 0.6, 0.9, 1.0, 0.0, 0.8, 1.0, 0.0, 0.0, 0.5, 1.0])
    bins = torch.tensor([0.0, 0.1, 0.2, 0.3, 0.4, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.3])
    pik = P.get_pack_infos_from_n(torch.tensor([5, 3, 4]))
    u = torch.linspace(0., 1., 42)[1:-1].expand([3, 40]).contiguous()
    ts, i1 = P.packed_invert_cdf(bins, cdfs, u, pik)
    i2 = P.packed_searchsorted(cdfs, u, pik)
    assert torch.equal(i1 - pik[:, 0:1], i2 - pik[:, 0:1]), "invert-cdf bin index == searchsorted (raysample.py:598)"
    put("rs.kat_cdfs", cdfs); put("rs.kat_bins", bins); put("rs.kat_pi", pik); put("rs.kat_samples", ts); put("rs.kat_idx", i1)
    s9, _ = RS.packed_sample_cdf(bins, cdfs, pik, 9)
    put("rs.kat_sample_cdf9", s9)
    w = torch.from_numpy(rng.random((6, 20)).astype(np.float32)); bb = torch.cumsum(torch.from_numpy(rng.random((6, 21)).astype(np.float32)), -1)
    put("rs.pdf_w", w); put("rs.pdf_bins", bb); put("rs.batch_sample_pdf", RS.batch_sample_pdf(bb, w, 12))

    # ---------------- merges (reference Python index algebra over the oracle kernel)
    va = torch.tensor([0.1, 0.2, 0.3, 0.4, 0.5, 0.2, 0.8]); pia = P.get_pack_infos_from_n(torch.tensor([5, 2]))
    vb = torch.tensor([0.0, 0.25, 0.26, 0.6, 0.1, 0.15, 0.3, 0.4]); pib = P.get_pack_infos_from_n(torch.tensor([4, 4]))
    pa, pb, _ = P.merge_two_packs_sorted_aligned(va, pia, vb, pib)
    assert pa.tolist() == [1, 2, 5, 6, 7, 11, 14] and pb.tolist() == [0, 3, 4, 8, 9, 10, 12, 13], "unit_test.py:956-965"
    va = torch.tensor([0.1, 0.2, 0.3, 0.4, 0.5, 11.1, 11.2, 0.2, 0.8]); pia = P.get_pack_infos_from_n(torch.tensor([5, 2, 2]))
    vb = torch.tensor([0.0, 0.25, 0.26, 0.6, 0.1, 0.2, 0.3, 0.4]); pib = P.get_pack_infos_from_n(torch.tensor([4, 4]))
    na, nb = torch.tensor([11, 12, 13]), torch.tensor([11, 13])
    pa, pb, pinf = P.merge_two_packs_sorted_a_includes_b(va, pia, na, vb, pib, nb)
    assert pa.tolist() == [1, 2, 5, 6, 7, 9, 10, 13, 16] and pb.tolist() == [0, 3, 4, 8, 11, 12, 14, 15], "unit_test.py:998-1011"
    assert pinf.tolist() == [[0, 9], [9, 2], [11, 6]]
    # random partial-overlap merge
    na = torch.tensor([0, 2, 3, 7, 9]); nb = torch.tensor([2, 4, 7, 8])
    ca, cb = torch.from_numpy(rng.integers(1, 9, 5)).long(), torch.from_numpy(rng.integers(1, 9, 4)).long()
    pia, pib = P.get_pack_infos_from_n(ca), P.get_pack_infos_from_n(cb)
    va = P.packed_cumsum(torch.from_numpy(rng.random(int(ca.sum())).astype(np.float32)), pia)
    vb = P.packed_cumsum(torch.from_numpy(rng.random(int(cb.sum())).astype(np.float32)), pib)
    pa, pb, pinf = P.merge_two_packs_sorted(va, pia, na, vb, pib, nb)
    for k, v in dict(va=va, pia=pia, na=na, vb=vb, pib=pib, nb=nb, pa=pa, pb=pb, pinf=pinf).items():
        put(f"merge_sorted.{k}", v)
    A = torch.sort(torch.from_numpy(rng.random((6, 9)).astype(np.float32)), -1).values
    Bv = torch.sort(torch.from_numpy(rng.random((3, 5)).astype(np.float32)), -1).values
    nA, nB = torch.arange(6), torch.tensor([1, 2, 5])
    pa, pb, pinf = P.merge_two_batch_a_includes_b(A, nA, Bv, nB)
    for k, v in dict(A=A, B=Bv, nA=nA, nB=nB, pa=pa, pb=pb, pinf=pinf).items():
        put(f"merge_batch.{k}", v)

    # ---------------- autograd rules of the reference wrappers
    f = torch.from_numpy(rng.normal(size=(S, 2)).astype(np.float32)).requires_grad_(True)
    wts = torch.from_numpy(rng.normal(size=(S, 2)).astype(np.float32))
    for name, fn in (("sum", lambda x: P.packed_sum(x, pi)), ("cumsum_excl", lambda x: P.packed_cumsum(x, pi, exclusive=True))):
        y = fn(f)
        g, = torch.autograd.grad((y * (wts if y.shape[0] == S else wts[:y.shape[0]])).sum(), f)
        put(f"grad.{name}.y", y); put(f"grad.{name}.g", g)
    f1d = f[:, 0].contiguous().detach().requires_grad_(True)   # the reference's diff adjoints handle 1-D features only (pack_ops.py:216)
    for name, fn in (("diff", lambda x: P.packed_diff(x, pi)), ("bdiff", lambda x: P.packed_backward_diff(x, pi))):
        y = fn(f1d)
        g, = torch.autograd.grad((y * wts[:, 0]).sum(), f1d)
        put(f"grad.{name}.y", y); put(f"grad.{name}.g", g)
    put("grad.f", f); put("grad.w", wts)
    other = (torch.from_numpy(rng.random(23).astype(np.float32)) + 0.5).requires_grad_(True)
    f1 = f[:, 0].contiguous().detach().requires_grad_(True)
    y = P.packed_div(f1, other, pi)
    gi, go = torch.autograd.grad((y * wts[:, 0]).sum(), [f1, other])
    put("grad.div.other", other); put("grad.div.y", y); put("grad.div.gi", gi); put("grad.div.go", go)
    al = (torch.from_numpy(rng.random(S).astype(np.float32)) * 0.4).requires_grad_(True)
    vw = P.packed_alpha_to_vw(al, pi)
    ga, = torch.autograd.grad((vw * wts[:, 0]).sum(), al)
    put("grad.a2vw.alpha", al); put("grad.a2vw.vw", vw); put("grad.a2vw.g", ga)

    path = os.path.join(ROOT, "tests", "golden", "ref_python.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
