"""oracle/glue.py pinned on the CPU, so that the GPU tests of csrc/neus_glue.cu (tests/test_glue_edges_gpu.py) do not compare the
kernels with a second opinion of the same author: the merge against oracle/pack_ops.py (itself pinned to the reference's kernel) and
the reference's known-answer vector, the boundary assembly against a serial k-way merge, numpy's stable sort and the reference
Python's stored merge_two_batch_a_includes_b, the slab test against float64, the scan against a loop, the derived sizes by hand."""
import os

import numpy as np
import torch

from oracle import glue as G
from oracle import pack_ops as opk

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_python.npz")


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def test_scan_counts_equals_a_loop():
    rng = np.random.default_rng(0)
    for n in (0, 1, 2, 9, 1000):
        c = (rng.integers(0, 7, n) * (rng.random(n) < 0.4)).astype(np.int32)
        src = np.arange(n) * 3 + 1
        s = G.scan_counts(c, src)
        run, first, nz = 0, [], []
        for i, v in enumerate(c):
            first.append(run)
            if v > 0:
                nz.append((i, run, int(v)))
            run += int(v)
        assert s["totals"] == (run, len(nz))
        assert s["first"].dtype == np.int32 and s["first"].tolist() == first
        assert s["info2"].tolist() == [[f, int(v)] for f, v in zip(first, c)]
        assert s["nz_index"].dtype == np.int64 and s["nz_index"].tolist() == [i for i, _, _ in nz] == np.nonzero(c)[0].tolist()
        assert s["nz_pack"].reshape(-1, 2).tolist() == [[f, v] for _, f, v in nz]
        assert s["nz_src"].tolist() == [3 * i + 1 for i, _, _ in nz]
        assert np.array_equal(s["first"], np.cumsum(c, dtype=np.int64) - c)


def test_scan_counts_carries_64_bits():
    c = np.full(1_100_000, 2047, np.int32)                                # sum = 2.25e9 > 2^31
    s = G.scan_counts(c)
    assert s["totals"] == (2047 * c.size, c.size)
    assert s["nz_pack"][-1].tolist() == [2047 * (c.size - 1), 2047]       # int64 by contract
    assert s["first"][-1] == np.int64(2047 * (c.size - 1)).astype(np.int32) < 0     # the int32 output has wrapped


def _merge_case(rng, lens, nb, ties):
    P = len(lens)
    first = np.cumsum(lens) - lens
    dep_a = np.concatenate([np.sort(rng.random(n)) for n in lens] + [np.zeros(0)]).astype(np.float32)
    dep_b = np.sort(rng.random((P, nb)), -1).astype(np.float32)
    if ties:
        for p in range(P):
            if lens[p] >= 3:
                dep_b[p, :min(nb, 3)] = dep_a[first[p] + 1]               # one a equal to several b
                dep_a[first[p] + lens[p] - 2:first[p] + lens[p]] = dep_b[p, -1] = max(dep_b[p, -1], dep_a[first[p] + lens[p] - 1])
        dep_b.sort(-1)
    return dep_a, np.stack([first, lens], 1).astype(np.int64), dep_b


def test_merge_vals_equals_the_reference_rule():
    rng = np.random.default_rng(1)
    for nb, ties in ((1, False), (9, False), (9, True), (33, True)):
        lens = np.array([0, 1, 2, 5, 40, 3, 0, 64, 7])
        dep_a, pi_a, dep_b = _merge_case(rng, lens, nb, ties)
        sdf_a, sdf_b = rng.standard_normal(dep_a.size).astype(np.float32), rng.standard_normal(dep_b.shape).astype(np.float32)
        P = len(lens)
        pi_b = np.stack([np.arange(P) * nb, np.full(P, nb)], 1)
        pa, pb, pim = opk.try_merge_two_packs_sorted_aligned(torch.from_numpy(dep_a), torch.from_numpy(pi_a), torch.from_numpy(dep_b.reshape(-1)),
                                                             torch.from_numpy(pi_b), True)
        ref_d, ref_s = np.empty(dep_a.size + P * nb, np.float32), np.empty(dep_a.size + P * nb, np.float32)
        ref_d[pa.numpy()], ref_d[pb.numpy()] = dep_a, dep_b.reshape(-1)
        ref_s[pa.numpy()], ref_s[pb.numpy()] = sdf_a, sdf_b.reshape(-1)
        dep_m, sdf_m, pi_m = G.merge_vals(dep_a, sdf_a, pi_a, dep_b, sdf_b)
        assert np.array_equal(pi_m, pim.numpy()) and np.array_equal(bits(dep_m), bits(ref_d)) and np.array_equal(bits(sdf_m), bits(ref_s))
        assert G.merge_vals(dep_a, None, pi_a, dep_b, None)[1] is None


def test_merge_vals_known_answer_of_the_reference():
    """pack_ops/unit_test.py:956-965 of the reference, re-cut into rows of b (the kernel's b is [P, nb])"""
    ka = np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.2, 0.8], np.float32)
    kb = np.array([[0.0, 0.25, 0.26, 0.6], [0.1, 0.15, 0.3, 0.4]], np.float32)
    dep_m, sdf_m, pi_m = G.merge_vals(ka, np.arange(7, dtype=np.float32), [[0, 5], [5, 2]], kb, 100 + np.arange(8, dtype=np.float32).reshape(2, 4))
    ga, gb = [1, 2, 5, 6, 7, 11, 14], [0, 3, 4, 8, 9, 10, 12, 13]
    assert sdf_m[ga].tolist() == list(range(7)) and sdf_m[gb].tolist() == [100 + k for k in range(8)]
    assert np.array_equal(dep_m[ga], ka) and np.array_equal(dep_m[gb], kb.reshape(-1)) and pi_m.tolist() == [[0, 9], [9, 6]]


def _kway(runs):
    """serial stable merge of sorted runs: always take the smallest head, the earliest run on a tie"""
    heads, out = [0] * len(runs), []
    while True:
        best = None
        for q, run in enumerate(runs):
            if heads[q] < len(run) and (best is None or run[heads[q]] < runs[best][heads[best]]):
                best = q
        if best is None:
            return out
        out.append(runs[best][heads[best]])
        heads[best] += 1


def test_assemble_boundary_is_the_stable_merge():
    rng = np.random.default_rng(2)
    for R, nc, run_len in ((17, 5, [3, 3, 7]), (9, 1, [4]), (20, 65, [9, 9, 33]), (6, 3, [1] * 8), (5, 4, [])):
        nf = sum(run_len)
        # a coarse grid of values so that ties within and across runs are frequent, with both zeros among them
        vals = np.concatenate([np.round(rng.random(40) * 8) / 8, [0.0, -0.0]]).astype(np.float32)
        coarse = np.sort(rng.choice(vals, (R, nc)), -1)
        hit = np.sort(rng.choice(R, R // 2, replace=False))
        fine = np.concatenate([np.sort(rng.choice(vals, (hit.size, n)), -1) for n in run_len] + [np.zeros((hit.size, 0), np.float32)], 1)
        out = G.assemble_boundary(coarse, hit, fine, run_len)
        pi = out["pack_infos"]
        assert pi[:, 0].tolist() == (np.cumsum(pi[:, 1]) - pi[:, 1]).tolist() and out["d1"].size == R * nc + hit.size * nf
        for r in range(R):
            b, n = pi[r]
            j = np.flatnonzero(hit == r)
            row = np.concatenate([coarse[r], fine[j[0]]]) if j.size else coarse[r]
            assert n == row.size
            assert np.array_equal(bits(out["d1"][b:b + n]), bits(np.sort(row, kind="stable")))
            if j.size:
                cuts = np.cumsum([0] + run_len) + nc
                runs = [list(coarse[r])] + [list(fine[j[0]][cuts[q] - nc:cuts[q + 1] - nc]) for q in range(len(run_len))]
                assert np.array_equal(bits(out["d1"][b:b + n]), bits(np.array(_kway(runs), np.float32)))
            assert (out["ridx_all"][b:b + n] == r).all()
            d = out["d1"][b:b + n]
            mid = [np.float32(d[k] + np.float32(np.float32(d[k + 1] - d[k]) * np.float32(0.5))) for k in range(n - 1)] + [np.float32(d[-1] + np.float32(0))]
            assert np.array_equal(bits(out["mid"][b:b + n]), bits(np.array(mid)))
    # the tie order is visible in the sign bit: the coarse zero comes first
    out = G.assemble_boundary(np.array([[0.0, 1.0]], np.float32), [0], np.array([[-0.0, 2.0]], np.float32), [2])
    assert bits(out["d1"]).tolist() == bits([0.0, -0.0, 1.0, 2.0]).tolist()
    out = G.assemble_boundary(np.array([[-0.0, 1.0]], np.float32), [0], np.array([[0.0, 2.0]], np.float32), [2])
    assert bits(out["d1"]).tolist() == bits([-0.0, 0.0, 1.0, 2.0]).tolist()
    assert bits(G.interval_mid(np.array([-1.0, -0.0], np.float32), 2)).tolist() == bits([-0.5, 0.0]).tolist()     # last: -0.0 + 0 = +0.0


def test_assemble_boundary_live_counts_and_ray_subset():
    rng = np.random.default_rng(3)
    coarse = np.sort(rng.random((12, 4)), -1).astype(np.float32)
    hit, fine = np.array([1, 4, 5, 9, 11]), np.sort(rng.random((5, 3)), -1).astype(np.float32)
    full = G.assemble_boundary(coarse[:10], hit[:3], fine[:3], [3])
    cut = G.assemble_boundary(coarse, hit, fine, [3], n_rays=10, n_hit=3)               # ray 9 is listed past the live hits: a coarse pack
    assert all(np.array_equal(full[k], cut[k], equal_nan=True) for k in full) and cut["pack_infos"][9].tolist() == [9 * 4 + 3 * 3, 4]
    part = G.assemble_boundary(coarse, hit, fine, [3], rays=[0, 5])
    whole = G.assemble_boundary(coarse, hit, fine, [3])
    assert np.array_equal(part["pack_infos"], whole["pack_infos"])
    for r in (0, 5):
        b, n = whole["pack_infos"][r]
        assert np.array_equal(part["d1"][b:b + n], whole["d1"][b:b + n]) and np.array_equal(part["mid"][b:b + n], whole["mid"][b:b + n])
    assert np.isnan(part["d1"]).sum() == whole["d1"].size - 4 - 7


def test_assemble_boundary_equals_the_reference_python():
    z = np.load(GOLDEN)
    A, B, nB = z["merge_batch.A"], z["merge_batch.B"], z["merge_batch.nB"]
    assert z["merge_batch.nA"].tolist() == list(range(A.shape[0]))
    out = G.assemble_boundary(A, nB, B, [B.shape[1]])
    assert np.array_equal(out["pack_infos"], z["merge_batch.pinf"])
    assert np.array_equal(out["d1"][z["merge_batch.pa"]], A) and np.array_equal(out["d1"][z["merge_batch.pb"]], B)
    assert np.array_equal(out["ridx_all"][z["merge_batch.pb"]], np.broadcast_to(nB[:, None], B.shape))


def test_compact_samples_by_hand():
    pi = [[0, 3], [3, 0], [3, 4], [7, 2]]
    sel = np.array([0, 2, 0, 1, 0, 0, 255, 0, 0], np.uint8)
    d1 = np.array([1, 2, 4, 10, 11, 13, 17, 5, 6], np.float32)
    alpha = np.arange(9, dtype=np.float32) / 16
    out = G.compact_samples(sel, pi, [0, 1, 1, 3], [1, 0, 2, 0], alpha, d1=d1)
    assert out["pidx"].tolist() == [1, 3, 6] and out["ridx_c"].tolist() == [0, 2, 2]
    assert out["t_c"].tolist() == [3.0, 10.5, 17.0] and out["alpha_c"].tolist() == [1 / 16, 3 / 16, 6 / 16]
    out = G.compact_samples(sel, pi, [0, 1, 1, 3], [1, 0, 2, 0], alpha, ridx_all=np.arange(9) + 50, t=d1 * 2, n_out=5)
    assert out["ridx_c"].tolist() == [51, 53, 56, -1, -1] and out["t_c"][:3].tolist() == [4.0, 20.0, 34.0] and np.isnan(out["t_c"][3:]).all()


def test_small_kernels():
    assert G.flag_nonzero(np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, 2.0], np.float32)).tolist() == [0, 0, 1, 1, 1, 1, 1]
    assert G.flag_nonzero(np.ones(5, np.float32), n_live=2).tolist() == [1, 1, 0, 0, 0]
    assert G.scatter_f32([5.0, 6.0], [3, 0], 4).tolist() == [6.0, 0.0, 0.0, 5.0]
    a, b = G.gather_rays([2, 0], np.arange(9).reshape(3, 3), np.arange(3))
    assert a.tolist() == [[6, 7, 8], [0, 1, 2]] and b.tolist() == [2, 0]


def test_min_max_propagate_nan_and_order_the_zeros():
    nan, pz, nz = np.float32(np.nan), np.float32(0.0), np.float32(-0.0)
    a, b = np.array([1, nan, 2, pz, nz, nz, -np.inf], np.float32), np.array([nan, 1, 3, nz, pz, nz, np.inf], np.float32)
    assert bits(G.max_nan(a, b)).tolist() == [0x7FC00000, 0x7FC00000] + bits([3, pz, pz, nz, np.inf]).tolist()
    assert bits(G.min_nan(a, b)).tolist() == [0x7FC00000, 0x7FC00000] + bits([2, nz, nz, nz, -np.inf]).tolist()


def test_ray_test_aabb_equals_a_float64_slab_test():
    rng = np.random.default_rng(4)
    c, r = np.array([0.1, -0.2, 0.05]), np.array([1.0, 0.7, 1.3])
    n = 4000
    o = rng.standard_normal((n, 3)) * 2
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    o32, d32 = o.astype(np.float32), d.astype(np.float32)
    for near, far in ((None, None), (0.01, None), (0.5, 3.2)):
        got = G.ray_test_aabb(o32, d32, c.astype(np.float32), r.astype(np.float32), near, far)
        on, dn = (o32.astype(np.float64) - c.astype(np.float32)) / r.astype(np.float32), d32.astype(np.float64) / r.astype(np.float32)
        ta, tb = (-1 - on) / dn, (1 - on) / dn
        tn, tf = np.minimum(ta, tb).max(-1), np.maximum(ta, tb).min(-1)
        tn_c = tn if near is None else np.maximum(tn, np.float32(near))
        tf_c = tf if far is None else np.minimum(tf, np.float32(far))
        m = (tf_c > tn_c) & (tf_c > (0 if near is None else np.float32(near)))
        if far is not None:
            m &= tn_c < np.float32(far)
        margin = np.minimum(np.abs(tf_c - tn_c), np.abs(tf_c - (0 if near is None else near)))
        if far is not None:
            margin = np.minimum(margin, np.abs(tn_c - far))
        clear = margin > 1e-4                                             # rays that are not near a decision boundary
        assert clear.mean() > 0.95 and 0.05 < m.mean() < 0.95
        assert np.array_equal(got["flag"][clear], m[clear].astype(np.int32))
        assert np.allclose(got["o_n"], on, rtol=2e-7, atol=0) and np.allclose(got["d_n"], dn, rtol=2e-7, atol=0)
        tol = 1e-6 * ((1 + np.abs(on)) / np.abs(dn)).max(-1)                # (+-1 - o') cancels, and the quotient by d' amplifies it
        assert (np.abs(got["near"] - tn_c) <= tol).all() and (np.abs(got["far"] - tf_c) <= tol).all()


def test_ray_test_aabb_nan_zero_components_and_side_results():
    one = np.ones(3, np.float32)
    # origin on the x = -1 slab with a zero x direction: 0 / 0 = NaN reaches near and far and clears the flag, clamps or not
    for near, far in ((None, None), (0.1, 5.0)):
        g = G.ray_test_aabb([[-1.0, 0.0, 0.0]], [[0.0, 1.0, 0.0]], 0 * one, one, near, far)
        assert np.isnan(g["near"][0]) and np.isnan(g["far"][0]) and g["flag"][0] == 0
    # an axis-parallel ray inside the slabs of its zero components: +-inf there, a finite interval from the third axis
    g = G.ray_test_aabb([[-3.0, 0.5, 0.5]], [[1.0, 0.0, -0.0]], 0 * one, one)
    assert (g["near"][0], g["far"][0], g["flag"][0]) == (2.0, 4.0, 1)
    g = G.ray_test_aabb([[-3.0, 1.5, 0.5]], [[1.0, 0.0, 0.0]], 0 * one, one)
    assert g["flag"][0] == 0
    # image-ordered rays: W - 1 steps forward, one back
    for W, H in ((2, 3), (3, 4), (8, 5), (800, 3), (7, 1)):
        x, y = np.meshgrid(np.arange(W) - W / 2 + 0.5, np.arange(H) - H / 2 + 0.5)
        d = np.stack([x.ravel(), y.ravel(), np.full(W * H, 8.0 * W)], -1)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        g = G.ray_test_aabb(np.tile([0.0, 0.0, -3.0], (W * H, 1)), d, 0 * one, one)
        assert g["row_len"] == (W if H > 1 else -1)
        if W >= 8:
            assert g["coherent_pairs"] == (W - 1) * H                       # the steps inside a row are neighbour pairs, the returns are not
    assert G.ray_test_aabb(np.zeros((2, 3)), np.ones((2, 3)), 0 * one, one)["row_len"] == -1


def test_query_counts_by_hand():
    c = np.arange(100, 132, dtype=np.int64)
    c[[0, 3, 4, 6, 7, 20]] = [1000, 5000, 300, 777, 90, 0]
    # three stages of 9, 9, 33 fine samples on 65 coarse: the merged buffer grows by 9 per hit ray and merged stage
    p0 = G.query_counts(c, 0, 65, [9, 9, 33], march_cap=5000 + 300 * 18, kept_cap=0)
    want = {12: 5000, 13: 300, 14: 2700, 15: 2700, 16: 9900, 17: 0, 22: 7700, 23: 10400, 24: 10400, 25: 10400, 18: 65000 + 300 * 51, 20: 0}
    assert all(p0[k] == v for k, v in want.items())
    assert all(p0[k] == c[k] for k in range(32) if k not in want)
    p1 = G.query_counts(p0, 1, 65, [9, 9, 33], march_cap=0, kept_cap=777)
    assert (p1[19], p1[21], p1[26], p1[20]) == (777, 90, 1000, 0) and all(p1[k] == p0[k] for k in range(32) if k not in (19, 21, 26))
    # one stage of 16, and both capacities one short: nothing is merged after the only stage, so M alone must fit
    c[20] = 0
    q0 = G.query_counts(c, 0, 8, [16], march_cap=4999, kept_cap=0)
    assert (q0[12], q0[13], q0[14], q0[15], q0[22], q0[25], q0[18], q0[20]) == (0, 0, 0, 0, 0, 0, 8000, 1)
    assert G.query_counts(c, 0, 8, [16], march_cap=5000, kept_cap=0)[[12, 13, 14, 22, 18, 20]].tolist() == [5000, 300, 4800, 5000, 8000 + 4800, 0]
    q1 = G.query_counts(q0, 1, 8, [16], march_cap=0, kept_cap=776)
    assert (q1[19], q1[21], q1[26], q1[20]) == (0, 0, 0, 3)                   # the flag is OR-ed
