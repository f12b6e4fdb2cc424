"""The CPU oracle of `_pack_ops` (oracle/pack_ops.py) at the edges its GPU tests use: the closed-form merge rule that
k_merge_sorted_aligned (csrc/pack_ops.cu) evaluates, against the oracle's serial bookkeeping; the alpha_to_vw backward on a NaN
alpha; the per-pack sort's contract (a permutation, ascending, stable, NaN last) on gapped and empty-pack layouts; and the
interleave_linstep index past 2^24."""
import numpy as np
import pytest
import torch

from oracle import pack_ops as opk

NAN, INF = float("nan"), float("inf")


def _layout(lens, gaps=None):
    lens = np.asarray(lens, np.int64)
    gaps = np.zeros_like(lens) if gaps is None else np.asarray(gaps, np.int64)
    begin = np.cumsum(gaps + lens) - lens
    return torch.from_numpy(np.stack([begin, lens], 1))


def merge_closed_form(va, pia, vb, pib):
    """k_merge_sorted_aligned's rule: m = the numbers at the head of b (NaNs last), key_j = b_j for j < m else b_{m-1};
    position of a_i = i + (c if c < m else |b|), c = #{j < m : !(a_i < b_j)}; position of b_j = j + #{a : a < key_j}"""
    pa, pb = pia.numpy(), pib.numpy()
    n = pa[:, 1] + pb[:, 1]
    first = np.cumsum(n) - n
    ia, ib = np.zeros(va.shape[0], np.int64), np.zeros(vb.shape[0], np.int64)
    for p in range(pa.shape[0]):
        a = va[pa[p, 0]:pa[p, 0] + pa[p, 1]]
        b = vb[pb[p, 0]:pb[p, 0] + pb[p, 1]]
        m = int(np.sum(~np.isnan(b)))
        assert not np.isnan(b[:m]).any()
        for i, x in enumerate(a):
            c = int(np.sum(~(x < b[:m])))
            ia[pa[p, 0] + i] = first[p] + i + (c if c < m else len(b))
        for j in range(len(b)):
            key = b[j] if (j < m or m == 0) else b[m - 1]
            ib[pb[p, 0] + j] = first[p] + j + int(np.sum(a < key))
    return ia, ib


def naive_closed_form(va, pia, vb, pib):
    """the rule without the NaN tail of b: a_i -> i + #{b : !(a_i < b)}, b_j -> j + #{a : a < b_j}"""
    pa, pb = pia.numpy(), pib.numpy()
    n = pa[:, 1] + pb[:, 1]
    first = np.cumsum(n) - n
    ia, ib = np.zeros(va.shape[0], np.int64), np.zeros(vb.shape[0], np.int64)
    for p in range(pa.shape[0]):
        a = va[pa[p, 0]:pa[p, 0] + pa[p, 1]]
        b = vb[pb[p, 0]:pb[p, 0] + pb[p, 1]]
        for i, x in enumerate(a):
            ia[pa[p, 0] + i] = first[p] + i + int(np.sum(~(x < b)))
        for j, y in enumerate(b):
            ib[pb[p, 0] + j] = first[p] + j + int(np.sum(a < y))
    return ia, ib


def merge_edge_packs(seed, b_nan):
    """aligned packs a, b, each ascending with NaNs last (torch.sort's order): ties inside a, inside b and across them, -0.0 in a
    against +0.0 in b, +-inf, NaN tails, empty a / empty b / both empty, and packs longer than 64"""
    rng = np.random.default_rng(seed)
    pool = np.array([-INF, -1.0, -0.0, 0.0, 0.25, 0.5, 0.5, 1.0, 2.0, INF], np.float32)
    la = [0, 3, 0, 1, 2, 7, 31, 33, 65, 100, 5, 0]
    lb = [0, 0, 4, 1, 3, 9, 33, 31, 70, 64, 5, 2]
    va, vb = [], []
    for p, (na, nb) in enumerate(zip(la, lb)):
        a = rng.choice(pool, na)
        b = rng.choice(pool, nb)
        a[a == 0] = -0.0                                  # the zeros of a are -0.0, those of b +0.0
        b[b == 0] = 0.0
        if na > 4 and p % 2:
            a[-2:] = NAN
        if b_nan and nb > 2 and p % 3 != 1:
            b[-(1 + p % 2):] = NAN
        if b_nan and p == len(la) - 1:
            b[:] = NAN                                    # a b of NaNs only
        va.append(torch.from_numpy(a).sort(stable=True).values)
        vb.append(torch.from_numpy(b).sort(stable=True).values)
    return torch.cat(va), _layout(la), torch.cat(vb), _layout(lb)


@pytest.mark.parametrize("b_nan", [False, True])
def test_merge_closed_form_equals_serial_bookkeeping(b_nan):
    va, pia, vb, pib = merge_edge_packs(7, b_nan)
    ra, rb, rp = opk.try_merge_two_packs_sorted_aligned(va, pia, vb, pib, True)
    ca, cb = merge_closed_form(va.numpy(), pia, vb.numpy(), pib)
    assert np.array_equal(ca, ra.numpy()) and np.array_equal(cb, rb.numpy())
    # every element lands in its merged pack, once
    both = np.concatenate([ra.numpy(), rb.numpy()])
    assert np.array_equal(np.sort(both), np.arange(both.size))
    na, nb = naive_closed_form(va.numpy(), pia, vb.numpy(), pib)
    if not b_nan:
        assert np.array_equal(na, ra.numpy()) and np.array_equal(nb, rb.numpy())
    else:
        # with numbers and NaNs in one b, the rule without the NaN tail is not the reference's (nor a permutation)
        assert not (np.array_equal(na, ra.numpy()) and np.array_equal(nb, rb.numpy()))
    # a b element equal to an a element goes first, -0.0 == +0.0 included (pack 3: a = [-0.0?], b = [+0.0?] when drawn)
    merged = np.empty(both.size, np.float32)
    merged[ra.numpy()], merged[rb.numpy()] = va.numpy(), vb.numpy()
    for b, n in rp.tolist():
        seg = merged[b:b + n]
        num = seg[~np.isnan(seg)]
        assert np.all(num[1:] >= num[:-1])


def test_merge_b_before_equal_a_signed_zero():
    va, vb = torch.tensor([-0.0, 1.0]), torch.tensor([0.0, 1.0])
    pi = torch.tensor([[0, 2]])
    ra, rb, _ = opk.try_merge_two_packs_sorted_aligned(va, pi, vb, pi, True)
    assert rb.tolist() == [0, 2] and ra.tolist() == [1, 3]
    ca, cb = merge_closed_form(va.numpy(), pi, vb.numpy(), pi)
    assert ca.tolist() == ra.tolist() and cb.tolist() == rb.tolist()


def test_alpha_to_vw_backward_nan_alpha_is_finite():
    """fmaxf(1 - NaN, 1e-10f) is 1e-10f: the NaN sample itself gets (gw*T - accum) / 1e-10, finite when the weights are; the samples
    after it see T = NaN.  (With the forward's own weights, the NaN weight makes accum NaN for the whole pack.)"""
    a = torch.tensor([0.25, NAN, 0.5, 0.5], dtype=torch.float32)
    pi = torch.tensor([[0, 4]])
    w = opk.packed_alpha_to_vw_forward(a, pi, 1e-4, 0.0, False)[0]
    assert w[0] == 0.25 and torch.isnan(w[1:]).all()
    assert torch.isnan(opk.packed_alpha_to_vw_backward(w, torch.ones(4), a, pi, 1e-4, 0.0)).all()
    w = torch.tensor([0.25, 0.0, 0.0, 0.0])                               # finite weights, e.g. after a nan_to_num
    ga = opk.packed_alpha_to_vw_backward(w, torch.tensor([1.0, 1.0, 0.0, 0.0]), a, pi, 1e-4, 0.0)
    f = np.float32
    assert ga[0] == f(f(1.0) - f(0.25)) / f(0.75)                        # accum = 0.25
    assert ga[1] == f(f(0.75) / f(1e-10)) and np.isfinite(float(ga[1]))   # (1 * 0.75 - 0) / fmaxf(NaN, 1e-10f)
    assert torch.isnan(ga[2:]).all()


@pytest.mark.parametrize("gapped", [False, True])
def test_sort_is_a_permutation_nan_last(gapped):
    rng = np.random.default_rng(3)
    lens = [1, 0, 2, 31, 0, 32, 33, 1024, 0]
    gaps = [2, 0, 1, 0, 3, 5, 0, 7, 1] if gapped else None
    pi = _layout(lens, gaps)
    S = int(pi[-1, 0] + pi[-1, 1])
    pool = np.array([NAN, -INF, -0.0, 0.0, 1.0, 1.0, -2.5, INF], np.float32)
    v = torch.from_numpy(rng.choice(pool, S))
    old = v.clone()
    idx = opk.packed_sort_qsort(v, pi, True).numpy()
    in_pack = np.zeros(S, bool)
    for b, n in pi.tolist():
        in_pack[b:b + n] = True
        seg_i = idx[b:b + n]
        assert np.array_equal(np.sort(seg_i), np.arange(b, b + n))    # a permutation of its own pack
        seg = v.numpy()[b:b + n]
        k = int(np.sum(~np.isnan(seg)))
        assert np.isnan(seg[k:]).all() and not np.isnan(seg[:k]).any()   # NaN last
        assert np.all(seg[1:k] >= seg[:k - 1])
        ties = (seg[1:] == seg[:-1]) | (np.isnan(seg[1:]) & np.isnan(seg[:-1]))
        assert np.all(seg_i[1:][ties] > seg_i[:-1][ties])                # stable: ties (-0.0 with +0.0, NaN with NaN) by index
    assert np.array_equal(v.numpy().view(np.uint32), old.numpy()[idx].view(np.uint32))
    assert np.array_equal(idx[~in_pack], np.arange(S)[~in_pack])        # elements between packs keep their place
    assert np.array_equal(v.numpy()[~in_pack].view(np.uint32), old.numpy()[~in_pack].view(np.uint32))


def test_linstep_rounds_the_index_past_2_24():
    """the reference computes start + (float)j * step: j = 2^24 + 1 is 2^24 in float"""
    n = (1 << 24) + 3
    start, step = torch.tensor([0.5], dtype=torch.float32), torch.tensor([3.0], dtype=torch.float32)
    out, _ = opk.interleave_linstep(start, torch.tensor([n]), step, False)
    j = np.array([(1 << 24), (1 << 24) + 1, (1 << 24) + 2], np.int64)
    want = (np.float64(0.5) + j.astype(np.float32).astype(np.float64) * 3.0).astype(np.float32)
    assert np.array_equal(out.numpy()[j], want)
    assert out[(1 << 24) + 1] == out[1 << 24]
