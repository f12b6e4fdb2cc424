"""The index-bookkeeping kernels of the per-ray query (csrc/neus_glue.cu) through the C ABI against oracle/glue.py, bit for bit: at sizes
where their sweep and grid-stride loops run several times (sized from the SM count by restating the launchers' grid arithmetic; every
such case asserts the blocks / sweeps / trips it reaches), and at their segment, chunk, tie and device-count edges.
tests/test_glue_gpu.py compares the same kernels with this package's op-by-op wrapper chain at one small shape each."""
import ctypes

import numpy as np
import pytest
import torch

from neuralsim_b200 import _lib as L
from neuralsim_b200.graphics import neus_fused as NF
from neuralsim_b200.graphics.neus_static import _call, _scan
from oracle import glue as G

pytestmark = pytest.mark.gpu

SWEEP = 1024 * 8                                           # k_scan_counts: kScanT threads x kScanI items per sweep
I32, I64 = torch.int32, torch.int64


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def wave_grid(work_items, block, ctas_per_sm=8):
    """csrc/nsb_common.cuh: whole waves of resident CTAs, at most 8 of them; grid-stride loops cover the rest"""
    need, wave = -(-work_items // block), sms() * ctas_per_sm
    return max(need, 1) if need <= wave else min(-(-need // wave), 8) * wave


def warp_trips(n_items, n_launch, items_per_warp=1):
    """(fewest, most) loop trips of a warp of the one-warp-per-item kernels (256 threads per CTA) launched for n_launch items"""
    warps = wave_grid(n_launch * 32, 256) * 8
    units = -(-n_items // items_per_warp)
    return units // warps, -(-units // warps)


def thread_trips(n):
    threads = wave_grid(n, 256) * 256
    return n // threads, -(-n // threads)


def scan_layout(n):
    """nsb_scan_counts: blocks, segment length, sweeps of the first and of the last block"""
    nb = max(1, min(-(-n // SWEEP), min(sms(), 128)))
    seg = -(-(-(-n // nb)) // 8) * 8
    last = n - (nb - 1) * seg
    return nb, seg, -(-min(seg, n) // SWEEP), -(-last // SWEEP), last


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def same(t, ref, what="", any_nan=False):
    """bit-equality of a device tensor with an oracle array (floats as bit patterns, NaN included).  any_nan: every NaN equals every
    NaN, for values that arithmetic on a NaN input produces (the payload of those is the processor's choice, not the kernel's)"""
    ref = np.ascontiguousarray(ref)
    assert tuple(t.shape) == ref.shape, (what, t.shape, ref.shape)
    r = torch.from_numpy(ref).cuda()
    if any_nan:
        assert torch.equal(t.isnan(), r.isnan()), what
        t, r = torch.where(t.isnan(), 0.0, t), torch.where(r.isnan(), 0.0, r)
    if t.dtype == torch.float32:
        t, r = t.view(I32), r.view(I32)
    if not torch.equal(t, r):
        bad = (t != r).reshape(t.shape[0], -1).any(-1).nonzero()[:5, 0].tolist() if t.numel() else []
        raise AssertionError(f"{what}: first differing rows {bad}: {t[bad].tolist()} != {r[bad].tolist()}")


def refused(rc, text):
    assert rc == 2 and text in L.lib().nsb_last_error().decode(), (rc, L.lib().nsb_last_error())


def counts_block(**slots):
    cnt = torch.zeros(32, dtype=I64, device="cuda")
    for k, v in slots.items():
        cnt[int(k[1:])] = v
    return cnt


# ================================================================================================ scan
def _ws(n=1):
    return torch.zeros(n, NF._scan_ws_bytes(), dtype=torch.uint8, device="cuda")


def run_scan(c, want=("first", "info2", "index", "pack", "src"), check=None):
    """device-slot form (ticket 0, totals into a counts block) with sentinel-filled outputs; compares every requested output"""
    n = c.shape[0]
    o = G.scan_counts(c.cpu().numpy())
    src = torch.arange(n + 1, device="cuda") * 3 + 1 if "src" in want else None      # n + 1: a pointer that is not NULL at n = 0
    first = torch.full((n,), -5, dtype=I32, device="cuda") if "first" in want else None
    info2 = torch.full((n, 2), -5, dtype=I32, device="cuda") if "info2" in want else None
    index = torch.full((n + 3,), -5, dtype=I64, device="cuda") if "index" in want else None
    pack = torch.full((n + 3, 2), -5, dtype=I64, device="cuda") if "pack" in want else None
    nz_src = torch.full((n + 3,), -5, dtype=I64, device="cuda") if src is not None else None
    cnt = counts_block(s5=-1, s8=-1)
    _scan(c, cnt, 6, first=first, info2=info2, index=index, pack=pack, src=src, nz_src=nz_src, ws=_ws()[0])
    tot, m = o["totals"]
    assert cnt.tolist() == [0] * 5 + [-1, tot, m, -1] + [0] * 23              # the two totals and nothing else
    check = check or want
    if "first" in check:
        same(first, o["first"], "first")
    if "info2" in check:
        same(info2, o["info2"], "info2")
    if "index" in check:
        same(index[:m], o["nz_index"], "nz_index")
        assert bool((index[m:] == -5).all())
    if "pack" in check:
        same(pack[:m], o["nz_pack"], "nz_pack")
        assert bool((pack[m:] == -5).all())
    if "src" in check:
        same(nz_src[:m], 3 * o["nz_index"] + 1, "nz_src")
        assert bool((nz_src[m:] == -5).all())
    return o


def sparse_counts(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randint(0, 7, (n,), generator=g, device="cuda") * (torch.rand(n, generator=g, device="cuda") < 0.4)).to(I32)


def test_scan_sizes_around_sweeps_and_the_block_cap():
    cap = min(sms(), 128)
    sizes = [0, 1, 7, 8, 9, SWEEP - 1, SWEEP, SWEEP + 1, 2 * SWEEP + 1, cap * SWEEP - 1, cap * SWEEP, cap * SWEEP + 1, 3 * cap * SWEEP + 5]
    lay = {n: scan_layout(n) for n in sizes if n}
    assert lay[SWEEP][:3] == (1, SWEEP, 1) and lay[SWEEP + 1][0] == 2 and lay[2 * SWEEP + 1][0] == 3
    assert lay[cap * SWEEP - 1][0] == cap and lay[cap * SWEEP][:4] == (cap, SWEEP, 1, 1)       # every segment ends on its only sweep's edge
    assert lay[cap * SWEEP + 1][:3] == (cap, SWEEP + 8, 2)                                     # the second sweep holds 8 items
    nb, seg, s0, s1, last = lay[3 * cap * SWEEP + 5]
    assert nb == cap and s0 >= 4 and s1 >= 3 and seg % SWEEP and last % SWEEP                  # >= 3 sweeps, segments end inside one
    for n in sizes:
        run_scan(sparse_counts(n, n % 1000))


def test_scan_frame_of_boundary_samples():
    n = 27_800_000                                                             # one scan entry per boundary sample of an 800 x 600 frame
    nb, seg, s0, s1, last = scan_layout(n)
    assert nb == min(sms(), 128) and s0 >= 3 and s1 >= 3 and seg % SWEEP and last % SWEEP
    run_scan(sparse_counts(n, 7), want=("first", "index", "pack"))


def test_scan_count_patterns():
    cap = min(sms(), 128)
    n = 3 * cap * SWEEP + 5
    nb, seg, s0, s1, last = scan_layout(n)
    assert s0 >= 4 and s1 >= 3
    i = torch.arange(n, device="cuda")
    pats = {
        "all zero": torch.zeros(n, dtype=I32, device="cuda"),
        "all one": torch.ones(n, dtype=I32, device="cuda"),
        "only entry 0": (i == 0).to(I32) * 5,
        "only entry n - 1": (i == n - 1).to(I32) * 5,
        "one block's segment": ((i // seg == nb // 2) & (i % 3 == 0)).to(I32) * 4,
        "from the third sweep of every segment on": ((i % seg) >= 2 * SWEEP).to(I32) * ((i % 5) + 1).to(I32),
        "the first sweep of every segment": ((i % seg) < SWEEP).to(I32) * ((i % 2) * 3).to(I32),
    }
    for name, c in pats.items():
        o = run_scan(c)
        assert o["totals"][0] == int(c.sum()), name
    assert s1 == 3 and pats["from the third sweep of every segment on"][(nb - 1) * seg + 2 * SWEEP:].sum() > 0


def test_scan_sums_near_and_above_int32():
    n = 1_049_000                                                              # 2047 n = 2 147 303 000 < 2^31 by 180 648
    assert 0 < 2 ** 31 - 2047 * n < 200_000 and scan_layout(n)[0] == min(sms(), 128)
    run_scan(torch.full((n,), 2047, dtype=I32, device="cuda"))
    # above 2^31 only the int64 outputs are meaningful: the totals and nz_pack
    n = 1_100_000
    o = run_scan(torch.full((n,), 2047, dtype=I32, device="cuda"), check=("pack",))
    assert o["totals"][0] == 2047 * n > 2 ** 31
    n = 4 * min(sms(), 128) * SWEEP                                            # >= 4 sweeps per block, each sweep's carry past 2^31
    c = torch.full((n,), 2047, dtype=I32, device="cuda")
    assert 2047 * n / 2 > 2 ** 31 and scan_layout(n)[2] == 4
    run_scan(c, check=("pack", "index"))


def test_scan_each_output_alone_and_the_host_slot_form():
    n = 3 * SWEEP + 11
    c = sparse_counts(n, 3)
    for want in (("first",), ("info2",), ("index",), ("pack",), ("index", "src"), ()):
        run_scan(c, want=want)
    o = G.scan_counts(c.cpu().numpy())
    extra = torch.tensor([41, 42], device="cuda")
    sc = NF.scan_counts(c, want_first=True, want_info2=True, want_index=True, want_pack=True, src=torch.arange(n, device="cuda") * 3 + 1, extra=extra)
    assert (sc["total"], sc["n_nonzero"]) == o["totals"] and sc["extra"] == [41]        # totals[2] = *extra_src
    same(sc["first"], o["first"]), same(sc["info2"], o["info2"]), same(sc["index"], o["nz_index"]), same(sc["pack"], o["nz_pack"])
    same(sc["src"], 3 * o["nz_index"] + 1)
    empty = NF.scan_counts(c[:0], want_index=True)
    assert (empty["total"], empty["n_nonzero"], empty["index"].numel()) == (0, 0, 0)


def test_four_scans_back_to_back_on_one_fill():
    """the graph step's pattern: four workspaces zeroed by one fill, four scans on one stream, totals in four slots of one block"""
    cap = min(sms(), 128)
    ns = [2 * cap * SWEEP + 3, 480_000, SWEEP + 1, 100_000]
    cs = [sparse_counts(n, 11 + k) for k, n in enumerate(ns)]
    ws = _ws(4)
    cnt = counts_block()
    outs = [(torch.empty(n, dtype=I32, device="cuda"), torch.empty(n, dtype=I64, device="cuda")) for n in ns]
    for k, c in enumerate(cs):
        _scan(c, cnt, 3 * k, first=outs[k][0], index=outs[k][1], ws=ws[k])
    for k, c in enumerate(cs):
        o = G.scan_counts(c.cpu().numpy())
        assert tuple(cnt[3 * k:3 * k + 2].tolist()) == o["totals"]
        same(outs[k][0], o["first"]), same(outs[k][1][:o["totals"][1]], o["nz_index"])


# ================================================================================================ merge
def merge_inputs(rng, lens, nb, lo=0.0, hi=3.0):
    lens = np.asarray(lens, np.int64)
    P, S = lens.size, int(lens.sum())
    first = np.cumsum(lens) - lens
    key = np.repeat(np.arange(P), lens)
    dep_a = (lo + (hi - lo) * rng.random(S)).astype(np.float32)
    dep_a = dep_a[np.lexsort((dep_a, key))]                                    # sorted inside every pack
    dep_b = np.sort(lo + (hi - lo) * rng.random((P, nb)), -1).astype(np.float32)
    return dep_a, np.stack([first, lens], 1), dep_b


def run_merge(dep_a, sdf_a, pi_a, dep_b, sdf_b, n_live=None, with_sdf=True):
    P, nb = dep_b.shape
    n_out = dep_a.size + P * nb
    d = [dev(x) for x in (dep_a, sdf_a, pi_a, dep_b, sdf_b)]
    dep_m = torch.full((n_out,), float("nan"), device="cuda")
    sdf_m = torch.full((n_out,), float("nan"), device="cuda") if with_sdf else None
    pi_m = torch.full((P, 2), -3, dtype=I64, device="cuda")
    p = L.ptr
    args = (p(d[0]), p(d[1]) if with_sdf else None, p(d[2]), p(d[3]), p(d[4]) if with_sdf else None, L.c_i64(P), L.c_i32(nb), p(dep_m),
            p(sdf_m, allow_none=True), p(pi_m), L.stream_ptr())
    if n_live is None:
        L.check(L.lib().nsb_merge_sorted_vals(*args), "merge")
    else:
        _call(L.lib().nsb_merge_sorted_vals, "merge", counts_block(s5=n_live), 5, None, *args)
    live = P if n_live is None else n_live
    o_dep, o_sdf, o_pi = G.merge_vals(dep_a, sdf_a if with_sdf else None, pi_a[:live], dep_b[:live], sdf_b[:live] if with_sdf else None, n_out=n_out)
    same(dep_m, o_dep, "dep_m")
    if with_sdf:
        same(sdf_m, o_sdf, "sdf_m")
    same(pi_m[:live], o_pi, "pi_m")
    assert bool((pi_m[live:] == -3).all())


def test_merge_three_trips_per_warp():
    rng = np.random.default_rng(20)
    warps = 8 * 8 * sms() * 8
    P = 3 * warps + 5
    assert warp_trips(P, P) == (3, 4)
    lens = rng.integers(0, 41, P)
    lens[[0, 1, warps, 2 * warps + 1, P - 1]] = [0, 1, 0, 1, 40]
    dep_a, pi_a, dep_b = merge_inputs(rng, lens, 9)
    dep_b[::7, 2:5] = dep_b[::7, 2:3]                                          # ties inside b, trip after trip
    run_merge(dep_a, rng.standard_normal(dep_a.size).astype(np.float32), pi_a, dep_b, rng.standard_normal(dep_b.shape).astype(np.float32))


@pytest.mark.parametrize("nb", [1, 9, 32, 33, 1024])
def test_merge_row_lengths(nb):
    rng = np.random.default_rng(21)
    lens = np.array([0, 1, 2, 31, 32, 33, 64, 65, 200, 1, 0, 1500, 7] * 3)
    dep_a, pi_a, dep_b = merge_inputs(rng, lens, nb)
    sdf_a, sdf_b = np.arange(dep_a.size, dtype=np.float32), -np.arange(dep_b.size, dtype=np.float32).reshape(dep_b.shape) - 1
    run_merge(dep_a, sdf_a, pi_a, dep_b, sdf_b)
    run_merge(dep_a, sdf_a, pi_a, dep_b, sdf_b, with_sdf=False)


def test_merge_refuses_row_lengths_outside_1_to_1024():
    t = torch.zeros(4, device="cuda")
    pi = torch.tensor([[0, 1]], device="cuda")
    before = L.launch_count()
    for nb in (0, 1025):
        refused(L.lib().nsb_merge_sorted_vals(L.ptr(t), None, L.ptr(pi), L.ptr(t), None, L.c_i64(1), L.c_i32(nb), L.ptr(t), None, L.ptr(pi), L.stream_ptr()),
                "n_b must be in [1, 1024]")
    assert L.launch_count() == before


def test_merge_ties_carry_their_own_payloads():
    """every payload is distinct, so the place of each element of a tie is visible: a b equal to an a goes before it"""
    inf, tiny = np.float32(np.inf), np.float32(1e-45)
    packs = [
        ([1, 2, 2, 2, 3], [2, 2, 4]),                       # a b equal to several a
        ([1, 2, 3], [2, 2, 2]),                             # an a equal to several b
        ([5, 5, 5, 5], [5, 5, 5]),                          # a whole pack of one value
        ([0.0, 1], [-0.0, -0.0, 1]),                        # +0.0 in a against -0.0 in b
        ([-0.0, -0.0], [0.0, 0.0, 0.0]),                    # and the reverse
        ([-inf, -inf, inf], [-inf, inf, inf]),
        ([-tiny, 0.0, tiny, 2 * tiny], [-tiny, tiny, tiny]),
        ([], [1, 1, 2]),
        ([7], [7, 7, 7]),
    ]
    dep_a = np.array([v for a, _ in packs for v in a], np.float32)
    lens = np.array([len(a) for a, _ in packs])
    pi_a = np.stack([np.cumsum(lens) - lens, lens], 1)
    dep_b = np.array([b for _, b in packs], np.float32)
    sdf_a, sdf_b = 100 + np.arange(dep_a.size, dtype=np.float32), -np.arange(dep_b.size, dtype=np.float32).reshape(dep_b.shape) - 1
    run_merge(dep_a, sdf_a, pi_a, dep_b, sdf_b)
    run_merge(dep_a, sdf_a, pi_a, dep_b, sdf_b, with_sdf=False)
    o_dep, o_sdf, _ = G.merge_vals(dep_a, sdf_a, pi_a, dep_b, sdf_b)
    assert o_sdf[:8].tolist() == [100, -1, -2, 101, 102, 103, 104, -3]       # pack 0 written out: both b = 2 before the three a = 2


def test_merge_device_count_below_the_capacity():
    rng = np.random.default_rng(22)
    lens = rng.integers(0, 50, 3000)
    dep_a, pi_a, dep_b = merge_inputs(rng, lens, 9)
    sdf_a, sdf_b = rng.standard_normal(dep_a.size).astype(np.float32), rng.standard_normal(dep_b.shape).astype(np.float32)
    for live in (0, 1, 1777):
        b = dep_b.copy()
        b[live:] = np.nan                                                      # entries past the count: in-range pack infos, NaN depths
        run_merge(dep_a, sdf_a, pi_a, b, sdf_b, n_live=live)


# ================================================================================================ boundary assembly
def run_assemble(coarse, hit, fine, run_len, live=None, mid=True, ridx=True, mid_any_nan=False):
    R, nc = coarse.shape
    nf = fine.shape[1] if fine is not None else 0
    n_hit = 0 if hit is None else len(hit)
    S = R * nc + n_hit * nf
    pad = 64 * (nc + nf)                                    # slack behind every buffer and 64 more rows of fine: a kernel that miscounts the listed
    c, h = dev(coarse), (dev(np.asarray(hit, np.int64)) if n_hit else None)            # rays must give a wrong number, not touch foreign memory
    f = torch.full((n_hit + 64, max(nf, 1)), float("nan"), device="cuda") if n_hit else None
    if n_hit and nf:
        f[:n_hit] = dev(fine)
    d1 = torch.full((S + pad,), float("nan"), device="cuda")
    md = torch.full((S + pad,), float("nan"), device="cuda") if mid else None
    ra = torch.full((S + pad,), -1, dtype=I64, device="cuda") if ridx else None
    pi = torch.full((R, 2), -3, dtype=I64, device="cuda")
    runs = (ctypes.c_int32 * max(len(run_len), 1))(*run_len)
    p = L.ptr
    args = (p(c), L.c_i64(R), L.c_i32(nc), p(h, allow_none=True), L.c_i64(n_hit), p(f, allow_none=True), L.c_i32(nf), runs, L.c_i32(len(run_len)), p(d1),
            p(md, allow_none=True), p(ra, allow_none=True), p(pi), L.stream_ptr())
    if live is None:
        L.check(L.lib().nsb_assemble_boundary(*args), "assemble")
        o = G.assemble_boundary(coarse, hit, fine, run_len)
    else:
        _call(L.lib().nsb_assemble_boundary, "assemble", counts_block(s5=live[0], s6=live[1]), 5, 6, *args)
        o = G.assemble_boundary(coarse, hit, fine, run_len, n_rays=live[0], n_hit=live[1])
    Rl, Sl = o["pack_infos"].shape[0], o["d1"].size
    same(pi[:Rl], o["pack_infos"], "pack_infos")
    same(d1[:Sl], o["d1"], "d1")
    if mid:
        same(md[:Sl], o["mid"], "mid", any_nan=mid_any_nan)
    if ridx:
        same(ra[:Sl], o["ridx_all"], "ridx_all")
    assert bool((pi[Rl:] == -3).all()) and bool(d1[Sl:].isnan().all())       # nothing past the live rays is written
    assert (md is None or bool(md[Sl:].isnan().all())) and (ra is None or bool((ra[Sl:] == -1).all()))
    return o


def boundary_inputs(rng, R, nc, run_len, hit, scale=1.0):
    coarse = np.sort(scale * (0.5 + rng.random((R, nc))), -1).astype(np.float32)
    fine = np.concatenate([np.sort(scale * (0.4 + 1.2 * rng.random((len(hit), n))), -1) for n in run_len] + [np.zeros((len(hit), 0))], 1).astype(np.float32)
    return coarse, fine


def hit_patterns(R):
    r = np.arange(R)
    return {"none": r[:0], "every ray": r, "position 0 of every chunk": r[r % 8 == 0], "position 7 of every chunk": r[r % 8 == 7],
            "7 and 0 of neighbouring chunks": r[(r % 16 == 7) | (r % 16 == 8)], "all eight of every other chunk": r[(r // 8) % 2 == 1],
            "only the last ray": r[-1:], "only ray 0": r[:1]}


@pytest.mark.parametrize("R", [1, 7, 8, 9, 15, 16, 17, 701])
def test_assemble_chunk_edges(R):
    rng = np.random.default_rng(30 + R)
    for name, hit in hit_patterns(R).items():
        coarse, fine = boundary_inputs(rng, R, 5, [3, 4], hit)
        run_assemble(coarse, hit, fine, [3, 4])
    coarse, _ = boundary_inputs(rng, R, 5, [], [])
    run_assemble(coarse, None, None, [])                                       # n_hit = 0 with ridx_hit = fine = NULL


@pytest.mark.parametrize("nc,run_len", [(65, [51]), (65, [9, 9, 33]), (65, [8, 8, 32]), (65, [1, 32, 64, 33]), (65, [1] * 8), (65, []), (1, [9, 9, 33]),
                                        (1, []), (1, [1023]), (512, [256, 256])])
def test_assemble_run_layouts(nc, run_len):
    rng = np.random.default_rng(31)
    R = 41
    hit = np.sort(rng.choice(R, 17, replace=False))
    coarse, fine = boundary_inputs(rng, R, nc, run_len, hit)
    run_assemble(coarse, hit, fine, run_len)                                   # with run_len = []: hit rays that carry no fine sample
    run_assemble(coarse, hit, fine, run_len, mid=False, ridx=False)           # d1 and the pack infos do not depend on the optional outputs


def test_assemble_refuses_what_it_cannot_hold():
    t = torch.zeros(2048, device="cuda")
    i = torch.zeros(16, dtype=I64, device="cuda")

    def rc(nc, nf, runs):
        arr = (ctypes.c_int32 * max(len(runs), 1))(*runs)
        return L.lib().nsb_assemble_boundary(L.ptr(t), L.c_i64(1), L.c_i32(nc), L.ptr(i), L.c_i64(1), L.ptr(t), L.c_i32(nf), arr, L.c_i32(len(runs)), L.ptr(t),
                                             None, None, L.ptr(i), L.stream_ptr())
    before = L.launch_count()
    refused(rc(65, 960, [960]), "must be <= 1024")
    refused(rc(65, 9, [1] * 9), "at most 8 sorted runs")
    refused(rc(65, 51, [9, 9, 32]), "must add up to n_fine")
    refused(rc(0, 51, [51]), "must be <= 1024")
    assert L.launch_count() == before


def test_assemble_ties_keep_the_order_coarse_run0_run1():
    pz, nz = 0.0, -0.0
    rows = [
        ([1, 2, 3], [[2, 5], [2, 6], [0, 7]]),              # a fine sample equal to a coarse one, and equal in two runs
        ([1, 2, 3], [[2, 2], [2, 2], [2, 2]]),              # equal samples in three runs
        ([4, 4, 4], [[4, 4], [4, 4], [4, 4]]),              # a row of one value
        ([pz, 1, 2], [[nz, 1], [nz, 2], [pz, 3]]),          # +0.0 coarse against -0.0 fine: the stable order shows in the sign bit
        ([nz, nz, 2], [[pz, pz], [nz, pz], [nz, nz]]),      # and the reverse
        ([-np.inf, 0, np.inf], [[-np.inf, np.inf], [-np.inf, -np.inf], [np.inf, np.inf]]),
    ]
    coarse = np.array([c for c, _ in rows] + [[9, 9, 9]], np.float32)
    fine = np.array([np.concatenate(f) for _, f in rows], np.float32)
    o = run_assemble(coarse, np.arange(len(rows)), fine, [2, 2, 2], mid_any_nan=True)     # inf - inf between equal infinities
    assert o["d1"][27:36].view(np.uint32).tolist() == np.array([pz, nz, nz, pz, 1, 1, 2, 2, 3], np.float32).view(np.uint32).tolist()
    assert o["d1"][36:45].view(np.uint32).tolist() == np.array([nz, nz, pz, pz, nz, pz, nz, nz, 2], np.float32).view(np.uint32).tolist()


def test_assemble_mid_is_three_rounded_operations():
    rng = np.random.default_rng(32)
    R, nc, run_len = 600, 33, [9, 22]
    hit = np.sort(rng.choice(R, 300, replace=False))
    scale = (10.0 ** rng.uniform(-3, 3, (R, 1)))
    coarse = np.sort(scale * (0.5 + rng.random((R, nc))), -1).astype(np.float32)
    fine = np.concatenate([np.sort(scale[hit] * (0.4 + 1.2 * rng.random((hit.size, n))), -1) for n in run_len], 1).astype(np.float32)
    # x + d * 0.5 in one fused operation equals the three rounded ones whenever d * 0.5 is exact, i.e. unless it underflows: only
    # intervals whose half is not representable tell the two apart.  Rows of odd multiples of the smallest denormal:
    tiny = np.float32(1e-45)
    coarse[5] = np.cumsum(2 * np.arange(nc) + 1).astype(np.float32) * tiny
    coarse[6, :12] = (np.float32(1e-38) + np.cumsum(2 * np.arange(12) + 1).astype(np.float32) * tiny).astype(np.float32)
    o = run_assemble(coarse, hit, fine, run_len)
    d = o["d1"].astype(np.float64)
    pi = o["pack_infos"]
    inner = np.ones(d.size, bool)
    inner[pi[:, 0] + pi[:, 1] - 1] = False
    fused = (d + np.append(np.diff(d), 0) * 0.5).astype(np.float32)           # what one fused multiply-add would give
    assert (fused[inner] != o["mid"][inner]).sum() >= 10                      # the inputs tell the two apart


def test_assemble_production_shape():
    rng = np.random.default_rng(33)
    R = 60_000
    hit = np.flatnonzero(rng.random(R) < 0.4)
    coarse, fine = boundary_inputs(rng, R, 65, [9, 9, 33], hit)
    fine[:, 0] = coarse[hit, 7]                                                # a fine sample equal to a coarse one on every listed ray
    fine[:, 0:9].sort(-1)
    fine[:, 12] = fine[:, 2]                                                   # equal samples in two runs
    fine[:, 9:18].sort(-1)
    run_assemble(coarse, hit, fine, [9, 9, 33])


def test_assemble_three_trips_per_warp():
    rng = np.random.default_rng(34)
    warps = 8 * 8 * sms() * 8
    R = 3 * warps * 8 + 5
    assert warp_trips(R, R, items_per_warp=8) == (3, 4)
    hit = np.flatnonzero(rng.random(R) < 0.4)
    vals = (np.arange(16) / 8).astype(np.float32)                              # few values: ties in most rows
    coarse = np.sort(rng.choice(vals, (R, 2)), -1)
    fine = np.concatenate([np.sort(rng.choice(vals, (hit.size, 2)), -1), rng.choice(vals, (hit.size, 1))], 1)
    run_assemble(coarse, hit, fine, [2, 1])


def test_assemble_device_counts_below_the_capacity():
    rng = np.random.default_rng(35)
    R = 1000
    hit = np.flatnonzero(rng.random(R) < 0.5)
    coarse, fine = boundary_inputs(rng, R, 9, [4, 3], hit)
    for rays_live, hits_live in ((R, hit.size - 40), (613, int((hit < 613).sum())), (613, int((hit < 613).sum()) - 9), (8, 0), (0, 0)):
        f = fine.copy()
        f[hits_live:] = np.nan                                                 # past the counts: in-range ray indices, NaN depths
        run_assemble(coarse, hit, f, [4, 3], live=(rays_live, hits_live))


# ================================================================================================ compaction and the small kernels
def run_compact(lens, sel, alpha, *, d1=None, t=None, ridx_all=None, live=None, extra_out=3):
    lens = np.asarray(lens, np.int64)
    P = lens.size
    pi = np.stack([np.cumsum(lens) - lens, lens], 1)
    pack_of = np.repeat(np.arange(P), lens)
    kept = np.bincount(pack_of[sel != 0], minlength=P).astype(np.int32)
    if live is not None:
        kept[live:] = 0
    first = (np.cumsum(kept) - kept).astype(np.int32)
    K = int(kept.sum())
    o = G.compact_samples(sel, pi[:live], first, kept[:live], alpha, ridx_all=ridx_all, t=t, d1=d1, n_out=K + extra_out)
    outs = [torch.full((K + extra_out,), -1, dtype=I64, device="cuda") for _ in range(2)] + [torch.full((K + extra_out,), float("nan"), device="cuda") for _ in range(2)]
    p = L.ptr
    keep = [dev(x) for x in (sel, pi, first, kept, alpha)] + [dev(x) if x is not None else None for x in (ridx_all, t, d1)]
    args = (p(keep[0], "u8"), p(keep[1]), p(keep[2]), p(keep[3]), L.c_i64(P), p(keep[5], allow_none=True), p(keep[6], allow_none=True), p(keep[7], allow_none=True),
            p(keep[4]), *[p(x) for x in outs], L.stream_ptr())
    if live is None:
        L.check(L.lib().nsb_compact_samples(*args), "compact")
    else:
        _call(L.lib().nsb_compact_samples, "compact", counts_block(s5=live), 5, None, *args)
    for got, k in zip(outs, ("pidx", "ridx_c", "t_c", "alpha_c")):
        same(got, o[k], k)
    return o


def test_compact_pack_lengths_and_kept_patterns():
    rng = np.random.default_rng(40)
    lens = [0, 1, 31, 32, 33, 64, 65, 4096]
    pats = {"none": lambda k, n: k < 0, "all": lambda k, n: k >= 0, "first only": lambda k, n: k == 0, "last only": lambda k, n: k == n - 1,
            "lane 31 of chunk 0 and lane 0 of chunk 1": lambda k, n: (k == 31) | (k == 32), "every 33rd": lambda k, n: k % 33 == 0,
            "all kept before the pack ends": lambda k, n: k < np.minimum(n, 40) // 2}
    all_lens = np.array([n for _ in pats for n in lens])
    S = int(all_lens.sum())
    k = np.concatenate([np.arange(n) for n in all_lens])
    n_of = np.repeat(all_lens, all_lens)
    pat = np.repeat(np.arange(len(pats)), len(lens))
    which = np.repeat(pat, all_lens)
    sel = np.zeros(S, np.uint8)
    for j, f in enumerate(pats.values()):
        sel[(which == j) & f(k, n_of)] = 1
    sel[sel != 0] = rng.choice(np.array([1, 2, 0xFF], np.uint8), int((sel != 0).sum()))      # any non-zero byte keeps the sample
    alpha = rng.random(S).astype(np.float32)
    pos = 0.5 + np.cumsum(rng.random(S)).astype(np.float32)                   # ascending inside every pack
    run_compact(all_lens, sel, alpha, t=rng.random(S).astype(np.float32), ridx_all=rng.integers(0, 999, S))
    run_compact(all_lens, sel, alpha, d1=pos)                                 # the depth derived from d1, the ray from the pack


def test_compact_depth_from_d1_equals_the_assembled_mid():
    rng = np.random.default_rng(41)
    R = 500
    hit = np.flatnonzero(rng.random(R) < 0.4)
    coarse, fine = boundary_inputs(rng, R, 65, [9, 9, 33], hit)
    b = G.assemble_boundary(coarse, hit, fine, [9, 9, 33])
    S = b["d1"].size
    sel = (rng.random(S) < 0.3).astype(np.uint8)
    last = b["pack_infos"][:, 0] + b["pack_infos"][:, 1] - 1
    sel[last[::3]] = 1                                                         # the last sample of a pack: mid = its own depth
    o = run_compact(b["pack_infos"][:, 1], sel, rng.random(S).astype(np.float32), d1=b["d1"])
    K = int((sel != 0).sum())
    assert np.array_equal(o["t_c"][:K].view(np.uint32), b["mid"][sel != 0].view(np.uint32))
    assert np.array_equal(o["ridx_c"][:K], b["ridx_all"][sel != 0])


def test_compact_three_trips_per_warp_and_a_device_count():
    rng = np.random.default_rng(42)
    warps = 8 * 8 * sms() * 8
    P = 3 * warps + 5
    assert warp_trips(P, P) == (3, 4)
    lens = rng.integers(0, 70, P)
    lens[[0, warps, 2 * warps, 3 * warps, P - 1]] = 40
    S = int(lens.sum())
    pack_of = np.repeat(np.arange(P), lens)
    keeps = rng.random(P) < 0.25                                               # most packs keep nothing: the warp goes on to its next pack
    keeps[[0, warps, 2 * warps, 3 * warps, P - 1]] = True
    sel = ((rng.random(S) < 0.4) & keeps[pack_of]).astype(np.uint8)
    pos = 0.5 + np.cumsum(rng.random(S)).astype(np.float32)
    alpha = rng.random(S).astype(np.float32)
    run_compact(lens, sel, alpha, d1=pos)
    run_compact(lens, sel, alpha, d1=pos, live=2 * warps + 17)


def test_flag_scatter_gather_sizes_and_device_counts():
    rng = np.random.default_rng(43)
    p = L.ptr
    big = 3 * 8 * 8 * sms() * 256 + 77
    assert thread_trips(big) == (3, 4)
    for n in (1, 1000, big):
        v = rng.standard_normal(n).astype(np.float32) * (rng.random(n) < 0.5)
        v[:min(n, 6)] = np.array([-0.0, np.nan, np.inf, -np.inf, 1e-45, 0.0], np.float32)[:min(n, 6)]
        idx = rng.permutation(n + 5)[:n]                                        # unique targets in a destination of n + 5
        rays = [rng.standard_normal((n + 5, 3)).astype(np.float32) for _ in range(2)] + [rng.standard_normal(n + 5).astype(np.float32) for _ in range(2)]
        for live in (None, n // 3):
            m = n if live is None else live
            cnt = counts_block(s5=m)
            call = (lambda fn, what, *a: L.check(fn(*a), what)) if live is None else (lambda fn, what, *a: _call(fn, what, cnt, 5, None, *a))
            vd, flag = dev(v), torch.full((n,), -5, dtype=I32, device="cuda")
            call(L.lib().nsb_flag_nonzero, "flag", p(vd), L.c_i64(n), p(flag), L.stream_ptr())
            same(flag, G.flag_nonzero(v, m), "flag")                            # zero between the count and the capacity
            dst, src, ix = torch.zeros(n + 5, device="cuda"), dev(v), dev(idx)
            call(L.lib().nsb_scatter_f32, "scatter", p(src), p(ix), L.c_i64(n), p(dst), L.stream_ptr())
            same(dst, G.scatter_f32(v[:m], idx[:m], n + 5), "scatter")
            for cols in ((0, 1, 4, 7) if n < big else (4,)):
                extra = rng.standard_normal((n + 5, max(cols, 1))).astype(np.float32)
                ins = [dev(x) for x in rays] + [dev(extra)]
                outs = [torch.full((n, 3), float("nan"), device="cuda") for _ in range(2)] + [torch.full((n,), float("nan"), device="cuda") for _ in range(2)]
                ex_c = torch.full((n, max(cols, 1)), float("nan"), device="cuda")
                call(L.lib().nsb_gather_rays, "gather", p(ix), L.c_i64(n), *[p(x) for x in ins[:4]], *[p(x) for x in outs], p(ins[4]) if cols else None,
                     p(ex_c) if cols else None, L.c_i32(cols), L.stream_ptr())
                want = G.gather_rays(idx[:m], *rays, extra)
                for got, w in zip(outs + [ex_c] * (cols > 0), want):
                    same(got[:m], w, "gather")
                    assert bool(got[m:].isnan().all())
                assert cols or bool(ex_c.isnan().all())
    for fn, args in ((L.lib().nsb_flag_nonzero, (None, L.c_i64(0), None)), (L.lib().nsb_scatter_f32, (None, None, L.c_i64(0), None))):
        assert fn(*args, L.stream_ptr()) == 0                                   # n = 0: nothing to do, nothing read


CENTER, RADIUS = np.array([0.25, -0.5, 0.125], np.float32), np.array([1.0, 0.5, 2.0], np.float32)     # a non-cubic box, exact in fp32
CLIPS = [(None, None), (0.5, None), (0.5, 3.0)]


def run_ray_test(o, d, near, far, side=True):
    o, d = np.ascontiguousarray(o, np.float32).reshape(-1, 3), np.ascontiguousarray(d, np.float32).reshape(-1, 3)
    n = o.shape[0]
    od, dd = dev(o) if n else None, dev(d) if n else None
    outs = [torch.full((n, 3), 7.0, device="cuda") for _ in range(2)] + [torch.full((n,), 7.0, device="cuda") for _ in range(2)]
    flag = torch.full((n,), -5, dtype=I32, device="cuda")
    pr = torch.tensor([100, 55], dtype=I64, device="cuda")                      # pairs are added to; the row length is set
    p = L.ptr
    L.check(L.lib().nsb_ray_test_aabb(p(od, allow_none=True), p(dd, allow_none=True), L.c_i64(n), (ctypes.c_float * 3)(*CENTER), (ctypes.c_float * 3)(*RADIUS),
                                      ctypes.c_int(near is not None), L.c_f32(near or 0.), ctypes.c_int(far is not None), L.c_f32(far or 0.),
                                      *[p(x) if n else None for x in outs], p(flag) if n else None, p(pr) if side else None, p(pr[1:]) if side else None,
                                      L.stream_ptr()), "ray_test")
    g = G.ray_test_aabb(o, d, CENTER, RADIUS, near, far)
    for got, k in zip(outs + [flag], ("o_n", "d_n", "near", "far", "flag")):
        same(got, g[k], k, any_nan=k in ("o_n", "d_n"))                         # near / far: the kernel's own NaN, bit for bit
    if n:
        assert pr.tolist() == ([100 + g["coherent_pairs"], g["row_len"]] if side else [100, 55])
    return g


def world(o_n, d_n):
    """rays whose normalised form is exactly (o_n, d_n): the box's centre and radius are powers of two or sums of two"""
    return np.asarray(o_n, np.float32) * RADIUS + CENTER, np.asarray(d_n, np.float32) * RADIUS


@pytest.mark.parametrize("near,far", CLIPS)
def test_ray_test_edges(near, far):
    nan, inf = np.nan, np.inf
    cases = [
        ([-3, 0.5, 0.5], [1, 0.0, -0.0]),                   # direction components +0 and -0 inside their slabs
        ([-3, 0.5, 0.5], [1, -0.0, 0.0]),
        ([-3, 1.5, 0.5], [1, 0.0, 0.0]),                    # ... and outside one of them
        ([-1, 0.0, 0.0], [0.0, 1, 0]),                      # on the x = -1 slab with a zero x component: 0 / 0
        ([1, 0.0, 0.0], [-0.0, 0, 1]),
        ([0.25, 0.125, -0.375], [0.375, -0.5, 0.75]),       # origin inside
        ([-1, 0.25, 0.375], [1, 0.125, 0.125]),             # on a face, entering
        ([-1, 0.25, 0.375], [-1, 0.125, 0.125]),            # on a face, leaving
        ([-1, 1, -1], [1, -1, 1]),                          # on a corner, along the diagonal: zeros of both signs meet in the max
        ([-1, 1, -1], [-1, 1, -1]),
        ([-1, -1, -1], [1, 1, 1]),
        ([-2, -2, 0.0], [1, 1, 0.0]),                       # through the edge x = y = -1 ... = 1
        ([-2, 0.0, 0.0], [1, 1, 0.0]),                      # grazing the edge x = -1 .. y = 1: tf == tn
        ([-3, 0, 0], [1, 0, 0]), ([-3, 0, 0], [-1, 0, 0]),
        ([nan, 0, 0], [1, 0, 0]), ([0, 0, 0], [nan, 1, 0]), ([-3, 0, 0], [inf, 0, 0]), ([inf, 0, 0], [1, 0, 0]), ([-inf, 0, 0], [inf, 1, 1]),
        ([0, 0, 0], [0.0, 0.0, 0.0]), ([5, 5, 5], [-0.0, 0.0, -0.0]),
        ([-1.5, 0, 0], [1, 0, 0]),                          # tn = 0.5 = near_clip, tf = 2.5
        ([-2, 0, 0], [1, 0, 0]),                            # tn = 1, tf = 3 = far_clip
        ([0.5, 0, 0], [1, 0, 0]),                           # tf = 0.5 exactly near_clip: not valid with the near clip
        ([-4, 0, 0], [1, 0, 0]),                            # tn = 3 exactly far_clip: not valid with the far clip
        ([-4.5, 0, 0], [1, 0, 0]),
    ]
    o, d = world([c[0] for c in cases], [c[1] for c in cases])
    g = run_ray_test(o, d, near, far)
    want_o = np.array([c[0] for c in cases], np.float32)
    assert np.array_equal(g["o_n"][np.isfinite(want_o)], want_o[np.isfinite(want_o)])         # the set-up is exact: dyadic values only
    assert np.isnan(g["near"][3]) and np.isnan(g["far"][3]) and g["flag"][3] == 0 and np.isnan(g["far"][4])
    assert g["near"][12] == g["far"][12] and g["flag"][12] == 0
    k = len(cases) - 5
    assert (g["near"][k], g["far"][k + 1]) == (0.5, 3.0)
    assert g["flag"][k + 2] == (near is None) and g["flag"][k + 3] == (far is None) and g["far"][k + 2] == 0.5 and g["near"][k + 3] == 3.0
    for n in (0, 1, 2, 3):
        run_ray_test(o[:n], d[:n], near, far)
    run_ray_test(o, d, near, far, side=False)


def image_rays(W, H):
    x, y = np.meshgrid(np.arange(W) - W / 2 + 0.5, np.arange(H) - H / 2 + 0.5)
    d = np.stack([x.ravel(), y.ravel(), np.full(W * H, 8.0 * W)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return np.tile(np.array([0.1, -0.4, -5.0]), (W * H, 1)), d


def test_ray_test_row_length_and_neighbour_pairs():
    for W, H in ((2, 3), (3, 3), (8, 6), (800, 4), (64, 1)):
        o, d = image_rays(W, H)
        g = run_ray_test(o, d, 0.01, None)
        assert g["row_len"] == (W if H > 1 else -1) and (W < 8 or g["coherent_pairs"] == (W - 1) * H)
    o, d = image_rays(40, 30)
    perm = np.random.default_rng(44).permutation(1200)
    g = run_ray_test(o[perm], d[perm], 0.01, None)
    assert g["coherent_pairs"] < 300


def test_ray_test_three_trips_per_thread():
    rng = np.random.default_rng(45)
    n = 3 * 8 * 8 * sms() * 256 + 77
    assert thread_trips(n) == (3, 4)
    o = (rng.standard_normal((n, 3)) * 2).astype(np.float32)
    d = rng.standard_normal((n, 3)).astype(np.float32)
    d[::1001, 1] = 0
    g = run_ray_test(o, d, 0.5, 3.0)
    assert 0.02 < g["flag"].mean() < 0.9


def run_query_counts(cnt, phase, nc, n_fine, march_cap, kept_cap):
    nf = (ctypes.c_int32 * max(len(n_fine), 1))(*n_fine)
    return L.lib().nsb_query_counts(L.ptr(cnt), L.c_i32(phase), L.c_i32(nc), nf, L.c_i32(len(n_fine)), L.c_i64(march_cap), L.c_i64(kept_cap), L.stream_ptr())


def test_query_counts():
    base = np.arange(1000, 1032, dtype=np.int64)
    base[[0, 3, 4, 6, 7, 20]] = [48_000, 700_000, 20_000, 333_333, 15_000, 0]
    for n_fine in ([], [16], [9, 33], [9, 9, 33], [1, 32, 64, 33]):
        worst = 700_000 + 20_000 * sum(n_fine[:-1])
        for march_cap in (worst - 1, worst, worst + 1):
            for K in (333_332, 333_333, 333_334):
                cnt = dev(base)
                L.check(run_query_counts(cnt, 0, 65, n_fine, march_cap, 0), "query_counts")
                want = G.query_counts(base, 0, 65, n_fine, march_cap, 0)
                assert cnt.tolist() == want.tolist() and want[20] == (march_cap < worst) and (want[12] == 0) == (march_cap < worst)
                L.check(run_query_counts(cnt, 1, 65, n_fine, 0, K), "query_counts")           # bit 1 after bit 0: OR-ed into the same slot
                want = G.query_counts(want, 1, 65, n_fine, 0, K)
                assert cnt.tolist() == want.tolist() and want[20] == (march_cap < worst) + 2 * (K < 333_333)
                assert [want[k] for k in (1, 2, 5, 8, 9, 10, 11, 27, 28, 29, 30, 31)] == [base[k] for k in (1, 2, 5, 8, 9, 10, 11, 27, 28, 29, 30, 31)]
    cnt = dev(base)
    refused(run_query_counts(cnt, 0, 65, [1, 2, 3, 4, 5], 10 ** 9, 0), "at most 4 up-sampling stages")
    assert cnt.tolist() == base.tolist()
