"""The ray-tiled SDF query (k_fused_sdf_tc<2>, csrc/fused_tc.cu: gather warps hand A tiles over a ring of shared-memory slots to a wgmma
consumer warpgroup) against the ray-major query (mode 1) on the same samples, bit for bit: a point's sdf does not depend on which tile,
slot or row it is evaluated in.  Covered: packs of 0..116 samples and one far longer ray, pack counts that are not a multiple of 32, the
block order and none, a device count below the capacity (CTAs with no group), rings that wrap many times, 1, 5, 12 and 16 levels with and
without max_level, and the occupancy collection (its grid bit-equal too)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import scene as oscene
from test_partial_levels_gpu import _model

pytestmark = pytest.mark.gpu


def _query(model, rays_o, rays_d, t, max_level, *, ridx=None, packs=None, collect_res=None, count=None):
    """sdf of the samples t (NaN where the launch writes nothing), and the collected occupancy grid (or None)"""
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.fields.networks import sdf_fwd
    s = model.implicit_surface
    grid16, dec = s._fused_state()
    sdf = torch.full((t.numel(),), float("nan"), device="cuda")
    pcl = coll = None
    if collect_res is not None:
        pcl = torch.zeros(collect_res, dtype=torch.float32, device="cuda")
        coll = L.OccCollectC(pcl.data_ptr(), (ctypes.c_int32 * 3)(*collect_res), 3.5)
    ml = s._ml(max_level)
    sdf_fwd(s.encoding.meta, grid16, dec, sdf, ml, rays_o=rays_o, rays_d=rays_d, t=t, ridx=ridx, packs=packs, collect=coll, count=count)
    torch.cuda.synchronize()
    return sdf, pcl


def _samples(counts, seed, H=None, W=None):
    """packs of the given sample counts on camera rays through the box (one pinhole view when H, W are given), t ascending in each pack;
    -> rays_o, rays_d, pack_infos [n, 2], pack_ray [n], t, ridx (the ray of every sample)"""
    g = torch.Generator().manual_seed(seed)
    n = len(counts)
    if H is None:
        H, W = 1, n
    ro, rd = oscene.pinhole_rays(H, W, oscene.orbit_camera(seed % 8, 8, radius=3.0, elev_deg=25.0))
    R = ro.shape[0]
    ray = torch.randperm(R, generator=g)[:n] if n <= R else torch.randint(0, R, (n,), generator=g)
    cnt = torch.as_tensor(counts, dtype=torch.int64)
    first = cnt.cumsum(0) - cnt
    total = int(cnt.sum())
    u = torch.rand(total, generator=g)
    pid = torch.repeat_interleave(torch.arange(n), cnt)
    k = torch.arange(total) - first[pid]
    t = 1.6 + 2.8 * (k.float() + u) / cnt[pid].clamp(min=1).float()              # inside [1.6, 4.4]: the box seen from radius 3
    pinfo = torch.stack([first, cnt], 1)
    return (ro.cuda().contiguous(), rd.cuda().contiguous(), pinfo.cuda(), ray.cuda(), t.cuda().contiguous(), ray[pid].cuda().contiguous())


def _assert_bit_equal(a, b):
    assert a.shape == b.shape
    same = (a.view(torch.int32) == b.view(torch.int32))
    assert bool(same.all()), f"{int((~same).sum())} of {a.numel()} differ"


def _compare(model, counts, seed, *, max_level=None, order=False, live=None, collect_res=None, H=None, W=None):
    ro, rd, pinfo, pray, t, ridx = _samples(counts, seed, H, W)
    n = pinfo.shape[0]
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed + 1)).cuda() if order else None
    count = None
    if live is not None:                                   # the launch is sized for n packs; the device count says `live`
        cnt = torch.tensor([live], dtype=torch.int64, device="cuda")
        count = (cnt, 0)
    got, pcl2 = _query(model, ro, rd, t, max_level, packs=(pinfo, pray, perm), collect_res=collect_res, count=count)
    # the oracle: mode 1 on the samples of the packs the launch covers (packs order[:live] or [:live])
    covered = torch.ones(n, dtype=torch.bool, device="cuda")
    if live is not None:
        covered[:] = False
        covered[perm[:live] if order else torch.arange(live, device="cuda")] = True
    sel = torch.nonzero(torch.repeat_interleave(covered, pinfo[:, 1])).view(-1)     # the samples of the covered packs (packs are contiguous)
    ref_sel, pcl1 = _query(model, ro, rd, t[sel].contiguous(), max_level, ridx=ridx[sel].contiguous(), collect_res=collect_res)
    want = torch.full_like(got, float("nan"))
    want[sel] = ref_sel
    _assert_bit_equal(got, want)
    assert torch.isfinite(got[sel]).all()
    if collect_res is not None:
        _assert_bit_equal(pcl2, pcl1)
        assert float(pcl1.max()) > 0
    return got


@pytest.fixture(scope="module")
def models():
    return {L: _model(L, seed=100 + L) for L in (1, 5, 12, 16)}


EDGE_COUNTS = [0, 1, 3, 4, 5, 65, 116]


@pytest.mark.parametrize("order", [False, True])
def test_edge_pack_sizes(cuda, models, order):
    """every edge size in every lane position; 7 * 11 + 2 packs: not a multiple of 32"""
    counts = (EDGE_COUNTS * 11 + [116, 0])
    _compare(models[16], counts, seed=3, order=order)


@pytest.mark.parametrize("L,max_level", [(1, None), (5, None), (5, 2), (12, None), (12, 7), (16, None), (16, 9)])
def test_levels(cuda, models, L, max_level):
    rng = np.random.default_rng(L)
    counts = rng.choice(EDGE_COUNTS, 517).tolist()
    _compare(models[L], counts, seed=L, max_level=max_level, order=True)


def test_ring_wraps_many_times(cuda, models):
    """about 40 groups per CTA of 116-sample rays: every CTA's ring of slots is reused hundreds of times"""
    n = 132 * 32 * 40 + 13
    rng = np.random.default_rng(5)
    counts = np.where(rng.random(n) < 0.9, 116, rng.integers(0, 117, n)).tolist()
    _compare(models[16], counts, seed=7, order=True, H=400, W=600)


@pytest.mark.parametrize("order", [False, True])
@pytest.mark.parametrize("live", [0, 1, 40, 3001])
def test_device_count_below_capacity(cuda, models, order, live):
    """the grid is sized for the capacity (up to one CTA per SM); with a small live count most CTAs get no group"""
    rng = np.random.default_rng(live)
    counts = rng.choice(EDGE_COUNTS, 6000).tolist()
    _compare(models[12], counts, seed=11, order=order, live=live)


@pytest.mark.parametrize("L", [12, 16])
def test_occupancy_collection(cuda, models, L):
    rng = np.random.default_rng(17)
    counts = rng.choice(EDGE_COUNTS, 2500).tolist()
    _compare(models[L], counts, seed=13, order=True, collect_res=(32, 32, 32))


def test_long_ray(cuda, models):
    """one ray whose max_n (5003 samples) is far past any per-ray buffer, among short ones"""
    counts = [3, 5003, 0, 116] + [1] * 40
    _compare(models[16], counts, seed=19, order=False)


def test_frame_scale_view(cuda, models):
    """the boundary samples of a 400 x 300 view (65 + 51 per ray, 13.9 M points) in the 8 x 4 pixel-block order"""
    H, W = 300, 400
    n = H * W
    py, px = np.arange(n) // W, np.arange(n) % W
    blk = np.lexsort(((py % 4) * 8 + px % 8, px // 8, py // 4))
    ro, rd = oscene.pinhole_rays(H, W, oscene.orbit_camera(2, 8, radius=3.0, elev_deg=25.0))
    ro, rd = ro.cuda().contiguous(), rd.cuda().contiguous()
    cnt = torch.full((n,), 116, dtype=torch.int64)
    first = cnt.cumsum(0) - cnt
    g = torch.Generator().manual_seed(23)
    t = (1.6 + 2.8 * (torch.arange(116).float()[None, :] + torch.rand(n, 116, generator=g)) / 116).reshape(-1).cuda().contiguous()
    pinfo = torch.stack([first, cnt], 1).cuda()
    order = torch.from_numpy(blk).cuda()
    got, _ = _query(models[16], ro, rd, t, None, packs=(pinfo, None, order))
    ridx = torch.arange(n, device="cuda").repeat_interleave(116)
    want, _ = _query(models[16], ro, rd, t, None, ridx=ridx)
    _assert_bit_equal(got, want)
