"""The occupancy-grid marcher (csrc/march.cu) at street-scale grids and launch edges, every check bit-exact.

* The single-grid and batched kernels and oracle/march.c against the reference's own kernels (oracle/_ref/_occ_grid, digests in
  tests/golden/ref__occ_grid_edges.npz): cfg3's street box with ego cameras and a LiDAR inside it, exact +-0.0 direction components,
  axis-parallel rays, origins on a face / edge / corner, rays on a roi face, grids on both sides of the shared-memory limit, dt_gamma
  with max_step_size clamping, rays capped at max_steps, five batched grids with distinct rois, and a 1920 x 1280 frame.
* The global-memory march against the shared-memory one, the listed rounds as the NeuS query calls them (march_args / march_listed),
  the recorded march on a global-memory grid, nsb_pack_occ_bits, and the one-launch step on a grid above the shared-memory limit.
* The float64 meaning checks of tests/march64.py on the kernel's samples."""
import numpy as np
import pytest
import torch

import march64
import march_cases as mc
from oracle import march as omarch
from refgold import Golden

pytestmark = pytest.mark.gpu
SMEM_CELLS = 96 * 1024 * 8          # the largest grid the marcher keeps in shared memory (bits)


@pytest.fixture(scope="module")
def gold():
    G = Golden("_occ_grid_edges", "_occ_grid")
    yield G
    G.save()


@pytest.fixture(scope="module")
def street():
    return mc.street_rays()


def _on(xs, cuda):
    return tuple(x.to(cuda) for x in xs)


def _oracle_outputs(c, batched=False):
    """oracle/march.py's outputs in the layout and shapes of the binding's: t as [M, 1]; batched: (.., ridx, bidx, gidx)"""
    out = [c[0], c[1].unsqueeze(-1), c[2].unsqueeze(-1), c[3]]
    return out + ([c[5], c[4]] if batched else [c[4]])


def _pin(G, key, ours, ref_fn, oracle=None):
    """every output of ours (and of the oracle) bit for bit the reference's ref_fn(module) -- run once per key when recording"""
    cache = []

    def ref(k):
        if not cache:
            cache.append([t.detach().clone() for t in ref_fn(G.ref)])
        return cache[0][k]
    for outs in (ours, oracle) if oracle is not None else (ours,):
        for k, y in enumerate(outs):
            G.equal(f"{key}.out{k}", y, lambda _m, k=k: ref(k))


@pytest.mark.parametrize("case", mc.SINGLE, ids=[c[0] for c in mc.SINGLE])
def test_single_grid_against_reference(cuda, gold, street, case):
    from neuralsim_b200.bindings import _occ_grid as ours
    name, kind, res, roi, gamma, dt_max, max_steps = case
    grid, roi = mc.grid(kind, res), torch.tensor(roi)
    args = (*_on(street, cuda), roi.to(cuda), grid.to(cuda))
    got = ours.ray_marching(*args, ours.ContractionType.AABB, mc.STEP, dt_max, gamma, max_steps, True)
    c = omarch.ray_marching(*street, roi, grid, mc.STEP, dt_max, gamma, max_steps)
    _pin(gold, name, got, lambda ref: ref.ray_marching(*args, ref.ContractionType.AABB, mc.STEP, dt_max, gamma, max_steps, True),
         _oracle_outputs(c))
    cnt = got[0][:, 1]
    if kind == "empty":
        assert got[1].shape[0] == 0
    else:
        assert int(cnt.sum()) > 0
    if max_steps < mc.MAX_STEPS:
        assert int((cnt == max_steps).sum()) > 1000                           # rays that reach max_steps exactly


@pytest.mark.parametrize("layout", ["batch_inds", "batch_data_size"])
def test_batched_against_reference(cuda, gold, street, layout):
    """five grids with distinct rois; gidx is flat over [B, X, Y, Z] (batched_marching.cu:62,115)"""
    from neuralsim_b200.bindings import _occ_grid as ours
    grid, rois = mc.batched_grid(mc.SMALL)
    B = grid.shape[0]
    R = street[0].shape[0] // B * B
    o, d, n, f = (x[:R].contiguous() for x in street)
    if layout == "batch_inds":
        bi, bds, gamma, dt_max = torch.from_numpy(np.random.default_rng(9).integers(0, B, R)).int(), None, 0.0, 1e10
    else:
        bi, bds, gamma, dt_max = None, R // B, 0.01, 1.0
    args = (*_on((o, d, n, f), cuda), None if bi is None else bi.to(cuda), bds, rois.to(cuda), grid.to(cuda))
    got = ours.batched_ray_marching(*args, ours.ContractionType.AABB, mc.STEP, dt_max, gamma, mc.MAX_STEPS, True)
    bic = bi if bi is not None else (torch.arange(R) // bds).int()
    c = omarch.ray_marching(o, d, n, f, rois, grid, mc.STEP, dt_max, gamma, mc.MAX_STEPS, batch_inds=bic)
    _pin(gold, f"batched_{layout}", got,
         lambda ref: ref.batched_ray_marching(*args, ref.ContractionType.AABB, mc.STEP, dt_max, gamma, mc.MAX_STEPS, True), _oracle_outputs(c, True))
    bidx, gidx = got[4], got[5]
    assert int(bidx.max()) == B - 1 and bool((gidx // grid[0].numel() == bidx).all())


def test_frame_against_reference(cuda, gold):
    """a 1920 x 1280 frame from inside the street box on a global-memory grid: the whole frame against the reference, 1/16 of its rays
    against the C oracle"""
    from neuralsim_b200.bindings import _occ_grid as ours
    rays = mc.frame_rays()
    R = rays[0].shape[0]
    grid, roi = mc.grid("blocks", mc.LARGE), torch.tensor(mc.ROI)
    assert R == 1920 * 1280 and grid.numel() > SMEM_CELLS
    args = (*_on(rays, cuda), roi.to(cuda), grid.to(cuda))
    got = ours.ray_marching(*args, ours.ContractionType.AABB, mc.STEP, 1e10, 0.0, mc.MAX_STEPS, True)
    _pin(gold, "frame", got, lambda ref: ref.ray_marching(*args, ref.ContractionType.AABB, mc.STEP, 1e10, 0.0, mc.MAX_STEPS, True))
    sub = torch.arange(0, R, 16)
    c = omarch.ray_marching(*(x[sub].contiguous() for x in rays), roi, grid, mc.STEP, 1e10, 0.0, mc.MAX_STEPS)
    info = got[0].cpu()
    cnt = info[sub, 1]
    assert torch.equal(cnt, c[0][:, 1])
    rows = torch.repeat_interleave(info[sub, 0].long() - c[0][:, 0].long(), cnt.long()) + torch.arange(int(cnt.sum()))
    assert torch.equal(got[1].squeeze(-1).cpu()[rows], c[1]) and torch.equal(got[2].squeeze(-1).cpu()[rows], c[2])
    assert torch.equal(got[3].cpu()[rows].long(), sub[c[3].long()]) and torch.equal(got[4].cpu()[rows], c[4])


@pytest.mark.parametrize("case", ["small_blocks_gamma", "small_checker", "smem_edge_blocks", "roi_face_full"])
def test_global_memory_equals_shared_memory(cuda, street, case):
    """the batched entry with B = 1 always reads the grid from global memory; on a grid that fits shared memory it must give the
    single-grid march's outputs"""
    from neuralsim_b200.bindings import _occ_grid as ours
    _, kind, res, roi, gamma, dt_max, max_steps = next(c for c in mc.SINGLE if c[0] == case)
    grid, roi = mc.grid(kind, res).to(cuda), torch.tensor(roi, device=cuda)
    assert grid.numel() <= SMEM_CELLS
    rays = _on(street, cuda)
    a = ours.ray_marching(*rays, roi, grid, ours.ContractionType.AABB, mc.STEP, dt_max, gamma, max_steps, True)
    bi = torch.zeros(rays[0].shape[0], dtype=torch.int32, device=cuda)
    b = ours.batched_ray_marching(*rays, bi, None, roi.view(1, 6), grid[None].contiguous(), ours.ContractionType.AABB, mc.STEP, dt_max, gamma,
                                  max_steps, True)
    for k, (x, y) in enumerate(zip(a, [b[0], b[1], b[2], b[3], b[5]])):
        assert torch.equal(x, y), k
    assert int(b[4].abs().sum()) == 0


def _scan(num):
    num = num.int()
    return torch.stack([num.cumsum(0, dtype=torch.int32) - num, num], -1).contiguous()


@pytest.mark.parametrize("packed", [False, True], ids=["grid", "grid_bits"])
def test_listed_rounds(cuda, street, packed):
    """the two rounds as the NeuS query calls them (march_args / march_listed: t_ends, gidx and bidx NULL), on output buffers
    prefilled with sentinels"""
    from neuralsim_b200.bindings import _occ_grid as ours
    from neuralsim_b200.graphics import neus_fused as NF
    o, d, n, f = _on(street, cuda)
    R = o.shape[0]
    grid, roi = mc.grid("blocks", mc.SMALL).to(cuda), torch.tensor(mc.ROI, device=cuda)
    ref = ours.ray_marching(o, d, n, f, roi, grid, ours.ContractionType.AABB, mc.STEP, 1e10, 0.0, mc.MAX_STEPS, True)
    want_n, want_t, want_r = ref[0][:, 1], ref[1].squeeze(-1), ref[3]
    M = want_t.shape[0]
    margs = NF.march_args(o, d, n, f, roi, grid, mc.STEP, 1e10, 0.0, mc.MAX_STEPS)
    bits = NF.pack_occ_bits(grid) if packed else None
    # first round with a device-resident ray count: rows past it read 0, nothing past R is written
    for n_live in (0, 1, R - 37, R):
        num = torch.full((R + 64,), -5, dtype=torch.int32, device=cuda)
        NF.march_listed(margs, bits, num_steps=num, count=(torch.tensor([n_live], dtype=torch.int64, device=cuda), 0))
        assert torch.equal(num[:n_live], want_n[:n_live]), n_live
        assert int(num[n_live:R].abs().sum()) == 0 and bool((num[R:] == -5).all()), n_live
    # second round over a shuffled list of the rays with samples
    info2 = _scan(want_n)
    hit = torch.nonzero(want_n).flatten()
    lst = hit[torch.randperm(hit.numel(), generator=torch.Generator().manual_seed(3)).to(cuda)].contiguous()
    t, r = torch.full((M + 8,), -7.0, device=cuda), torch.full((M + 8,), -7, dtype=torch.int32, device=cuda)
    NF.march_listed(margs, bits, info2=info2, t_starts=t, ridx=r, ray_list=lst, n_list=lst.numel())
    assert torch.equal(t[:M], want_t) and torch.equal(r[:M], want_r)
    assert bool((t[M:] == -7.0).all()) and bool((r[M:] == -7).all())
    # ... with a device count below the list's length: only the first k listed rays are written
    k = lst.numel() // 3
    t.fill_(-7.0); r.fill_(-7)
    NF.march_listed(margs, bits, info2=info2, t_starts=t, ridx=r, ray_list=lst, n_list=lst.numel(),
                    count=(torch.tensor([k], dtype=torch.int64, device=cuda), 0))
    w = torch.isin(want_r.long(), lst[:k])
    assert torch.equal(t[:M][w], want_t[w]) and torch.equal(r[:M][w], want_r[w])
    assert bool((t[:M][~w] == -7.0).all()) and bool((t[M:] == -7.0).all())
    # ... with packed counts below the first round's: each ray's first counts (the packed count is the cap, as the reference's);
    # the buffers hold M samples, so that no write can leave them
    less = want_n // 2
    info2 = _scan(less)
    M2 = int(less.sum())
    t.fill_(-7.0); r.fill_(-7)
    hit2 = torch.nonzero(less).flatten().contiguous()
    NF.march_listed(margs, bits, info2=info2, t_starts=t, ridx=r, ray_list=hit2, n_list=hit2.numel())
    pos = torch.arange(M, device=cuda) - ref[0][want_r.long(), 0]
    keep = pos < less[want_r.long()]
    assert torch.equal(t[:M2], want_t[keep]) and torch.equal(r[:M2], want_r[keep])
    assert bool((t[M2:] == -7.0).all()) and bool((r[M2:] == -7).all())


def test_recorded_march_on_global_memory_grid(cuda, street):
    """nsb_ray_marching_record (k_ray_marching<false, true>) + nsb_march_compact == the two-round march, on a grid above the
    shared-memory limit"""
    import ctypes
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.bindings import _occ_grid as ours
    sel = torch.arange(0, street[0].shape[0], 17)
    o, d, n, f = _on((x[sel].contiguous() for x in street), cuda)
    R, max_steps = o.shape[0], 1024
    grid, roi = mc.grid("blocks", mc.LARGE).to(cuda), torch.tensor(mc.ROI, device=cuda)
    assert grid.numel() > SMEM_CELLS
    ref = ours.ray_marching(o, d, n, f, roi, grid, ours.ContractionType.AABB, mc.STEP, 1e10, 0.0, max_steps, False)
    lib, P = L.lib(), L.ptr
    num = torch.full((R,), -1, dtype=torch.int32, device=cuda)
    rec = torch.full((R * max_steps,), float("nan"), device=cuda)
    L.check(lib.nsb_ray_marching_record(L.c_i64(R), P(o), P(d), P(n), P(f), P(roi), L.c_i32(grid.shape[0]), L.c_i32(grid.shape[1]),
                                        L.c_i32(grid.shape[2]), P(grid.view(torch.uint8)), L.c_f32(mc.STEP), L.c_f32(1e10), L.c_f32(0.0),
                                        ctypes.c_uint32(max_steps), P(num), P(rec), None, L.stream_ptr()), "record")
    assert torch.equal(num, ref[0][:, 1])
    hit = torch.nonzero(num).flatten().contiguous()
    M = int(num.sum())
    t, ridx = torch.full((M + 8,), -7.0, device=cuda), torch.full((M + 8,), -7, dtype=torch.int32, device=cuda)
    L.check(lib.nsb_march_compact(P(rec), ctypes.c_uint32(max_steps), P(_scan(num)), P(hit), L.c_i64(hit.numel()), P(t), P(ridx),
                                  L.stream_ptr()), "compact")
    assert torch.equal(t[:M], ref[1].squeeze(-1)) and torch.equal(ridx[:M], ref[3])
    assert bool((t[M:] == -7.0).all()) and bool((ridx[M:] == -7).all())


@pytest.mark.parametrize("res", [mc.SMALL, mc.LARGE, (3, 5, 7)], ids=str)
def test_pack_occ_bits(cuda, res):
    """nsb_pack_occ_bits against a torch packing (cell c -> bit c % 32 of word c / 32) on cell counts that are not multiples of 32"""
    from neuralsim_b200.graphics import neus_fused as NF
    g = torch.from_numpy(np.random.default_rng(4).random(res) < 0.4)
    cells = g.numel()
    assert cells % 32 != 0
    flat = torch.zeros((cells + 31) // 32 * 32, dtype=torch.int64)
    flat[:cells] = g.reshape(-1).long()
    want = (flat.view(-1, 32) << torch.arange(32)).sum(-1)
    want = torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()
    assert torch.equal(NF.pack_occ_bits(g.to(cuda)).cpu(), want)


@pytest.mark.parametrize("case", ["small_blocks_gamma", "large_checker", "small_full_cap", "batched"])
def test_kernel_samples_mean_what_they_should(cuda, case):
    """tests/march64.py's float64 checks on the kernel's samples"""
    from neuralsim_b200.bindings import _occ_grid as ours
    rays = mc.street_rays(n_azim=250, cam_hw=(24, 32), n_axis=32, n_boundary=64)
    if case == "batched":
        grid, rois = mc.batched_grid(mc.SMALL)
        bi = torch.from_numpy(np.random.default_rng(5).integers(0, grid.shape[0], rays[0].shape[0])).int()
        got = ours.batched_ray_marching(*_on(rays, cuda), bi.to(cuda), None, rois.to(cuda), grid.to(cuda), ours.ContractionType.AABB, mc.STEP,
                                        1.0, 0.01, mc.MAX_STEPS, True)
        march64.check(*rays, rois, grid, mc.STEP, 1.0, 0.01, mc.MAX_STEPS, *got[:4], got[5], batch_inds=bi, bidx=got[4])
        return
    _, kind, res, roi, gamma, dt_max, max_steps = next(c for c in mc.SINGLE if c[0] == case)
    grid, roi = mc.grid(kind, res), torch.tensor(roi)
    got = ours.ray_marching(*_on(rays, cuda), roi.to(cuda), grid.to(cuda), ours.ContractionType.AABB, mc.STEP, dt_max, gamma, max_steps, True)
    march64.check(*rays, roi, grid, mc.STEP, dt_max, gamma, max_steps, *got)


@pytest.mark.parametrize("onepass", ["0", "1"], ids=["two_rounds", "recorded"])
def test_static_step_on_global_memory_grid(cuda, monkeypatch, onepass):
    """a model whose occupancy grid is above the shared-memory limit: the one-launch step's march (either form) gives march_lean's
    samples, and the step renders the host-sized step's images and buffers bit for bit"""
    from neuralsim_b200.graphics import neus_static as NS
    from neuralsim_b200.graphics.neus_fused import march_lean
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from oracle import scene as oscene
    from util import make_pair
    monkeypatch.setattr(NS, "MARCH_ONEPASS", onepass)
    _, model = make_pair(cuda)
    model.accel.occ.set_occ_grid(oscene.make_occ_grid(100).to(cuda))
    assert model.accel.occ.occ_grid.numel() > SMEM_CELLS
    ro, rd = oscene.pinhole_rays(36, 48, oscene.orbit_camera(1, 8, radius=3.0, elev_deg=25.0))
    ro, rd = ro.to(cuda), rd.to(cuda)
    ha = torch.zeros(ro.shape[0], 4, device=cuda)
    model.train()
    with torch.no_grad():
        ref = SingleVolumeRenderer(dict(near=0.01)).train().render(model, ro, rd, rays_h_appear=ha, return_buffer=True, return_details=True)
        rt = ref["ray_tested"]
        lean = march_lean(model.accel.occ.occ_grid, rt["rays_o"].contiguous(), rt["rays_d"].contiguous(), rt["near"].contiguous(),
                          rt["far"].contiguous(), step_size=0.005, max_steps=4096)          # make_pair's march_cfg
        rendered, cnt, buffers = NS.render_static(model, ro, rd, ha, near=0.01, march_cap=1 << 19, kept_cap=1 << 17)
    c = cnt.tolist()
    assert c[20] == 0 and c[0] == rt["num_rays"]
    assert c[3] == lean[2].shape[0] == int(ref["details"]["march.num_per_ray"].sum()) and c[4] == lean[0].shape[0]
    for k in ("rgb_volume", "depth_volume", "normals_volume", "mask_volume"):
        assert torch.equal(rendered[k], ref["rendered"][k]), k
    vb = NS.sliced_volume_buffer(buffers, cnt)
    for k in ("t", "opacity_alpha", "rgb", "nablas", "rays_inds_hit", "pack_infos_hit"):
        assert torch.equal(vb[k], ref["volume_buffer"][k]), k
