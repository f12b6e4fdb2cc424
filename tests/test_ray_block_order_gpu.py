"""The 8 x 4 pixel-block order of the ray-tiled SDF query (csrc/neus_glue.cu: k_ray_block_order, the row length of k_ray_test_aabb):
a permutation of the live packs that changes which samples share a gather instruction and nothing else, so every sdf and every
rendered image stays bit-equal to the strip order and to the ray-major query."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import scene as oscene
from util import make_pair

pytestmark = pytest.mark.gpu
KEYS = ("rgb_volume", "depth_volume", "normals_volume", "mask_volume")


def _rays(H, W, k=1, radius=3.0):
    ro, rd = oscene.pinhole_rays(H, W, oscene.orbit_camera(k, 8, radius=radius, elev_deg=25.0))
    return ro.cuda().contiguous(), rd.cuda().contiguous()


def _ray_test(ro, rd):
    """nsb_ray_test_aabb against the box [-1, 1]^3 -> (flag, int64[2] = (coherent neighbour pairs, row length))"""
    from neuralsim_b200 import _lib as L
    R = ro.shape[0]
    o_n, d_n = torch.empty(R, 3, device="cuda"), torch.empty(R, 3, device="cuda")
    nr, fr = torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
    flag = torch.empty(R, dtype=torch.int32, device="cuda")
    pairs = torch.zeros(2, dtype=torch.int64, device="cuda")
    c3, r3 = (ctypes.c_float * 3)(0., 0., 0.), (ctypes.c_float * 3)(1., 1., 1.)
    L.check(L.lib().nsb_ray_test_aabb(L.ptr(ro, "f32"), L.ptr(rd, "f32"), L.c_i64(R), c3, r3, ctypes.c_int(1), L.c_f32(0.01), ctypes.c_int(0),
                                      L.c_f32(0.), L.ptr(o_n), L.ptr(d_n), L.ptr(nr), L.ptr(fr), L.ptr(flag), L.ptr(pairs), L.ptr(pairs[1:]),
                                      L.stream_ptr()), "ray_test_aabb")
    return flag, pairs


def _expected_order(pix, W):
    """the packs (ascending pixels) sorted by (py / 4, px / 8, (py % 4) 8 + px % 8)"""
    py, px = pix // W, pix % W
    return np.lexsort(((py % 4) * 8 + px % 8, px // 8, py // 4))


@pytest.mark.parametrize("H,W", [(5, 800), (3, 801), (20, 7)])
def test_row_length_is_found(cuda, H, W):
    ro, rd = _rays(H, W, radius=1.5)
    _, pairs = _ray_test(ro, rd)
    assert int(pairs[1]) == W


def test_order_is_the_block_permutation_of_the_live_packs(cuda):
    """count-aware: order[:count] is the block order of the first `count` packs; the slots past the count are not written"""
    from neuralsim_b200.graphics.neus_static import CNT_SLOTS, _block_order
    H, W = 37, 45                                        # H % 4 != 0, W % 8 != 0; the box test leaves ragged rows
    ro, rd = _rays(H, W)
    flag, pairs = _ray_test(ro, rd)
    assert int(pairs[1]) == W
    pix = torch.nonzero(flag).view(-1)
    n = pix.shape[0]
    assert 0 < n < H * W
    cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
    cnt[CNT_SLOTS["pairs"]], cnt[CNT_SLOTS["row_len"]] = pairs[0], pairs[1]
    live = n - 77
    cnt[CNT_SLOTS["hit"]] = live
    order = _block_order(pix, None, H * W, cnt, CNT_SLOTS["hit"])
    got = order[:live].cpu().numpy()
    np.testing.assert_array_equal(got, _expected_order(pix[:live].cpu().numpy(), W))
    assert sorted(got.tolist()) == list(range(live))
    # the fine-stage form: pack p lies on pixel pix[via[p]]
    via = torch.arange(0, n, 3, device="cuda")
    cnt[CNT_SLOTS["hit"]] = via.shape[0] - 5
    order_v = torch.full((via.shape[0],), -7, dtype=torch.int64, device="cuda")
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.neus_static import _call, _slot
    _call(L.lib().nsb_ray_block_order, "ray_block_order", cnt, CNT_SLOTS["hit"], None, L.ptr(pix, "i64"), L.ptr(via, "i64"), L.c_i64(via.shape[0]),
          L.c_i64(H * W), _slot(cnt, CNT_SLOTS["pairs"]), _slot(cnt, CNT_SLOTS["row_len"]), L.ptr(order_v), L.stream_ptr())
    live_v = via.shape[0] - 5
    np.testing.assert_array_equal(order_v[:live_v].cpu().numpy(), _expected_order(pix[via[:live_v]].cpu().numpy(), W))
    assert (order_v[live_v:] == -7).all()


@pytest.mark.parametrize("case", ["random_pixels", "single_row"])
def test_order_is_the_identity_without_row_structure(cuda, case):
    from neuralsim_b200.graphics import neus_fused
    if case == "random_pixels":
        ro, rd = _rays(40, 50)
        p = torch.randperm(ro.shape[0], generator=torch.Generator().manual_seed(3)).cuda()
        ro, rd = ro[p].contiguous(), rd[p].contiguous()
    else:
        ro, rd = _rays(1, 300, radius=1.5)
    flag, pairs = _ray_test(ro, rd)
    if case == "single_row":
        assert int(pairs[1]) == -1
    pix = torch.nonzero(flag).view(-1)
    order = neus_fused.block_order(pix, None, (ro.shape[0], pairs))
    assert torch.equal(order, torch.arange(pix.shape[0], device="cuda"))


def test_block_order_sdf_is_bit_equal(cuda):
    """mode 2 with the block order == mode 2 in strip order == mode 1 (ray-major), sdf and the in-kernel occupancy collection"""
    from neuralsim_b200.fields import LoTDNeuSModel
    from neuralsim_b200.fields.space import AABBSpace
    from neuralsim_b200.graphics import neus_fused
    from util import random_packs
    P, model0 = make_pair(cuda)
    model = LoTDNeuSModel(surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=P.lotd_cfg)), radiance_cfg=dict(n_appear_embedding=P.n_appear),
                          accel_cfg=dict(resolution=[64, 64, 64], update_from_samples_cfg=dict()), device=cuda)
    model.load_state_dict(model0.state_dict(), strict=False)
    model.train()
    H, W = 37, 45
    ro, rd = _rays(H, W)
    rt = AABBSpace(2.0, device="cuda").ray_test(ro, rd, near=0.01)
    assert rt["rays_coherent"] and int(rt["rays_row"][1][1]) == W and rt["num_rays"] < H * W
    order = neus_fused.block_order(rt["rays_inds"], None, rt["rays_row"])
    assert not torch.equal(order, torch.arange(order.shape[0], device="cuda"))
    n = rt["num_rays"]
    pi = random_packs(np.random.default_rng(5), n, 0, 70, "cuda")           # ragged packs, some empty
    S = int(pi[-1].sum())
    t = (rt["near"].repeat_interleave(pi[:, 1]) + 2.0 * torch.rand(S, generator=torch.Generator().manual_seed(5)).cuda()).contiguous()
    ridx = torch.repeat_interleave(torch.arange(n, device="cuda"), pi[:, 1])
    o, d = rt["rays_o"].contiguous(), rt["rays_d"].contiguous()
    occ = model.accel.occ
    assert occ.collect_struct() is not None
    out = []
    for packs in ((pi, None, order), (pi, None), None):
        occ._occ_val_grid_pcl.zero_()
        with torch.no_grad():
            sdf = model.forward_sdf_on_rays(ridx, t, o, d, packs=packs)["sdf"]
        out.append((sdf, occ._occ_val_grid_pcl.clone()))
    assert float(out[0][1].max()) > 0
    for sdf, grid in out[1:]:
        assert torch.equal(out[0][0], sdf)
        assert torch.equal(out[0][1], grid)


def test_graph_step_renders_the_same_with_and_without_the_order(cuda, monkeypatch):
    from neuralsim_b200.graphics import neus_static
    _, model = make_pair(cuda)
    model.train()
    H, W = 90, 101                                       # >= 8192 rays: the fine stages run as ray-tiled queries too
    ro, rd = _rays(H, W)
    ha = torch.zeros(ro.shape[0], 4, device=cuda)
    images = []
    for use_order in (True, False):
        if not use_order:
            monkeypatch.setattr(neus_static, "_block_order", lambda *a, **k: None)
        frame = neus_static.StaticFrame(model, ro.shape[0], near=0.01, slack=2.0)
        frame.step(ro, rd, ha)
        frame.step(ro, rd, ha)                          # a replay
        assert frame.captures == 1 and frame.coherent
        c = frame.counts()
        assert c["overflow"] == 0 and (c["row_len"] == W if use_order else True)
        images.append({k: frame.rendered[k].clone() for k in KEYS})
    for k in KEYS:
        assert torch.equal(images[0][k], images[1][k]), k
