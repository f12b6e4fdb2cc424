"""oracle/lidar64.py (the float64 restatement the GPU tests of csrc/lidar_loss.cu compare against) pinned on the CPU to a direct torch float64
evaluation of the reference's formulas (app/loss/lidar.py LidarLoss.forward, DepthLoss, LineOfSightLoss.fn_for_neus_unisim; recon.py l1_loss /
relative_l2_loss with loss/utils.py reduce), gradients by autograd; and the milestones annealer's bisect at its boundaries.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import lidar64

from neuralsim_b200.loss.lidar import LidarLoss, anneal_milestones


def _torch_reference(pred, mask_pred, gt, t, vw, pinfo, rih, *, fn_type, w_depth, w_los, eps, thresh=1e-7, discard_toofar=None, factor=100.0):
    """the reference's LidarLoss.forward, written out in torch float64 (sort, repeat_interleave and all)"""
    pred = torch.tensor(pred, dtype=torch.float64, requires_grad=True)
    vw = torch.tensor(vw, dtype=torch.float64, requires_grad=True)
    gt, mask_pred, t = (torch.tensor(a, dtype=torch.float64) for a in (gt, mask_pred, t))
    pinfo, rih = torch.tensor(pinfo, dtype=torch.int64).view(-1, 2), torch.tensor(rih, dtype=torch.int64)
    mask = (mask_pred.data > thresh) & (gt > 0)
    if discard_toofar is not None and discard_toofar > 0:
        mask = gt <= discard_toofar
    if factor > 0:
        err = (pred - gt).abs() * mask
        sv, _ = torch.sort(err.data)
        mask[err > sv[pred.numel() // 2] * factor] = False
    if fn_type == "l1":
        f = (pred - gt).abs()
    else:
        f = (pred - gt) ** 2 / (pred ** 2 + 1e-2)
    out = {"depth": w_depth * (f * mask).mean()}
    if pinfo.shape[0]:
        gt_ex = torch.repeat_interleave(gt[rih], pinfo[:, 1], dim=0)
        empty = (t - gt_ex).abs() > eps
        per = torch.zeros(pinfo.shape[0], dtype=torch.float64).index_add(0, torch.repeat_interleave(torch.arange(pinfo.shape[0]), pinfo[:, 1]),
                                                                            empty * vw ** 2)
        out["los"] = w_los * (per * mask[rih]).mean()
    grads = torch.autograd.grad(sum(out.values()), [pred, vw], allow_unused=True)
    return {k: float(v.detach()) for k, v in out.items()}, mask.numpy(), [None if g is None else g.numpy() for g in grads]


def _case(rng, R=64, n_per=None, hit_frac=0.7):
    """R rays, a random subset kept with n_per samples each (0-sample packs when n_per says so); t around gt so both sides of eps occur"""
    gt = rng.uniform(1, 100, R)
    pred = gt + rng.normal(0, 2, R)
    mask_pred = rng.uniform(0, 1, R)
    rih = np.sort(rng.choice(R, int(R * hit_frac), replace=False))
    n = rng.integers(0, 40, rih.shape[0]) if n_per is None else np.full(rih.shape[0], n_per)
    first = np.concatenate([[0], np.cumsum(n)[:-1]])
    pinfo = np.stack([first, n], -1)
    t = np.concatenate([gt[r] + rng.normal(0, 3, k) for r, k in zip(rih, n)]) if n.sum() else np.zeros(0)
    vw = rng.uniform(0, 0.3, int(n.sum()))
    return pred, mask_pred, gt, t, vw, pinfo, rih


def _check(args, **kw):
    pred, mask_pred, gt, t, vw, pinfo, rih = args
    ref, mask, (g_pred, g_vw) = _torch_reference(pred, mask_pred, gt, t, vw, pinfo, rih, **kw)
    o = lidar64.lidar_loss(pred, mask_pred, gt, t, vw, pinfo, rih, fn_type=kw["fn_type"], w_depth=kw["w_depth"], w_los=kw["w_los"], epsilon=kw["eps"],
                           discard_toofar=kw.get("discard_toofar"), median_factor=kw.get("factor", 100.0), decide=np.float64)
    np.testing.assert_array_equal(o["mask"], mask)
    np.testing.assert_allclose(o["depth"], ref["depth"], rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(o["g_depth"], g_pred, rtol=1e-12, atol=1e-300)
    if "los" in ref:
        np.testing.assert_allclose(o["los"], ref["los"], rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(o["g_vw"], g_vw, rtol=1e-12, atol=1e-300)
    return o, ref


@pytest.mark.parametrize("fn_type", ["l1", "l2_relative"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_reference_formulas(fn_type, seed):
    rng = np.random.default_rng(seed)
    args = _case(rng, R=200)
    assert (args[5][:, 1] == 0).any()                      # rays with 0 samples
    o, _ = _check(args, fn_type=fn_type, w_depth=0.3, w_los=0.05, eps=1.5, discard_toofar=80.0)
    assert o["los"] > 0 and o["depth"] > 0


def test_discard_toofar_overrides_the_mask():
    """mask_pred below the threshold and gt <= 0 would mask a ray out; discard_toofar ASSIGNS the mask, so they are kept"""
    rng = np.random.default_rng(3)
    pred, mask_pred, gt, t, vw, pinfo, rih = _case(rng)
    gt[:10] = np.minimum(gt[:10], 70.0)
    mask_pred[:10] = 0.0
    gt[10:12] = -1.0
    o, _ = _check((pred, mask_pred, gt, t, vw, pinfo, rih), fn_type="l1", w_depth=1.0, w_los=1.0, eps=1.0, discard_toofar=80.0, factor=0.0)
    assert o["mask"][:12].all()
    assert not lidar64.lidar_mask(pred, mask_pred, gt, discard_toofar=None, median_factor=0.0, decide=np.float64)[0][:12].any()


def test_eps_boundary_is_strict():
    """|t - gt| == eps exactly is not selected (strict >), in float64 and in fp32"""
    gt = np.array([10.0, 20.0])
    t = np.array([10.5, 9.5, 10.25, 20.5, 21.0])
    vw = np.array([0.1, 0.2, 0.3, 0.4, 0.5])
    pinfo, rih = np.array([[0, 3], [3, 2]]), np.array([0, 1])
    for decide in (np.float32, np.float64):
        val, g, rows = lidar64.los_term(t, vw, pinfo, rih, gt, np.array([True, True]), 0.5, 1.0, decide=decide)
        assert rows[0] == 0.0 and rows[1] == pytest.approx(0.25) and g[:4].tolist() == [0.0, 0.0, 0.0, 0.0]
    _check((np.array([11.0, 19.0]), np.ones(2), gt, t, vw, pinfo, rih), fn_type="l1", w_depth=1.0, w_los=2.0, eps=0.5, factor=0.0)


def test_all_rays_masked():
    rng = np.random.default_rng(4)
    pred, mask_pred, gt, t, vw, pinfo, rih = _case(rng)
    mask_pred[:] = 0.0
    o, ref = _check((pred, mask_pred, gt, t, vw, pinfo, rih), fn_type="l2_relative", w_depth=1.0, w_los=1.0, eps=1.0)
    assert o["depth"] == 0.0 and o["los"] == 0.0 and not o["g_depth"].any() and not o["g_vw"].any()


def test_median_outliers_and_nan_order():
    err = np.array([3.0, np.nan, 0.0, np.inf, 1.0, 1.0, 2.0], np.float32)
    assert lidar64.kth_smallest(err, 3) == float(torch.sort(torch.from_numpy(err)).values[3]) == 2.0
    assert np.isnan(lidar64.kth_smallest(err, 6)) and lidar64.kth_smallest(err, 5) == np.inf
    gt = np.full(9, 10.0)
    pred = gt + np.array([0.1, 0.2, 0.1, 0.3, 0.2, 0.1, 50.0, 0.2, 0.1])      # one ray > 100 x the median error
    mask, _, med = lidar64.lidar_mask(pred, np.ones(9), gt, decide=np.float64)
    assert med == pytest.approx(0.2) and mask.tolist() == [True] * 6 + [False] + [True] * 2


@pytest.mark.parametrize("it,val", [(0, 1.5), (4999, 1.5), (5000, 0.75), (5001, 0.75), (9999, 0.75), (10000, 0.5), (10 ** 6, 0.5)])
def test_milestone_bisect_at_the_boundaries(it, val):
    """`milestones` mark interval ends: vals[bisect_right(milestones, it)] (the shipped epsilon schedule)"""
    assert anneal_milestones(it, [5000, 10000], [1.5, 0.75, 0.5]) == val
    los = LidarLoss(line_of_sight=dict(w=0.1, fn_type="neus_unisim", fn_param=dict(epsilon_anneal=dict(
        type="milestones", milestones=[5000, 10000], vals=[1.5, 0.75, 0.5])))).line_of_sight_loss
    assert los.epsilon(it) == val


@pytest.mark.parametrize("kw,name", [
    (dict(discard_outliers=0.1), "discard_outliers"),
    (dict(line_of_sight=dict(fn_type="nerf")), "nerf"),
    (dict(line_of_sight=dict(fn_type="neus_urban")), "neus_urban"),
    (dict(depth=dict(fn_type="l1_log")), "l1_log"),
    (dict(depth=dict(fn_type="l1", anneal=dict(type="linear", stop_it=10))), "linear"),
])
def test_unbuilt_options_raise_naming_them(kw, name):
    with pytest.raises(RuntimeError, match=name):
        LidarLoss(**kw)
