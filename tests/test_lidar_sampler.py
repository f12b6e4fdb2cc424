"""The LiDAR batch source of the one-launch step (neuralsim_b200/lidar_sampler.py) against the reference's own LidarDataset.sample_merged,
executed on the CPU (tests/golden/ref_lidar_sampler.npz, made by tests/golden/make_golden_lidar_sampler.py from seeded draws): the
package's torch restatement of the draw and the host split table bit for bit; the reservation; the refusals.  No GPU."""
import os

import numpy as np
import pytest
import torch

from neuralsim_b200 import lidar_sampler as LS
from neuralsim_b200.torch_rng import uniform_inc

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_lidar_sampler.npz"))
CASES = [k for k in range(3)]
CAP = 132 * 8                                 # torch's grid cap on an H100 SXM (132 SMs x 2048 / 256 threads)


def _eq(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a, b), f"{what}: not bit-equal"


def _sampler(k, num_rays=None, **kw):
    F, Ln, n, weighted = (int(v) for v in GOLD[f"case{k}.meta"])
    p = f"case{k}."
    o, d, r = (torch.from_numpy(GOLD[p + key].copy()) for key in ("rays_o", "rays_d", "ranges"))
    l2w = torch.zeros(F, Ln, 3, 4)
    mode = dict(multi_lidar_weight=GOLD[p + "weight"].tolist()) if weighted else dict(lidar_sample_mode="merged_equal")
    return LS.LidarSampler(o, d, r, GOLD[p + "counts"], l2w, num_rays or n, **{**mode, **kw})


@pytest.mark.parametrize("k", CASES)
def test_recipe_equals_reference(k):
    s = _sampler(k)
    for f in range(s.n_frames):
        q = f"case{k}.f{f}."
        g = torch.Generator().manual_seed(int(GOLD[q + "seed"]))
        out = s.recipe(f, generator=g)
        _eq(np.array(out["split"], np.int64), GOLD[q + "split"], q + "split")
        for key in ("inds", "li", "rays_o", "rays_d", "ranges"):
            _eq(out[key].numpy(), GOLD[q + key], q + key)
        _eq(np.full(s.num_rays, f, np.int64), GOLD[q + "rays_fidx"], q + "rays_fidx")


@pytest.mark.parametrize("k", CASES)
def test_host_split_table_equals_reference(k):
    s = _sampler(k)
    rows = s.rows(CAP)
    base = 0
    for f, row in enumerate(rows):
        split = GOLD[f"case{k}.f{f}.split"].tolist()
        counts = GOLD[f"case{k}.counts"][f].tolist()
        Ln = len(split)
        assert s.split[f] == split
        assert row[LS._N_LIDARS] == Ln and row[LS._DATA_OFF] == base and row[LS._POSE_BASE] == f * Ln
        assert row[LS._RAY_START:LS._RAY_START + Ln + 1] == [0, *np.cumsum(split).tolist()]
        assert row[LS._CUMU:LS._CUMU + Ln + 1] == [0, *np.cumsum(counts).tolist()]
        offs = [sum(uniform_inc(n, CAP) for n in split[:li]) for li in range(Ln)]
        assert row[LS._DRAW_OFF:LS._DRAW_OFF + Ln] == offs and row[LS._INC] == sum(uniform_inc(n, CAP) for n in split)
        base += sum(counts)
    assert len(rows[0]) == LS.TABLE_WIDTH


def test_golden_covers_the_split_edges():
    """an empty lidar, a truncation remainder on lidar 0 and on a later lidar, a lone lidar, and both modes"""
    splits = {(k, f): GOLD[f"case{k}.f{f}.split"] for k in CASES for f in range(int(GOLD[f"case{k}.meta"][0]))}
    counts = {(k, f): GOLD[f"case{k}.counts"][f] for k, f in splits}
    assert any((counts[kf] == 0).any() for kf in splits)
    w0 = GOLD["case0.weight"] / GOLD["case0.weight"].sum()
    assert splits[(0, 1)][0] > int(2048 * w0[0] / (1 - w0[2]))                  # lidar 2 empty: the remainder lands on lidar 0
    assert splits[(0, 2)][0] == 0 and splits[(0, 2)].sum() == 2048              # lidar 0 empty: the remainder on lidar 1
    assert (splits[(0, 3)] > 0).sum() == 1
    assert {int(GOLD[f"case{k}.meta"][3]) for k in CASES} == {0, 1}


@pytest.mark.parametrize("k", CASES)
def test_reservation_bounds_every_frame(k):
    s = _sampler(k)
    res = s.inc(s.num_rays, CAP)
    incs = [s.frame_inc(f, CAP) for f in range(s.n_frames)]
    assert res == max(incs) and all(sum(uniform_inc(n, CAP) for n in s.split[f]) <= res for f in range(s.n_frames))
    rows = s.rows(CAP)
    assert [r[LS._INC] for r in rows] == incs
    with pytest.raises(RuntimeError, match="num_rays"):
        s.inc(s.num_rays + 1, CAP)


def test_refusals():
    o, d, r = torch.zeros(10, 3), torch.zeros(10, 3), torch.zeros(10)
    l2w = torch.zeros(2, 2, 3, 4)
    ok = dict(multi_lidar_weight=[1.0, 1.0])
    LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64, **ok)
    with pytest.raises(RuntimeError, match="frame 1 has no beams"):
        LS.LidarSampler(o, d, r, [[6, 4], [0, 0]], l2w, 64, **ok)
    with pytest.raises(RuntimeError, match="NSB_LIDAR_MAX"):
        LS.LidarSampler(torch.zeros(9, 3), torch.zeros(9, 3), torch.zeros(9), [[1] * 9], torch.zeros(1, 9, 3, 4), 64,
                        lidar_sample_mode="merged_equal")
    with pytest.raises(RuntimeError, match="2\\^32"):
        LS.LidarSampler(o, d, r, np.array([[2 ** 32, 1], [1, 1]]), l2w, 64, **ok)
    for mode in ("merged_random", "merged_uniform", "single_uniform", "single_weighted"):
        with pytest.raises(RuntimeError, match=f"lidar_sample_mode='{mode}'"):
            LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64, lidar_sample_mode=mode, **ok)
    with pytest.raises(RuntimeError, match="point_batch"):
        LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64, equal_mode="point_batch", **ok)
    with pytest.raises(RuntimeError, match="needs multi_lidar_weight"):
        LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64)
    with pytest.raises(RuntimeError, match="no rays to its lidars"):
        LS.LidarSampler(o, d, r, [[3, 2], [0, 5]], l2w, 64, multi_lidar_weight=[1.0, 0.0])
    with pytest.raises(RuntimeError, match="l2w"):
        LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], torch.zeros(2, 3, 3, 4), 64, **ok)
    with pytest.raises(RuntimeError, match="rays_o"):
        LS.LidarSampler(o[:9], d, r, [[3, 2], [4, 1]], l2w, 64, **ok)
    s = LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64, **ok)
    for bad in (2, -1, True, 0.5):
        with pytest.raises(RuntimeError, match="frame_ind"):
            s.check_frame(bad)
    LS.LidarSampler(o, d, r, [[3, 2], [4, 1]], l2w, 64, lidar_sample_mode="merged_equal")       # equal weights: none needed


def test_lidar_loss_reads_ranges_from_the_ground_truth_with_it_none():
    """LidarLoss(None, ret, ground_truth=gt) with it=None reads gt's ranges in place and the weights of the last set_step(None, it)"""
    from neuralsim_b200.loss import LidarLoss
    lidar = LidarLoss(depth=dict(w=0.05, fn_type="l1", anneal=dict(type="milestones", milestones=[10], vals=[1.0, 2.0])))
    lidar.set_step(None, 20, device="cpu")
    assert lidar._blk.tolist()[0] == 2.0 and lidar.ranges is None
