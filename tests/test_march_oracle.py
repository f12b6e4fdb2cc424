"""CPU: the C oracle of the marcher (oracle/march.c) on the street-scale inputs of tests/march_cases.py against the float64 meaning
checks of tests/march64.py, and those checks against three deliberately wrong sample lists."""
import numpy as np
import pytest
import torch

import march64
import march_cases as mc
from oracle import march as omarch

CASES = ["small_blocks_gamma", "small_checker", "small_full_cap", "small_corner", "roi_face_full", "large_blocks"]


@pytest.fixture(scope="module")
def rays():
    return mc.street_rays(n_azim=120, cam_hw=(24, 32), n_axis=32, n_boundary=48)


def _case(name):
    _, kind, res, roi, gamma, dt_max, max_steps = next(c for c in mc.SINGLE if c[0] == name)
    return mc.grid(kind, res), torch.tensor(roi), gamma, dt_max, max_steps


@pytest.mark.parametrize("name", CASES)
def test_oracle_samples_mean_what_they_should(rays, name):
    grid, roi, gamma, dt_max, max_steps = _case(name)
    out = omarch.ray_marching(*rays, roi, grid, mc.STEP, dt_max, gamma, max_steps)
    assert march64.check(*rays, roi, grid, mc.STEP, dt_max, gamma, max_steps, *out)["samples"] > 0


def test_oracle_batched_samples_mean_what_they_should(rays):
    grid, rois = mc.batched_grid(mc.SMALL)
    bi = torch.from_numpy(np.random.default_rng(1).integers(-1, grid.shape[0], rays[0].shape[0])).int()
    out = omarch.ray_marching(*rays, rois, grid, mc.STEP, 1.0, 0.01, mc.MAX_STEPS, batch_inds=bi)
    assert int(out[0][bi < 0, 1].abs().sum()) == 0                        # rays with a negative batch index march nothing
    st = march64.check(*rays, rois, grid, mc.STEP, 1.0, 0.01, mc.MAX_STEPS, *out[:5], batch_inds=bi, bidx=out[5])
    assert st["samples"] > 0 and int(out[5].max()) == grid.shape[0] - 1


def _drop(out, k):
    """the sample list without sample k"""
    info, t0, t1, ridx, gidx = out[:5]
    keep = torch.ones(t0.shape[0], dtype=torch.bool)
    keep[k] = False
    cnt = info[:, 1].clone()
    cnt[int(ridx[k])] -= 1
    info = torch.stack([cnt.cumsum(0, dtype=torch.int32) - cnt, cnt], -1)
    return [info, t0[keep], t1[keep], ridx[keep], gidx[keep]] + [x[keep] for x in out[5:]]


def test_wrong_samples_fail(rays):
    grid, roi, gamma, dt_max, max_steps = _case("small_blocks_gamma")
    args = (roi, grid, mc.STEP, dt_max, gamma, max_steps)
    out = omarch.ray_marching(*rays, *args)
    march64.check(*rays, *args, *out)
    info, t0, t1, ridx, gidx = out
    # a sample in the middle of an occupied run of five: its neighbours start where the previous one ended, in the same voxel
    run = (t0[1:-1] == t1[:-2]) & (t0[2:] == t1[1:-1]) & (gidx[1:-1] == gidx[:-2]) & (gidx[2:] == gidx[1:-1]) & (ridx[2:] == ridx[:-2])
    k = int(torch.nonzero(run[1:-1] & run[:-2] & run[2:])[0, 0]) + 2
    with pytest.raises(AssertionError, match="skip over a step in an occupied voxel"):
        march64.check(*rays, *args, *_drop(out, k))
    # gidx of that sample moved by one cell (z + 1)
    moved = gidx.clone()
    moved[k] += 1
    with pytest.raises(AssertionError, match="not in the voxel gidx names|names an empty voxel"):
        march64.check(*rays, *args, info, t0, t1, ridx, moved)
    # the batched voxel index without the batch offset (the per-grid index)
    bgrid, rois = mc.batched_grid(mc.SMALL)
    bi = torch.from_numpy(np.random.default_rng(2).integers(0, bgrid.shape[0], rays[0].shape[0])).int()
    bout = omarch.ray_marching(*rays, rois, bgrid, mc.STEP, 1e10, 0.0, mc.MAX_STEPS, batch_inds=bi)
    bargs = (rois, bgrid, mc.STEP, 1e10, 0.0, mc.MAX_STEPS)
    march64.check(*rays, *bargs, *bout[:5], batch_inds=bi, bidx=bout[5])
    local = bout[4] - bout[5] * bgrid[0].numel()
    assert bool((local != bout[4]).any())
    with pytest.raises(AssertionError, match="flat over"):
        march64.check(*rays, *bargs, *bout[:4], local, batch_inds=bi, bidx=bout[5])


def test_batch_data_size_must_divide_the_rays():
    """_occ_grid.batched_ray_marching refuses a batch_data_size that does not divide n_rays (batched_marching.cu:206)"""
    from neuralsim_b200.bindings import _occ_grid
    o = torch.zeros(10, 3)
    t = torch.zeros(10)
    with pytest.raises(RuntimeError, match="divisor"):
        _occ_grid.batched_ray_marching(o, o, t, t, None, 4, torch.zeros(2, 6), torch.zeros(2, 4, 4, 4, dtype=torch.bool),
                                       _occ_grid.ContractionType.AABB, 0.1, 1e10, 0.0, 16, True)
