"""Perturbed samples of the one-launch step from torch's own CUDA random stream (csrc/perturb.cu, csrc/torch_uniform.cuh).

A perturbed NeuS query draws, in order, torch.rand([n_rays, nc1]) (coarse depths), rand_like of the M marched samples (the marcher's
jitter, discarded) and torch.rand([n_hit, nf_i]) per up-sampling stage (graphics/neus.py:_query_fused).  Draw k starts at base +
sum_{j<k} uniform_inc(N_j) (torch_rng.py); every N_j is a count of the step's device block (graphics/neus_static.py CNT_SLOTS), so the
kernels find their offsets on the device.  A step takes its (seed, base offset) from a device block `rng` = int64 [2] and reserves
`reservation(...)` offsets of the generator: a bound on every draw the step can make."""
from __future__ import annotations

import ctypes

from .. import _lib as L
from .. import torch_rng as TR
from ..torch_rng import cuda_generator, grid_cap, seed_i64, take, uniform_inc  # noqa: F401 -- public here before torch_rng.py held them

__all__ = ["grid_cap", "uniform_inc", "reservation", "cuda_generator", "take", "step_draws", "coarse_depths", "invert_cdf"]

MAX_DRAWS = 8               # entries of a draw list (csrc/perturb.cu kMaxDraws)


def reservation(n_rays: int, cfg, cap: int) -> int:
    """offsets a step of n_rays rays reserves: the coarse draw, the marcher's at n_rays * max_steps samples (M can not exceed it) and every
    stage's at n_rays hit rays -- each inc is monotone in N, so this bounds the step's sum whatever its counts.  Refuses a draw of 2^31 or more."""
    nc1 = cfg.num_coarse + 1
    sizes = [(n_rays * nc1, "coarse"), (n_rays * cfg.max_steps, "marcher")] + [(n_rays * nf, f"stage {i}") for i, nf in enumerate(cfg.num_fine)]
    for n, what in sizes:
        TR.check_draw(n, f"perturb=True: the {what}")
    if 2 + len(cfg.num_fine) > MAX_DRAWS:
        raise RuntimeError(f"perturb=True: at most {MAX_DRAWS - 2} up-sampling stages, got {len(cfg.num_fine)}")
    return sum(TR.uniform_inc(n, cap) for n, _ in sizes)


def step_draws(slots, nc1, num_fine):
    """the draw lists of one step, (count slot, multiplier) pairs in draw order: -> (coarse list, [stage i list])"""
    coarse = [(slots["n_rays"], nc1)]
    before = coarse + [(slots["marched"], 1)]
    stages = []
    for nf in num_fine:
        before = before + [(slots["hit"], nf)]
        stages.append(list(before))
    return coarse, stages


def _draws(draws):
    flat = [int(v) for pair in draws for v in pair]
    return (ctypes.c_int32 * len(flat))(*flat), L.c_i32(len(draws))


def coarse_depths(near, far, nc1, rng, cnt, draws, t, next_offset=None):
    """t [R, nc1] (R the capacity) := the perturbed coarse depths of rows below the count of the last draw (nsb_coarse_depths_perturbed)"""
    P = L.ptr
    d, nd = _draws(draws)
    L.check(L.lib().nsb_coarse_depths_perturbed(P(near, "f32", "near"), P(far, "f32", "far"), L.c_i64(t.shape[0]), L.c_i32(nc1), P(rng, "i64", "rng"),
                                                P(cnt, "i64", "cnt"), d, nd, P(t, "f32", "t"), P(next_offset, "i64", "next_offset", allow_none=True),
                                                L.stream_ptr()), "coarse_depths_perturbed")
    return t


def invert_cdf(bins, cdf, pack_infos, nf, rng, cnt, draws, samples, next_offset=None):
    """samples [P, nf] (P the capacity) := the perturbed inverse-cdf samples of the packs below the count of the last draw
    (nsb_packed_invert_cdf_perturbed)"""
    P = L.ptr
    d, nd = _draws(draws)
    L.check(L.lib().nsb_packed_invert_cdf_perturbed(P(bins, "f32", "bins"), P(cdf, "f32", "cdf"), P(pack_infos, "i64", "pack_infos"), L.c_i64(samples.shape[0]),
                                                    L.c_i32(nf), P(rng, "i64", "rng"), P(cnt, "i64", "cnt"), d, nd, P(samples, "f32", "samples"),
                                                    P(next_offset, "i64", "next_offset", allow_none=True), L.stream_ptr()), "packed_invert_cdf_perturbed")
    return samples
