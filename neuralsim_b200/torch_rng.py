"""torch's CUDA generator contract, the Python half of csrc/torch_uniform.cuh: what the kernels need to draw on the device what
torch.rand / torch.randint give from the same generator state.  torch advances a CUDA generator's offset by `uniform_inc(N)` per draw of
N values, so draw k of a sequence starts at base + sum_{j<k} uniform_inc(N_j).  A graph-captured consumer (the perturbed step, the
in-graph samplers, the occupancy update) bounds its draws by a reservation: before each replay `take` writes the generator's (seed,
offset) into a device block and advances the generator by the reservation -- host-side calls, no synchronisation -- and the kernels find
their offsets on the device.  From the same state a replay draws what the host-sized path draws; the host-sized path then advances the
generator by what it drew, a replay by the reservation, so runs of the two drift apart after the first step."""
from __future__ import annotations

import torch

__all__ = ["MAX_DRAW", "grid_cap", "uniform_inc", "check_draw", "cuda_generator", "seed_i64", "take"]

MAX_DRAW = 2 ** 31          # torch splits a draw of 2^31 or more values into 32-bit sub-iterators, each with its own offset


def grid_cap(device) -> int:
    """torch's cap on the grid of a draw on `device` (calc_execution_policy): SMs * (maxThreadsPerSM / 256) blocks"""
    p = torch.cuda.get_device_properties(device)
    return int(p.multi_processor_count) * (int(p.max_threads_per_multi_processor) // 256)


def uniform_inc(n: int, cap: int) -> int:
    """the generator offset a draw of n float32 values advances by (0 for an empty draw)"""
    n = int(n)
    if n <= 0:
        return 0
    stride = 256 * min((n + 255) // 256, int(cap))
    return ((n - 1) // (4 * stride) + 1) * 4


def check_draw(n, what):
    """refuse a draw bound of 2^31 or more values (`what` names the draw in the message)"""
    if n >= MAX_DRAW:
        raise RuntimeError(f"{what} draw may hold {n} >= 2^31 values, which torch splits into 32-bit sub-draws")


def cuda_generator(generator, device):
    """the CUDA generator a draw on `device` takes its state from: `generator`, or torch's default one of `device`"""
    if generator is not None and (not isinstance(generator, torch.Generator) or generator.device.type != "cuda"):
        raise RuntimeError(f"the generator must be a CUDA torch.Generator, got {getattr(generator, 'device', type(generator))}")
    device = torch.device(device)
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if generator is None:
        return torch.cuda.default_generators[idx]
    if (generator.device.index if generator.device.index is not None else torch.cuda.current_device()) != idx:
        raise RuntimeError(f"the generator is on {generator.device}, the draw on cuda:{idx}")
    return generator


def seed_i64(seed: int) -> int:
    """a uint64 Philox seed as the int64 of the same bits"""
    seed = int(seed)
    return seed - 2 ** 64 if seed >= 2 ** 63 else seed


def take(gen, reserve: int, out=None):
    """(seed, offset) of `gen` into the device block `out` (int64 [2]; made when None) by two fills -- no host read, no synchronisation --
    then the generator advanced by `reserve`.  -> out"""
    seed, off = seed_i64(gen.initial_seed()), int(gen.get_offset())
    if out is None:
        out = torch.empty(2, dtype=torch.int64, device=gen.device)
    out[0].fill_(seed)
    out[1].fill_(off)
    gen.set_offset(off + int(reserve))
    return out
