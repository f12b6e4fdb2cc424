"""The perturbed one-launch step's bookkeeping of torch's random stream, on the host: the offset increment of a draw against a restatement
of torch's launch policy, the element -> Philox call mapping, the step's reservation, and the refusals (torch_rng.py, graphics/perturb.py)."""
import random
import types

import pytest
import torch

import torch_uniform as TU
from neuralsim_b200 import torch_rng as TR
from neuralsim_b200.graphics import perturb as PT
from neuralsim_b200.graphics.neus import query_config

# (SMs, max threads per SM): an H100 SXM (132 SMs, cap 1056), an H100 PCIe (114), and small caps that reach the loop's later iterations
DEVICES = [(132, 2048), (114, 2048), (7, 1536), (1, 1024)]


@pytest.mark.parametrize("sms,threads", DEVICES)
def test_inc_matches_torchs_policy(sms, threads):
    cap = sms * (threads // 256)
    edges = [256 * cap, 4 * 256 * cap, 8 * 256 * cap]
    ns = list(range(1, 3000)) + [e + d for e in edges for d in (-257, -256, -255, -1, 0, 1, 255, 256, 257)] + [12 * 256 * cap + 3]
    for n in ns:
        assert TR.uniform_inc(n, cap) == TU.calc_execution_policy(n, sms, threads)[0], n
    assert TR.uniform_inc(0, cap) == 0                          # an empty draw is not launched and does not advance the offset


@pytest.mark.parametrize("sms,threads", [(1, 1024), (2, 512)])
def test_element_mapping_matches_the_grid_stride_loop(sms, threads):
    cap = sms * (threads // 256)
    for n in [1, 5, 255, 256, 257, 256 * cap - 1, 256 * cap, 256 * cap + 1, 4 * 256 * cap, 4 * 256 * cap + 1, 9 * 256 * cap + 77]:
        calls = TU.element_calls(n, sms, threads)
        assert sorted(calls) == list(range(n))
        inc = TR.uniform_inc(n, cap)
        for li, (idx, k, c) in calls.items():
            assert TU.element_call(li, n, cap) == (idx, k, c)
            assert 4 * k < inc                                  # every call lies inside the offsets the draw reserves


def test_inc_is_monotone():
    for cap in (4, 912, 1056):
        prev = 0
        for n in sorted(set(range(0, 20000, 7)) | set(range(256 * cap - 600, 256 * cap * 9, 911))):
            v = TR.uniform_inc(n, cap)
            assert v >= prev, (cap, n)
            prev = v


def test_reservation_bounds_every_step():
    cfg = query_config(num_coarse=128, num_fine=[8, 8, 32], upsample_inv_s_factors=(1, 4, 16), march_cfg=dict(max_steps=256))
    rng = random.Random(3)
    for cap in (4, 912, 1056):
        for n_rays in (1, 255, 4096, 8192, 65536):
            res = PT.reservation(n_rays, cfg, cap)
            for _ in range(200):
                n = rng.randint(0, n_rays)
                m = rng.randint(0, n * cfg.max_steps)
                hit = rng.randint(0, n)
                used = TR.uniform_inc(n * 129, cap) + TR.uniform_inc(m, cap) + sum(TR.uniform_inc(hit * nf, cap) for nf in cfg.num_fine)
                assert used <= res
            full = TR.uniform_inc(n_rays * 129, cap) + TR.uniform_inc(n_rays * cfg.max_steps, cap) + sum(TR.uniform_inc(n_rays * nf, cap) for nf in cfg.num_fine)
            assert res == full and res % 4 == 0


def test_step_draw_lists():
    slots = dict(n_rays=0, marched=12, hit=13)
    coarse, stages = PT.step_draws(slots, 129, (9, 9, 33))
    assert coarse == [(0, 129)]
    assert stages == [[(0, 129), (12, 1), (13, 9)], [(0, 129), (12, 1), (13, 9), (13, 9)], [(0, 129), (12, 1), (13, 9), (13, 9), (13, 33)]]


def test_refusals():
    cfg = query_config(num_coarse=128, march_cfg=dict(max_steps=512))
    with pytest.raises(RuntimeError, match="2\\^31"):
        PT.reservation(2 ** 31 // 512, cfg, 1056)                # the marcher's bound n_rays * max_steps reaches 2^31
    with pytest.raises(RuntimeError, match="2\\^31"):
        PT.reservation(2 ** 31 // 129 + 1, query_config(num_coarse=128, march_cfg=dict(max_steps=1)), 1056)
    PT.reservation(2 ** 31 // 512 - 1, cfg, 1056)
    with pytest.raises(RuntimeError, match="CUDA torch.Generator"):
        TR.cuda_generator(torch.Generator(), "cuda:0")
    with pytest.raises(RuntimeError, match="CUDA torch.Generator"):
        TR.cuda_generator(object(), "cuda:0")
    assert TR.seed_i64(2 ** 64 - 1) == -1 and TR.seed_i64(5) == 5


def test_static_frame_argument_checks():
    from neuralsim_b200.graphics.neus_static import StaticFrame
    model = types.SimpleNamespace(device=torch.device("cpu"), use_h_appear=False)
    with pytest.raises(RuntimeError, match="only with perturb=True"):
        StaticFrame(model, 16, h_appear_dim=0, generator=torch.Generator())
    with pytest.raises(RuntimeError, match="CUDA torch.Generator"):
        StaticFrame(model, 16, h_appear_dim=0, perturb=True, generator=torch.Generator())
