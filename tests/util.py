"""Shared helpers of the parity tests: identical weights in the oracle container and the product model."""
import numpy as np
import torch

from oracle import scene as oscene


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def small_lotd_cfg():
    """4 dense + 4 hashed levels with a 2^14 table: same code paths as CFG, seconds on the CPU oracle."""
    return dict(lod_res=[8, 12, 18, 24, 40, 64, 100, 160], lod_n_feats=[2] * 8, lod_types=["Dense"] * 4 + ["Hash"] * 4,
                hashmap_size=2 ** 14)


def make_pair(device, seed=42, ln_inv_s_init=0.5298, noise=2.0e-3, full=True):
    """(oracle params P, product model) with identical fp32 masters.  full=True -> CFG-sized LoTD (16 x 2, T=2^19)."""
    from neuralsim_b200.fields import LoTDNeuSModel
    P = oscene.make_sphere_params(seed=seed, ln_inv_s_init=ln_inv_s_init, noise=noise)
    model = LoTDNeuSModel(
        surface_cfg=dict(bounding_size=2.0, encoding_cfg=dict(lotd_cfg=P.lotd_cfg)),
        radiance_cfg=dict(n_appear_embedding=P.n_appear), var_ctrl_cfg=dict(ln_inv_s_init=ln_inv_s_init),
        accel_cfg=dict(resolution=[64, 64, 64], update_from_samples_cfg=None), device=device,
        ray_query_cfg=dict(query_mode="march_occ_multi_upsample_compressed", query_param=dict(
            nablas_has_grad=True, num_coarse=64, num_fine=[8, 8, 32], coarse_step_cfg=dict(step_mode="linear"),
            march_cfg=dict(step_size=0.005, max_steps=4096), upsample_inv_s=64.0, upsample_inv_s_factors=[1, 4, 16],
            upsample_use_estimate_alpha=True)))
    load_params(model, P)
    model.accel.occ.set_occ_grid(oscene.make_occ_grid().to(device))
    return P, model


def load_params(model, P):
    with torch.no_grad():
        dev = model.device
        model.implicit_surface.encoding.flattened_params.copy_(P.grid.to(dev))
        d = model.implicit_surface.decoder.layers
        d[0].weight.copy_(P.dec_W1.to(dev)); d[0].bias.copy_(P.dec_b1.to(dev))
        d[1].weight.copy_(P.dec_W2.to(dev)); d[1].bias.copy_(P.dec_b2.to(dev))
        r = model.radiance_net.blocks.layers
        r[0].weight.copy_(P.rad_W1.to(dev)); r[0].bias.copy_(P.rad_b1.to(dev))
        r[1].weight.copy_(P.rad_W2.to(dev)); r[1].bias.copy_(P.rad_b2.to(dev))
        r[2].weight.copy_(P.rad_W3.to(dev)); r[2].bias.copy_(P.rad_b3.to(dev))
        model.ctrl_var.ln_inv_s.copy_(P.ln_inv_s.to(dev))


def product_grads(model):
    d, r = model.implicit_surface.decoder.layers, model.radiance_net.blocks.layers
    g = lambda p: None if p.grad is None else p.grad.detach().float().cpu()
    return dict(grid=g(model.implicit_surface.encoding.flattened_params), dec_W1=g(d[0].weight), dec_b1=g(d[0].bias),
                dec_W2=g(d[1].weight), dec_b2=g(d[1].bias), rad_W1=g(r[0].weight), rad_b1=g(r[0].bias), rad_W2=g(r[1].weight),
                rad_b2=g(r[1].bias), rad_W3=g(r[2].weight), rad_b3=g(r[2].bias), ln_inv_s=g(model.ctrl_var.ln_inv_s))


def random_packs(rng, n_packs, lo, hi, device="cpu"):
    n = torch.from_numpy(rng.integers(lo, hi, n_packs)).long()
    return torch.stack([n.cumsum(0) - n, n], 1).to(device)


MERGE_MAX_HEADS = 24        # warp_merge_updates (csrc/lotd_device.cuh): a warp with more run heads on a level issues every lane's own updates


def merge_census(x, lotd_cfg, max_level=None, order=None, active=None):
    """The run structure that the warp-merged table-gradient scatter (warp_merge_updates / cell_key3, csrc/lotd_device.cuh) sees.

    x [N, 3]: network-space points.  order [W]: the point each work item (lane) loads, -1 for an invalid lane (it loads x = 0);
    default: the N points in their order.  W is padded with invalid lanes to whole warps of 32.  active [W] bool: the lanes that carry
    gradient (default: the valid ones; k_sdf_bwd_tc also makes a lane with a zero cotangent inactive).
    A lane is a run head if it is inactive, if the previous lane is inactive or if its cell differs from the previous lane's.
    -> dict(levels [L] (level of each contributing pseudo level), mergeable [L] (every axis resolution <= 1024), heads [W/32, L],
            cells [L] of uint32 [W, 3] (cell coordinates per lane), valid [W])"""
    from oracle import lotd as olotd
    from oracle.fused64 import Fused64
    meta = olotd.LoDMeta(3, **lotd_cfg)
    x = np.asarray(x, dtype=np.float32)
    order = np.arange(x.shape[0]) if order is None else np.asarray(order, dtype=np.int64)
    W = -(-order.shape[0] // 32) * 32
    order = np.concatenate([order, np.full(W - order.shape[0], -1, dtype=np.int64)])
    valid = order >= 0
    act = valid.copy() if active is None else np.concatenate([np.asarray(active, dtype=bool), np.zeros(W - len(active), dtype=bool)]) & valid
    xs = Fused64.xs_of(np.where(valid[:, None], x[np.maximum(order, 0)], np.float32(0.0)))
    prev_act = np.concatenate([[False], act[:-1]]).reshape(-1, 32)
    prev_act[:, 0] = False
    levels, mergeable, heads, cells = [], [], [], []
    for psl, lvl, loff, foff, ooff in olotd._level_iter(meta, meta.n_levels if max_level is None else max_level):
        res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
        cell, _ = olotd.pos_fract(xs, (res - 2).astype(np.float32))
        c = cell.reshape(-1, 32, 3)
        differs = np.ones(c.shape[:2], dtype=bool)
        differs[:, 1:] = (c[:, 1:] != c[:, :-1]).any(-1)
        head = ~act.reshape(-1, 32) | ~prev_act | differs
        levels.append(lvl)
        mergeable.append(bool((res <= 1024).all()))
        heads.append(head.sum(1))
        cells.append(cell)
    return dict(levels=np.array(levels), mergeable=np.array(mergeable), heads=np.stack(heads, 1), cells=cells, valid=valid)
