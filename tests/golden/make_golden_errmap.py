"""Generates tests/golden/ref_errmap.npz by EXECUTING THE REFERENCE'S OWN ErrorMap and ImpSampler (nr3d_lib/models/importance.py) on the
CPU, where a checkout of the reference project is found (oracle/build_ref.py: reference_root).  The reference is not part of this
repository, so the vectors are committed.

    python tests/golden/make_golden_errmap.py

torch.rand and torch.randint are replaced, while the reference runs, by functions that return draws made here from a fixed numpy seed
(with 0 and 1 - 2^-24 mixed in, so the clamp to [1e-6, 1 - 1e-6] acts) and recorded in the file in call order; tests/test_importance.py
feeds the same draws to the package's restatement.  The script runs under torch.use_deterministic_algorithms(True): without it CPU
torch's index_put_ splits a large batch over threads, and which of the rays that share a cell writes last varies from run to run.  Cases:
  update.*   update_error_map with many rays per cell and per corner statement, xy at 1e-6, 1 - 1e-6 and on cell edges, frames at both ends,
             several successive batches; error_map after each
  cdf.*      construct_cdf with max_pdf None and 1.0, on all-zero maps and on updated maps
  sample.*   ImpSampler.sample_img_pixel at frac_uniform 0, 0.5 and 1, odd n, error_map_hw (32, 64) and (5, 7)
  sched.*    step_error_map over 2000 steps: the steps at which the cdfs were rebuilt (128, x1.5, n_steps_max 500)
  state.*    the state dict of a reference ErrorMap
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_root  # noqa: E402


def import_reference_importance(ref):
    spec = importlib.util.spec_from_file_location("ref_importance", os.path.join(ref, "nr3d_lib", "nr3d_lib", "models", "importance.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


class Draws:
    """stand-ins of torch.rand / torch.randint that hand out (and record) draws from a numpy generator"""

    def __init__(self, seed):
        self.g = np.random.default_rng(seed)
        self.log = []

    def rand(self, *size, dtype=None, device=None, generator=None, **kw):
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple)) else tuple(size)
        v = self.g.random(shape).astype(np.float32)
        flat = v.reshape(-1)
        if flat.size >= 4:
            flat[:: max(flat.size // 3, 1)] = 0.0                       # clamps to 1e-6
            flat[1:: max(flat.size // 3, 1)] = np.float32(1 - 2 ** -24)   # clamps to 1 - 1e-6
        self.log.append(v.copy())
        return torch.from_numpy(v).to(dtype or torch.float32)

    def randint(self, high, size, dtype=None, device=None, generator=None, **kw):
        v = self.g.integers(0, high, tuple(size)).astype(np.int64)
        self.log.append(v.copy())
        return torch.from_numpy(v)


def update_batches(g, n_images, hw, n, n_batches):
    res_y, res_x = hw
    out = []
    for b in range(n_batches):
        fidx = g.choice([0, n_images - 1] if b == 0 else np.arange(n_images), n).astype(np.int64)
        cells = g.integers(0, 6, (n, 2))                            # few distinct cells: many rays per cell and statement
        xy = ((cells + g.choice([0.0, 0.25, 0.5, 0.999], (n, 2))) / np.array([res_x, res_y])).astype(np.float32)
        xy[:7] = np.array([[1e-6, 1e-6], [1 - 1e-6, 1 - 1e-6], [1e-6, 1 - 1e-6], [1.0 / res_x, 2.0 / res_y], [0.5, 0.5],
                           [(res_x - 1) / res_x, (res_y - 1) / res_y], [1 - 1e-6, 0.3]], np.float32)
        val = g.exponential(1.0, n).astype(np.float32)
        val[::11] = 0
        out.append((fidx, xy, val))
    return out


def main():
    if reference_root() is None:
        raise SystemExit("make_golden_errmap.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
    I = import_reference_importance(reference_root())
    torch.use_deterministic_algorithms(True)
    out = {}
    g = np.random.default_rng(7)
    # ---- updates
    for k, (n_images, hw, n, nb) in enumerate([(3, (4, 8), 200, 3), (5, (32, 64), 3001, 2), (1, (2, 2), 33, 2)]):
        m = I.ErrorMap(n_images, hw, device="cpu")
        for b, (fidx, xy, val) in enumerate(update_batches(g, n_images, hw, n, nb)):
            m.update_error_map(torch.from_numpy(fidx), torch.from_numpy(xy), torch.from_numpy(val))
            out.update({f"update{k}.b{b}.fidx": fidx, f"update{k}.b{b}.xy": xy, f"update{k}.b{b}.val": val,
                        f"update{k}.b{b}.error_map": m.error_map.numpy().copy()})
        out[f"update{k}.meta"] = np.array([n_images, hw[0], hw[1], nb], np.int64)
    # ---- cdfs
    for k, (n_images, hw, max_pdf, zero) in enumerate([(4, (32, 64), None, True), (4, (32, 64), None, False), (3, (5, 7), 1.0, False),
                                                       (2, (4, 8), 1.0, True)]):
        m = I.ErrorMap(n_images, hw, max_pdf=max_pdf, device="cpu")
        if not zero:
            m.error_map.copy_(torch.from_numpy((g.exponential(1.0, (n_images,) + hw) * (g.random((n_images,) + hw) > 0.4) * 3).astype(np.float32)))
        out[f"cdf{k}.error_map_in"] = m.error_map.numpy().copy()
        m.construct_cdf()
        out.update({f"cdf{k}.error_map_out": m.error_map.numpy().copy(), f"cdf{k}.cdf_x_cond_y": m.cdf_x_cond_y.numpy(), f"cdf{k}.cdf_y": m.cdf_y.numpy(),
                    f"cdf{k}.cdf_img": m.cdf_img.numpy(), f"cdf{k}.meta": np.array([n_images, hw[0], hw[1], -1 if max_pdf is None else 1], np.int64)})
    # ---- sampling
    for k, (n_images, hw, frac, n) in enumerate([(6, (32, 64), 0.5, 4097), (6, (32, 64), 0.0, 101), (6, (32, 64), 1.0, 77), (3, (5, 7), 0.5, 7),
                                                 (1, (32, 64), 0.5, 1001)]):
        m = I.ErrorMap(n_images, hw, device="cpu")
        m.error_map.copy_(torch.from_numpy((g.exponential(1.0, (n_images,) + hw) * (g.random((n_images,) + hw) > 0.5)).astype(np.float32)))
        m.construct_cdf()
        s = I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=frac)
        d = Draws(1000 + k)
        saved = torch.rand, torch.randint
        torch.rand, torch.randint = d.rand, d.randint
        try:
            i, xy = s.sample_img_pixel(n)
        finally:
            torch.rand, torch.randint = saved
        out.update({f"sample{k}.cdf_x_cond_y": m.cdf_x_cond_y.numpy(), f"sample{k}.cdf_y": m.cdf_y.numpy(), f"sample{k}.cdf_img": m.cdf_img.numpy(),
                    f"sample{k}.i": i.numpy(), f"sample{k}.xy": xy.numpy(), f"sample{k}.meta": np.array([n_images, hw[0], hw[1], n, len(d.log)], np.int64),
                    f"sample{k}.frac": np.array(frac)})
        for j, v in enumerate(d.log):
            out[f"sample{k}.draw{j}"] = v
    # ---- the host schedule
    m = I.ErrorMap(2, (4, 8), n_steps_max=500, device="cpu")
    rebuilt = []
    for it in range(2000):
        before = m.n_steps_between_update
        m.step_error_map(0, torch.full([1, 2], 0.5), torch.ones(1))
        if m.n_steps_since_update == 0:
            rebuilt.append((it, before))
    out["sched.rebuilt"] = np.array(rebuilt, np.int64)
    out["sched.state"] = np.array([m.n_steps_since_update, m.n_steps_between_update], np.int64)
    # ---- the state dict
    sd = I.ErrorMap(3, (4, 8), device="cpu").state_dict()
    out["state.keys"] = np.array(sorted(sd.keys()))
    path = os.path.join(ROOT, "tests", "golden", "ref_errmap.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
