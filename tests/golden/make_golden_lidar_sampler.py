"""Generates tests/golden/ref_lidar_sampler.npz by EXECUTING THE REFERENCE'S OWN LidarDataset.sample_merged
(dataio/data_loader/lidar_loader.py:119-204) on the CPU, where a checkout of the reference project is found (oracle/build_ref.py:
reference_root).  The reference is not part of this repository, so the vectors are committed.

    python tests/golden/make_golden_lidar_sampler.py

The scene loader is a stub that serves synthetic merged beams (5 lidars, each frame's beams ordered by lidar, as the reference's merged
data are); the loader's own imports (base_loader, sampler, nr3d_lib.utils) are stubbed as well, since sample_merged uses none of them.
Each draw runs after torch.manual_seed(seed) with the seed recorded, so tests/test_lidar_sampler.py replays it from a CPU generator of
that seed.  A fresh LidarDataset serves every frame: the reference zeroes empty lidars' weights inside its stored multi_lidar_weight
(lidar_loader.py:167-168), which would make a frame's split depend on the frames drawn before it.  Cases (case.meta = F, L, num_rays,
weighted):
  case0  merged_weighted with the shipped weights [0.4, 0.1, 0.1, 0.1, 0.1], 2048 rays: all lidars present (no remainder), lidar 2 empty
         (truncation leaves a remainder for lidar 0), lidar 0 empty (the remainder goes to lidar 1), one lidar alone
  case1  merged_weighted [3, 1, 1, 2, 0.5], 1000 rays: remainders of several rays
  case2  merged_equal, 777 rays, with an empty lidar
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_root  # noqa: E402


def import_reference_lidar_loader(ref):
    """the reference's lidar_loader.py as module ref_data_loader.lidar_loader, its package and nr3d_lib imports stubbed"""
    pkg = types.ModuleType("ref_data_loader")
    pkg.__path__ = []
    base = types.ModuleType("ref_data_loader.base_loader")
    base.SceneDataLoader = object
    sampler = types.ModuleType("ref_data_loader.sampler")
    sampler.get_frame_sampler = lambda *a, **k: (None, None)
    utils = types.ModuleType("nr3d_lib.utils")
    utils.collate_tuple_of_nested_dict = None
    nr3d = sys.modules.get("nr3d_lib") or types.ModuleType("nr3d_lib")
    sys.modules.update({"ref_data_loader": pkg, "ref_data_loader.base_loader": base, "ref_data_loader.sampler": sampler, "nr3d_lib": nr3d,
                        "nr3d_lib.utils": utils})
    spec = importlib.util.spec_from_file_location("ref_data_loader.lidar_loader", os.path.join(ref, "dataio", "data_loader", "lidar_loader.py"))
    m = importlib.util.module_from_spec(spec)
    sys.modules["ref_data_loader.lidar_loader"] = m
    spec.loader.exec_module(m)
    return m


class StubSceneLoader:
    """serves frame f's merged beams: rays_o, rays_d [N, 3], ranges [N], li [N] (non-decreasing)"""

    def __init__(self, frames, n_lidars):
        self.frames = frames
        self.lidar_id_list = [f"lidar_{i}" for i in range(n_lidars)]
        self.scene_bank = {"scene": None}
        self.device = torch.device("cpu")
        self.preload = True

    def get_merged_lidar_gts(self, scene_id, lidar_fi, device=None, filter_if_configured=False):
        return {k: torch.from_numpy(v) for k, v in self.frames[lidar_fi].items()}


def make_frames(g, counts):
    frames = []
    for c in counts:
        n = int(sum(c))
        d = g.normal(size=(n, 3))
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        frames.append(dict(rays_o=g.normal(scale=0.3, size=(n, 3)).astype(np.float32), rays_d=d.astype(np.float32),
                           ranges=g.uniform(1.0, 80.0, n).astype(np.float32), li=np.repeat(np.arange(len(c)), c).astype(np.int64)))
    return frames


CASES = [
    (dict(lidar_sample_mode="merged_weighted", multi_lidar_weight=[0.4, 0.1, 0.1, 0.1, 0.1]), 2048,
     [[3000, 601, 599, 620, 560], [1800, 420, 0, 380, 500], [0, 340, 360, 320, 300], [0, 0, 0, 800, 0]]),
    (dict(lidar_sample_mode="merged_weighted", multi_lidar_weight=[3, 1, 1, 2, 0.5]), 1000, [[500, 300, 200, 100, 50], [700, 0, 3, 5, 1]]),
    (dict(lidar_sample_mode="merged_equal"), 777, [[100, 200, 300, 0, 400], [64, 64, 64, 64, 64]]),
]


def main():
    if reference_root() is None:
        raise SystemExit("make_golden_lidar_sampler.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
    LL = import_reference_lidar_loader(reference_root())
    g = np.random.default_rng(11)
    out = {}
    for k, (kw, num_rays, counts) in enumerate(CASES):
        frames = make_frames(g, counts)
        loader = StubSceneLoader(frames, len(counts[0]))
        p = f"case{k}."
        out[p + "meta"] = np.array([len(counts), len(counts[0]), num_rays, int("weighted" in kw["lidar_sample_mode"])], np.int64)
        out[p + "weight"] = np.array(kw.get("multi_lidar_weight", [0.0] * len(counts[0])), np.float64)
        out[p + "counts"] = np.array(counts, np.int64)
        for key in ("rays_o", "rays_d", "ranges"):
            out[p + key] = np.concatenate([f[key] for f in frames])
        for f in range(len(counts)):
            ds = LL.LidarDataset(loader, num_rays=num_rays, equal_mode="ray_batch", frame_sample_mode="uniform", **kw)
            seed = 100 * k + f
            torch.manual_seed(seed)
            calls, randint = [], torch.randint

            def recording_randint(low, high, size, **kw):        # sample_merged returns neither the split nor the indices
                v = randint(low, high, size, **kw)
                calls.append((low, high, v.clone()))
                return v
            torch.randint = recording_randint
            try:
                sample, gt = ds.sample_merged("scene", f)
            finally:
                torch.randint = randint
            li = sample["rays_sel"].numpy()
            split = np.zeros(len(counts[0]), np.int64)
            cumu = [0, *np.cumsum(counts[f]).tolist()]
            for low, high, v in calls:
                split[[i for i in range(len(split)) if (cumu[i], cumu[i + 1]) == (low, high)][0]] = v.numel()
            inds = torch.cat([v for _, _, v in calls]).numpy()
            q = f"{p}f{f}."
            out.update({q + "seed": np.array(seed, np.int64), q + "split": split.astype(np.int64), q + "inds": inds, q + "li": li,
                        q + "rays_o": sample["rays_o"].numpy(), q + "rays_d": sample["rays_d"].numpy(), q + "ranges": gt["ranges"].numpy(),
                        q + "rays_fidx": sample["rays_fidx"].numpy()})
            assert np.array_equal(frames[f]["rays_o"][inds], out[q + "rays_o"]) and np.array_equal(frames[f]["li"][inds], li)
    path = os.path.join(ROOT, "tests", "golden", "ref_lidar_sampler.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
