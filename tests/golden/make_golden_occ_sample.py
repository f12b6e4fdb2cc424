"""Generates tests/golden/ref_occ_sample.npz, points drawn in listed voxels by EXECUTING THE REFERENCE'S OWN sample_pts_in_voxels
(nr3d_lib/models/accelerations/occgrid/utils.py:17-41) on the CPU under fixed seeds, where a checkout of the reference project is found
(oracle/build_ref.py: reference_root).  The reference is not part of this repository, so the vectors are committed.

    python tests/golden/make_golden_occ_sample.py

utils.py is loaded from its file with the three modules it imports at the top and does not use in the sampler (torch_scatter,
nr3d_lib.models.annealers, nr3d_lib.maths) registered as empty stand-ins.  The cases (tests/test_occ_update.py reads them from the file)
cover both branches of the sampler and their edge: one voxel, n = 2 nv (the n_per_vox branch), n = 2 nv - 1 (the randint branch) and
more voxels than points.
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

RES = (6, 5, 7)
# (number of listed voxels, points asked for, seed)
CASES = [(1, 1, 0), (1, 2, 1), (1, 9, 2), (17, 34, 3), (17, 33, 4), (40, 7, 5), (210, 100, 6), (210, 420, 7), (33, 1000, 8)]


def import_reference_utils(ref):
    for name in ("torch_scatter", "nr3d_lib", "nr3d_lib.models", "nr3d_lib.models.annealers", "nr3d_lib.maths"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["torch_scatter"].scatter_max = None
    sys.modules["nr3d_lib.models.annealers"].get_anneal_val = None
    sys.modules["nr3d_lib.maths"].normalized_logistic_density = None
    path = os.path.join(ref, "nr3d_lib", "nr3d_lib", "models", "accelerations", "occgrid", "utils.py")
    spec = importlib.util.spec_from_file_location("ref_occgrid_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def case_gidx(nv, seed):
    """nv distinct voxels of the RES grid, in nonzero() order (row-major, last axis fastest)"""
    cells = int(np.prod(RES))
    flat = np.sort(np.random.default_rng(1000 + seed).choice(cells, nv, replace=False))
    return np.stack(np.unravel_index(flat, RES), -1).astype(np.int64)


def main():
    if reference_root() is None:
        raise SystemExit("make_golden_occ_sample.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
    U = import_reference_utils(reference_root())
    out = {}
    for k, (nv, n, seed) in enumerate(CASES):
        gidx = case_gidx(nv, seed)
        torch.manual_seed(seed)
        pts, vidx = U.sample_pts_in_voxels(torch.from_numpy(gidx), n, torch.tensor(RES, dtype=torch.int32))
        for name, v in dict(gidx=gidx, num_pts=np.int64(n), seed=np.int64(seed), pts=pts.numpy(), vidx=vidx.numpy()).items():
            out[f"case{k}.{name}"] = v
    out["res"] = np.array(RES, np.int32)
    path = os.path.join(ROOT, "tests", "golden", "ref_occ_sample.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(CASES)} cases, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
