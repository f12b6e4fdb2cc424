"""Generates tests/golden/ref_anneal.npz, the LoTD level schedule, by EXECUTING THE REFERENCE'S OWN multires_annealer.py where a checkout of
the reference project is found (oracle/build_ref.py: reference_root).  The reference is not part of this repository, so the vectors are committed.

    python tests/golden/make_golden_anneal.py

The file is imported as `nr3d_lib.models.grid_encodings.multires_annealer` with the packages above it registered as *empty* packages whose
__path__ points at the reference tree (none of their __init__.py files runs, as in make_golden.py); its one import from the package,
`nr3d_lib.utils.check_to_torch`, is a stub.  What the vectors pin: MultiresAnnealer('hardmask')'s level at every iteration from start_it - 20
to stop_it + 20 (every level change, before start_it and after stop_it) and in its stop state (no iteration given), for the shipped StreetSurf
schedules (start_level 2) and the clamping edges of start_level.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_root  # noqa: E402

# (levels, start_level, update_every, start_it, stop_it) of the schedules in ref_anneal.npz (tests/test_lotd_anneal.py reads them from the file)
CASES = [(L, sl, ue, s0, s1) for L in (12, 16, 17) for sl in (-3, -1, 0, 2, L - 1, L + 2) for ue in (1, 7) for s0, s1 in ((0, 4000), (250, 3000))]


def import_reference_annealer(ref):
    for name, sub in (("nr3d_lib", ""), ("nr3d_lib.models", "/models"), ("nr3d_lib.models.grid_encodings", "/models/grid_encodings")):
        m = types.ModuleType(name)
        m.__path__ = [ref + sub]
        sys.modules[name] = m
    utils = types.ModuleType("nr3d_lib.utils")
    utils.check_to_torch = lambda x, dtype=None, device=None: torch.tensor(x, dtype=dtype, device=device)
    sys.modules["nr3d_lib.utils"] = utils
    return importlib.import_module("nr3d_lib.models.grid_encodings.multires_annealer").MultiresAnnealer


def main():
    if reference_root() is None:
        raise SystemExit("make_golden_anneal.py: no reference checkout found (set NR3D_REFERENCE, or place it next to this repository as `reference`)")
    MA = import_reference_annealer(os.path.join(reference_root(), "nr3d_lib", "nr3d_lib"))
    out = {}
    for k, (L, sl, ue, s0, s1) in enumerate(CASES):
        an = MA([2] * L, "hardmask", stop_it=s1, start_it=s0, update_every=ue, start_level=sl)
        its = np.arange(s0 - 20, s1 + 21)
        out[f"case{k}.cfg"] = np.array([L, sl, ue, s0, s1], dtype=np.int64)
        out[f"case{k}.max_level"] = np.array([an(int(i))[0] for i in its], dtype=np.int8)
        out[f"case{k}.stop_state"] = np.array(an()[0], dtype=np.int8)
    path = os.path.join(ROOT, "tests", "golden", "ref_anneal.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(CASES)} schedules, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
