"""The drop-in boundary from the reference's side: every backend name the reference's Python wrappers call resolves on the shims of
`install_as_nr3d_lib_bindings()` (SURVEY.md §8b: "all of these names must resolve").  The names were collected from the reference's files
(`_backend.<name>` in the files listed) into tests/golden/reference_backend_names.json."""
import json
import os
import sys
import types

import pytest
import torch  # noqa: F401  (the shims are torch modules)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_backend_names.json")


@pytest.fixture(scope="module")
def shim():
    saved = {k: v for k, v in sys.modules.items() if k == "nr3d_lib" or k.startswith("nr3d_lib.")}
    for k in saved:
        del sys.modules[k]
    import neuralsim_b200.bindings as B
    pkg = types.ModuleType("nr3d_lib")
    pkg.__path__ = []
    sys.modules["nr3d_lib"] = pkg
    B.install_as_nr3d_lib_bindings()
    yield B
    for k in [k for k in sys.modules if k == "nr3d_lib" or k.startswith("nr3d_lib.")]:
        del sys.modules[k]
    sys.modules.update(saved)


def test_every_backend_name_the_reference_calls_exists(shim):
    names = json.load(open(GOLDEN))
    assert set(names) == {"_pack_ops", "_occ_grid", "_lotd", "_shencoder"}
    for mod, rec in names.items():
        assert rec["names"], mod
        assert sys.modules[f"nr3d_lib.bindings.{mod}"] is getattr(shim, mod)
        assert not [n for n in rec["names"] if not hasattr(getattr(shim, mod), n)], mod


def test_placeholders_resolve_and_raise_on_use(shim):
    from nr3d_lib.bindings._forest import ForestMeta, raytrace_cuda_fixed            # the two import-time names (forest.py:26, raytest.py:198)
    import nr3d_lib.bindings._permuto as permuto
    with pytest.raises(RuntimeError, match="_forest.ForestMeta"):
        ForestMeta()
    with pytest.raises(RuntimeError, match="raytrace_cuda_fixed"):
        raytrace_cuda_fixed(None, None)
    with pytest.raises(RuntimeError, match="permutohedral"):
        permuto.permuto_enc_fwd(1, 2, 3)
    with pytest.raises(RuntimeError, match="not built"):
        shim._pack_ops.octree_mark_consecutive_segments(None)
