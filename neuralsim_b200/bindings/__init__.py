"""Host-side mirror of the reference's native-extension modules (`nr3d_lib.bindings._*`).

`neuralsim_b200.bindings._lotd / _pack_ops / _occ_grid / _shencoder` export the functions, argument orders and
error behaviour of the pybind11 modules built by nr3d_lib/setup.py, implemented by ctypes calls
into libneuralsim_b200.so.  `install_as_nr3d_lib_bindings()` registers them under the reference's module names so
that an unmodified `nr3d_lib` Python tree imports them (INTEGRATION.md).

The reference imports ALL of its extensions at module import time -- also the ones outside this build's scope
(`graphics/raytest.py:198` -> `_forest.raytrace_cuda_fixed`, `models/spatial/forest.py:26` -> `_forest.ForestMeta`,
`models/grid_encodings/permuto/permuto.py:47` -> `_permuto`, `models/embedders/sinusoidal_cuda/freq.py:13` -> `_freqencoder`,
`graphics/sphere_trace.py:11` -> `_sphere_trace`, `maths/pytorch3d_knn.py:33`, the 3DGS rasteriser).  For those names the
installer registers placeholder modules: every attribute resolves (so `import nr3d_lib.models.fields.neus` succeeds), and
USING one raises a RuntimeError that names the missing extension -- never a silent fallback.
"""
import sys
import types

from . import _lotd, _pack_ops, _occ_grid, _shencoder  # noqa: F401

BUILT = ("_lotd", "_pack_ops", "_occ_grid", "_shencoder")
# extension -> why it is a placeholder here (SURVEY.md §2.1 / §8f)
UNBUILT = {
    "_forest": "forest / octree block spaces (kaolin-based; code_multi large-scale backgrounds) are not built",
    "_permuto": "the permutohedral-lattice encoding (code_multi foreground objects) is not built",
    "_freqencoder": "the CUDA sinusoidal embedder is not built (no shipped NeuS training config selects it)",
    "_sphere_trace": "the sphere-tracing renderer (inference-only query mode) is not built",
    "_pytorch3d_knn": "kNN kernels of the 3DGS experiments are out of scope",
    "_simple_knn": "kNN kernels of the 3DGS experiments are out of scope",
    "_r3dg_rasterization": "the relightable-3DGS rasteriser is a different rendering paradigm, out of scope",
}


class _UnbuiltModule(types.ModuleType):
    """Every attribute resolves to a class that raises when it is called / instantiated."""

    def __init__(self, name, why):
        super().__init__(name)
        self.__dict__["_why"] = why
        self.__dict__["__path__"] = []

    def __getattr__(self, attr):
        if attr.startswith("__"):
            raise AttributeError(attr)
        mod, why = self.__name__, self._why

        class _Unbuilt:
            def __init__(self, *a, **k):
                raise RuntimeError(f"{mod}.{attr}: {why} in neuralsim_b200 (the four hot-path extensions {BUILT} are)")

        _Unbuilt.__name__ = _Unbuilt.__qualname__ = attr
        self.__dict__[attr] = _Unbuilt
        return _Unbuilt


def install_as_nr3d_lib_bindings():
    """Register the shims (and the placeholders) as `nr3d_lib.bindings._*`.  Call before the first `import nr3d_lib...`."""
    pkg = sys.modules.get("nr3d_lib.bindings")
    if pkg is None:
        pkg = types.ModuleType("nr3d_lib.bindings")
        pkg.__path__ = []
        sys.modules["nr3d_lib.bindings"] = pkg
    for name, mod in (("_lotd", _lotd), ("_pack_ops", _pack_ops), ("_occ_grid", _occ_grid), ("_shencoder", _shencoder)):
        sys.modules[f"nr3d_lib.bindings.{name}"] = mod
        setattr(pkg, name, mod)
    for name, why in UNBUILT.items():
        full = f"nr3d_lib.bindings.{name}"
        if full not in sys.modules:
            sys.modules[full] = _UnbuiltModule(full, why)
        setattr(pkg, name, sys.modules[full])
    return pkg
