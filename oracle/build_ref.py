"""Compiles the REFERENCE's own CUDA extensions, from the sources of a checkout of the reference project (neuralsim with its
nr3d_lib submodule), into oracle/_ref/*.so (git-ignored).  TEST INFRASTRUCTURE.  The checkout is found by reference_root():
the NR3D_REFERENCE environment variable if set, else a directory named `reference` next to this repository's checkout.

    python oracle/build_ref.py            # all four hot-path extensions, incremental

This is not the reference's build system (nr3d_lib/setup.py refuses to run without a CUDA device, setup.py:81-83):
the source lists, include directories and nvcc flags of setup.py:86-134 (_lotd), :140-184 (_pack_ops), :495-516
(_occ_grid) and :523-554 (_shencoder) are restated here and handed to torch.utils.cpp_extension.load with
TORCH_CUDA_ARCH_LIST=9.0a (what `compute_{cc}` resolves to on an H100).  No reference source is copied.

Uses: (1) GPU parity tests of our kernels against the reference kernels on identical inputs
(tests/golden/make_ref_golden.py records their outputs for tests/test_ref_parity_gpu.py); (2) the "reference nr3d_lib CUDA path on the
same GPU" timing of BASELINE.md B1.
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def reference_root():
    """the reference checkout: $NR3D_REFERENCE, else <parent of this repository>/reference; None if neither is a directory"""
    root = os.environ.get("NR3D_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
    return root if os.path.isdir(os.path.join(root, "nr3d_lib")) else None


OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")

COMMON = ["-O3", "-DNDEBUG", "-std=c++17", "-Xcompiler=-mf16c", "-Xcompiler=-Wno-float-conversion", "-Xcompiler=-fno-strict-aliasing",
          "-Xcudafe=--diag_suppress=unrecognized_gcc_pragma"]
HALF_ON = ["-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF2_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__"]
HALF_OFF = ["-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__"]

EXTS = {
    "_occ_grid": dict(sources=["csrc/occ_grid/src/ray_marching.cu", "csrc/occ_grid/src/batched_marching.cu", "csrc/occ_grid/src/forest_marching.cu",
                               "csrc/occ_grid/src/occ_grid.cpp"],
                      include=["csrc/occ_grid/include", "csrc/forest"], nvcc=HALF_ON + COMMON),
    # AT_DISPATCH_ALL_TYPES_AND_HALF was removed from ATen (torch >= 2.x spells it AT_DISPATCH_ALL_TYPES_AND(kHalf, ...));
    # the alias is force-included (oracle/ref_compat.h) so that the reference source compiles unmodified.
    "_pack_ops": dict(sources=["csrc/pack_ops/pack_ops_cuda.cu", "csrc/pack_ops/pack_ops.cpp"], include=["csrc/pack_ops"],
                      nvcc=HALF_OFF + COMMON + ["-include", os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_compat.h")]),
    "_shencoder": dict(sources=["externals/shencoder/shencoder.cu", "externals/shencoder/bindings.cpp"], include=["externals/shencoder"],
                       nvcc=HALF_ON + COMMON),
    "_lotd": dict(sources=["csrc/lotd/src/compile_split_1.cu", "csrc/lotd/src/compile_split_2.cu", "csrc/lotd/src/compile_split_3.cu",
                           "csrc/lotd/src/lotd_torch_api.cu", "csrc/lotd/src/lotd.cpp"],
                  include=["csrc/lotd/include", "csrc/forest"], nvcc=["--extended-lambda", "--expt-relaxed-constexpr"] + HALF_ON + COMMON),
}


def build(names=None, verbose=False):
    if reference_root() is None:
        print("oracle/build_ref.py: no reference checkout (set NR3D_REFERENCE, or place it next to this repository as `reference`) "
              "-- using prebuilt oracle/_ref if any")
        return []
    REF = os.path.join(reference_root(), "nr3d_lib")
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 8))
    from torch.utils import cpp_extension
    built = []
    for name in (names or EXTS):
        cfg = EXTS[name]
        bdir = os.path.join(OUT, name)
        os.makedirs(bdir, exist_ok=True)
        try:
            cpp_extension.load(name=name, sources=[os.path.join(REF, s) for s in cfg["sources"]],
                               extra_include_paths=[os.path.join(REF, i) for i in cfg["include"]], extra_cflags=["-O3", "-DNDEBUG", "-std=c++17"],
                               extra_cuda_cflags=cfg["nvcc"], build_directory=bdir, verbose=verbose, is_python_module=True)
            built.append(name)
            print(f"oracle/_ref/{name}: built")
        except Exception as ex:  # recorded, not fatal: the oracle restatement remains the checker
            print(f"oracle/_ref/{name}: BUILD FAILED: {str(ex)[-2000:]}")
    return built


def load(name):
    """Import a prebuilt reference extension from oracle/_ref (None if absent)."""
    import importlib.util
    import torch  # noqa: F401  (the extension links against libtorch)
    so = os.path.join(OUT, name, f"{name}.so")
    if not os.path.exists(so):
        return None
    spec = importlib.util.spec_from_file_location(name, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    build([a for a in sys.argv[1:] if not a.startswith("-")] or None, verbose="-v" in sys.argv)
