"""Builds libneuralsim_b200.so (C ABI, sm_90a only: H100) in-tree with nvcc.

    python -m neuralsim_b200.build            # incremental
    python -m neuralsim_b200.build --force

The library links only against cudart (static); no torch / ATen is involved, so it can be loaded by any host
(ctypes here, cgo/JNI/pybind11 elsewhere -- see INTEGRATION.md).  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_build")
LIB = os.path.join(HERE, "libneuralsim_b200.so")
SOURCES = ["common.cu", "lotd.cu", "march.cu", "pack_ops.cu", "sh.cu", "fused.cu", "fused_tc.cu", "neus_fused.cu", "neus_glue.cu", "color_tc.cu", "ray_upsample.cu", "occ_ema.cu", "mesh.cu", "lidar_loss.cu", "pose.cu", "perturb.cu", "importance.cu", "lidar_sample.cu", "occ_update.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I", os.path.join(os.path.dirname(HERE), "include")]


def _deps_mtime():
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            if f.endswith((".cuh", ".h")):
                m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def _compile(src, force, hdr_mtime, verbose):
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    path = os.path.join(CSRC, src)
    if (not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(path), hdr_mtime)):
        return obj, ""
    r = subprocess.run([NVCC, *FLAGS, "-c", path, "-o", obj], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
    log = r.stderr
    with open(obj + ".ptxas.log", "w") as f:
        f.write(log)
    return obj, log


def build_library(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr = _deps_mtime()
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        res = list(ex.map(lambda s: _compile(s, force, hdr, verbose), SOURCES))
    objs = [o for o, _ in res]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, *ARCH, "-cudart", "static"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        for _, log in res:
            for line in log.splitlines():
                if "registers" in line or "spill" in line and "0 bytes spill" not in line:
                    print(line)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
