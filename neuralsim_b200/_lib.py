"""ctypes loader of libneuralsim_b200.so (the C ABI of include/neuralsim_b200.h).

There is no CPU fallback: if the shared library is missing, or a tensor is not a contiguous CUDA tensor of the
expected dtype, the call raises.  PyTorch is used only to own device memory and streams.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libneuralsim_b200.so")

NSB_MAX_LEVELS, NSB_MAX_DIMS = 32, 4
LOD_DENSE, LOD_HASH = 0, 7


class LotdMetaC(ctypes.Structure):
    _fields_ = [
        ("n_dims_to_encode", ctypes.c_uint32), ("n_levels", ctypes.c_uint32), ("n_pseudo_levels", ctypes.c_uint32),
        ("n_feat_per_pseudo_lvl", ctypes.c_uint32), ("n_encoded_dims", ctypes.c_uint32), ("n_params", ctypes.c_uint32),
        ("level_res", (ctypes.c_uint32 * NSB_MAX_DIMS) * NSB_MAX_LEVELS),
        ("level_n_feats", ctypes.c_uint32 * NSB_MAX_LEVELS), ("level_types", ctypes.c_uint32 * NSB_MAX_LEVELS),
        ("level_sizes", ctypes.c_uint32 * NSB_MAX_LEVELS), ("level_offsets", ctypes.c_uint32 * (NSB_MAX_LEVELS + 1)),
        ("map_levels", ctypes.c_uint32 * (NSB_MAX_LEVELS * 4)), ("map_cnt", ctypes.c_uint32 * (NSB_MAX_LEVELS * 4)),
    ]


class LotdBatchC(ctypes.Structure):
    _fields_ = [("inds", ctypes.c_void_p), ("offsets", ctypes.c_void_p), ("data_size", ctypes.c_uint32)]


class SdfDecoderC(ctypes.Structure):
    _fields_ = [("W1", ctypes.c_void_p), ("b1", ctypes.c_void_p), ("W2", ctypes.c_void_p), ("b2", ctypes.c_void_p),
                ("width", ctypes.c_int32), ("beta", ctypes.c_float)]


class ColorNetC(ctypes.Structure):
    _fields_ = [(k, ctypes.c_void_p) for k in ("W1", "b1", "W2", "b2", "R1", "rb1", "R2", "rb2", "R3", "rb3")] + [
        ("width", ctypes.c_int32), ("rad_width", ctypes.c_int32), ("rad_in", ctypes.c_int32), ("n_appear", ctypes.c_int32),
        ("beta", ctypes.c_float), ("nablas_scale", ctypes.c_float * 3)]


class OccCollectC(ctypes.Structure):
    _fields_ = [("grid_pcl", ctypes.c_void_p), ("res", ctypes.c_int32 * 3), ("inv_s", ctypes.c_float)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"neuralsim_b200: {LIB_PATH} is missing. Build it with `python -m neuralsim_b200.build` "
                "(nvcc, sm_90a). There is no CPU fallback for this package.")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.nsb_last_error.restype = ctypes.c_char_p
        _lib.nsb_launch_count.restype = ctypes.c_uint64
        _lib.nsb_color_tile_bytes.restype = ctypes.c_int64
        _lib.nsb_color_act_bytes.restype = ctypes.c_int64
        _lib.nsb_color_act_bytes.argtypes = [ctypes.c_int64, ctypes.c_int32]
        _lib.nsb_upsample_rays_scratch_floats.restype = ctypes.c_int64
        _lib.nsb_kth_smallest_scratch_bytes.restype = ctypes.c_int64
        _lib.nsb_pose_grad_scratch_floats.restype = ctypes.c_int64
        # marching cubes (csrc/mesh.cu): `level` is a double, which an undeclared ctypes call would not pass
        vp, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
        _lib.nsb_mc_lattice_points.argtypes = [vp, vp, vp, i32, i32, i64, i64, vp, vp]
        _lib.nsb_mc_count.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, f64, vp, vp, vp, vp, vp]
        _lib.nsb_mc_vertices.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, f64, vp, vp, vp, vp, vp, vp, vp]
        _lib.nsb_mc_triangles.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp, vp, i64, vp, vp]
        # the colour backward with the appearance-code gradient: 8 pointers, n, max_level, 23 pointers (activations, cotangents, outputs), stream
        _lib.nsb_fused_color_bwd_appear.argtypes = [vp] * 8 + [i64, i32] + [vp] * 23 + [vp]
        # the backward passes with ray gradients (colour: + view_dirs, codes and rays; SDF: rays)
        _lib.nsb_fused_color_bwd_grads.argtypes = [vp] * 8 + [i64, i32] + [vp] * 28 + [vp]
        _lib.nsb_fused_sdf_bwd_rays.argtypes = [vp] * 9 + [i64, i32] + [vp] * 9 + [vp]
        # the adjoint of the ray test's normalisation and gather (count-aware): idx, n, radius3 (host float[3]), 6 pointers, stream
        _lib.nsb_gather_rays_backward.argtypes = [vp, i64] + [vp] * 7 + [vp]
        # the occupancy grid's update from the network (csrc/occ_update.cu, csrc/occ_ema.cu)
        f32 = ctypes.c_float
        _lib.nsb_occ_voxel_lists.argtypes = [vp, i64] + [vp] * 7
        _lib.nsb_occ_draw_pts.argtypes = [vp] * 5 + [i32] * 4 + [i64, i64, vp, vp, vp]
        _lib.nsb_occ_ema_update_count.argtypes = [vp, vp, vp, i64, i32, f32, i32, i32, i32, vp, vp, vp, vp, f32, f32, vp, vp, vp]
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().nsb_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what}: {msg}" if what else msg)


def slot(cnt, k):
    """device pointer of cnt[k] (an int64 device count block)"""
    return ctypes.c_void_p(cnt.data_ptr() + 8 * k)


def call(fn, what, *args, count=None, level=None):
    """fn(*args) checked.  count = (cnt, k0[, k1]): the launch processes the device-resident counts cnt[k0] (and cnt[k1]) instead of
    its size arguments, which then are the capacities (nsb_bind_device_counts: bound to this thread for the one call, then cleared).
    level: the max_level the call was given; when it is a device int32 scalar, the kernels read it there (nsb_bind_device_max_level, bound
    for the one call) and the host argument c_level(level) is a placeholder."""
    dev_level = isinstance(level, torch.Tensor)
    if count is None and not dev_level:
        check(fn(*args), what)
        return
    l = lib()
    if count is not None:
        l.nsb_bind_device_counts(slot(count[0], count[1]), slot(count[0], count[2]) if len(count) > 2 else _NULL)
    if dev_level:
        l.nsb_bind_device_max_level(ptr(level, "i32", "max_level"))
    try:
        rc = fn(*args)
    finally:
        l.nsb_bind_device_counts(_NULL, _NULL)
        l.nsb_bind_device_max_level(_NULL)
    check(rc, what)


def launch_count() -> int:
    return int(lib().nsb_launch_count())


def stream_ptr():
    """raw cudaStream_t of torch's current stream on the current device (the C-level getter: torch.cuda.current_stream() builds a
    Python Stream object and costs ~17 us per call -- 0.5 ms per step at 30 launches)"""
    try:
        return ctypes.c_void_p(torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice()))
    except AttributeError:       # private API moved: fall back to the public one
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


_DT = {"f32": torch.float32, "f16": torch.float16, "i64": torch.int64, "i32": torch.int32, "u8": torch.uint8,
       "bool": torch.bool}


_NULL = ctypes.c_void_p(0)


def ptr(t, dtype=None, name="tensor", allow_none=False):
    """Device pointer of a contiguous CUDA tensor (raises otherwise)."""
    if t is None:
        if allow_none:
            return _NULL
        raise RuntimeError(f"{name} must not be None")
    try:
        ok = t.is_cuda and t.is_contiguous()
    except AttributeError:
        ok = False
    if not ok:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor (neuralsim_b200 has no CPU path)")
        raise RuntimeError(f"{name} must be contiguous")
    if dtype is not None and t.dtype is not (_DT[dtype] if dtype.__class__ is str else dtype):
        raise RuntimeError(f"{name} must have dtype {_DT[dtype] if isinstance(dtype, str) else dtype}, got {t.dtype}")
    return ctypes.c_void_p(t.data_ptr())


def c_i64(v):
    return ctypes.c_int64(int(v))


def c_i32(v):
    return ctypes.c_int32(int(v))


def c_level(max_level):
    """the int32 max_level argument of a level-aware entry point; for a device level (see call) a placeholder the kernels do not read"""
    return c_i32(-1 if isinstance(max_level, torch.Tensor) else max_level)


def c_f32(v):
    return ctypes.c_float(float(v))


class KernelTimer:
    """Optional per-launch CUDA-event timing of this library's kernels (bench.py's roofline numbers).  Disabled by
    default: then `time()` costs one attribute test.  Events are recorded on the current stream, i.e. the stream the
    kernels are launched on."""

    def __init__(self):
        self.enabled = False
        self._rec = {}

    def enable(self):
        self._rec, self.enabled = {}, True

    def disable(self):
        self.enabled = False

    class _Span:
        def __init__(self, owner, name, units):
            self.o, self.name, self.units = owner, name, units

        def __enter__(self):
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record()

        def __exit__(self, *exc):
            self.b.record()
            self.o._rec.setdefault(self.name, []).append((self.a, self.b, self.units))

    class _Null:
        def __enter__(self):
            return None

        def __exit__(self, *exc):
            return False

    _NULL = _Null()

    def time(self, name, units=0):
        return self._Span(self, name, units) if self.enabled else self._NULL

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for name, spans in self._rec.items():
            out[name] = dict(ms=float(sum(a.elapsed_time(b) for a, b, _ in spans)), units=int(sum(u for _, _, u in spans)),
                             launches=len(spans))
        return out


KERNEL_TIMER = KernelTimer()
