"""neuralsim_b200 -- H100-native (sm_90a) NeuS volume-rendering hot path behind the nr3d_lib operator boundary.

Layout
  csrc/        hand-written CUDA kernels + the C ABI (include/neuralsim_b200.h) -> libneuralsim_b200.so
  bindings/    ctypes mirror of nr3d_lib.bindings._lotd / _pack_ops / _occ_grid / _shencoder
  graphics/    mirror of nr3d_lib.graphics (pack_ops, raysample, raymarch, neus, nerf utilities)
  fields/      LoTD encoding / LoTDSDF / RadianceNet / LoTDNeuS / occupancy grid accel (the objects ray_query drives)
  renderer.py  ray_test -> ray_query -> volume integration (+ backward), the call bench.py times
There is no CPU fallback: importing works anywhere, calling needs the built library and a CUDA device.
"""
__version__ = "0.1.0"
