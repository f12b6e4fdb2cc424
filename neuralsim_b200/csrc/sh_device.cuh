// Real spherical-harmonics basis (degree <= 4), shared by sh.cu and the fused colour kernel.
// Follows nr3d_lib/externals/shencoder/shencoder.cu:33-80.
#pragma once
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ void sh_basis(float x, float y, float z, int C, float *o) {
    o[0] = 0.28209479177387814f;
    if (C <= 1) return;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    if (C <= 2) return;
    const float xy = x * y, yz = y * z, xz = x * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    if (C <= 3) return;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

}  // namespace nsb
