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

// analytic d(basis)/d(x,y,z); rows dx, dy, dz of length C^2
__device__ __forceinline__ void sh_jacobian(float x, float y, float z, int C, float *dx, float *dy, float *dz) {
    dx[0] = dy[0] = dz[0] = 0.f;
    if (C <= 1) return;
    dx[1] = 0.f; dy[1] = -0.48860251190291987f; dz[1] = 0.f;
    dx[2] = 0.f; dy[2] = 0.f; dz[2] = 0.48860251190291987f;
    dx[3] = -0.48860251190291987f; dy[3] = 0.f; dz[3] = 0.f;
    if (C <= 2) return;
    const float x2 = x * x, y2 = y * y, z2 = z * z;
    dx[4] = 1.0925484305920792f * y;  dy[4] = 1.0925484305920792f * x;  dz[4] = 0.f;
    dx[5] = 0.f;                      dy[5] = -1.0925484305920792f * z; dz[5] = -1.0925484305920792f * y;
    dx[6] = 0.f;                      dy[6] = 0.f;                      dz[6] = 1.8923493915151199f * z;
    dx[7] = -1.0925484305920792f * z; dy[7] = 0.f;                      dz[7] = -1.0925484305920792f * x;
    dx[8] = 1.0925484305920792f * x;  dy[8] = -1.0925484305920792f * y; dz[8] = 0.f;
    if (C <= 3) return;
    dx[9] = -3.5402615395598609f * x * y;            dy[9] = 1.7701307697799304f * (y2 - x2);          dz[9] = 0.f;
    dx[10] = 2.8906114426405538f * y * z;            dy[10] = 2.8906114426405538f * x * z;             dz[10] = 2.8906114426405538f * x * y;
    dx[11] = 0.f;                                    dy[11] = 0.45704579946446572f * (1.0f - 5.0f * z2); dz[11] = -4.5704579946446572f * y * z;
    dx[12] = 0.f;                                    dy[12] = 0.f;                                     dz[12] = 1.1195289977703462f * (5.0f * z2 - 1.0f);
    dx[13] = 0.45704579946446572f * (1.0f - 5.0f * z2); dy[13] = 0.f;                                  dz[13] = -4.5704579946446572f * x * z;
    dx[14] = 2.8906114426405538f * x * z;            dy[14] = -2.8906114426405538f * y * z;            dz[14] = 1.4453057213202769f * (x2 - y2);
    dx[15] = 1.7701307697799304f * (y2 - x2);        dy[15] = 3.5402615395598609f * x * y;             dz[15] = 0.f;
}

}  // namespace nsb
