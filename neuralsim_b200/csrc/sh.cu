// Real spherical-harmonics embedding of view directions (degree <= 4 -> up to 16 channels) for sm_90a.
// Replaces `_shencoder.sh_encode_forward/backward` (nr3d_lib/externals/shencoder/shencoder.cu:33-,
// 364-387) for the degrees the path uses (CFG `degree: 4`); launches on the caller's stream (the reference ignores
// the current stream).  Outputs are [N, C^2] fp32, the optional Jacobian is [N, 3, C^2] as in the reference.
#include "sh_device.cuh"

namespace nsb {

__global__ void __launch_bounds__(256)
k_sh_fwd(const float *__restrict__ in, float *__restrict__ out, int64_t n, int C, float *__restrict__ dy_dx) {
    const int C2 = C * C;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float x = in[i * 3], y = in[i * 3 + 1], z = in[i * 3 + 2];
        float o[16];
        sh_basis(x, y, z, C, o);
        for (int c = 0; c < C2; ++c) out[i * C2 + c] = o[c];
        if (dy_dx) {
            float dx[16], dy[16], dz[16];
            sh_jacobian(x, y, z, C, dx, dy, dz);
            float *j = dy_dx + i * 3 * C2;
            for (int c = 0; c < C2; ++c) { j[c] = dx[c]; j[C2 + c] = dy[c]; j[2 * C2 + c] = dz[c]; }
        }
    }
}

__global__ void __launch_bounds__(256)
k_sh_bwd(const float *__restrict__ grad, const float *__restrict__ dy_dx, int64_t n, int C, float *__restrict__ gin) {
    const int C2 = C * C;
    const int64_t total = n * 3, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t i = t / 3;
        const int d = (int)(t - i * 3);
        const float *g = grad + i * C2, *j = dy_dx + (i * 3 + d) * C2;
        float a = 0.f;
        for (int c = 0; c < C2; ++c) a = fmaf(g[c], j[c], a);
        gin[t] = a;
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_sh_encode_forward(const float *inputs, float *outputs, int64_t n, int32_t degree, float *dy_dx, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(inputs && outputs, "nsb_sh_encode_forward: NULL argument");
    NSB_REQUIRE(degree >= 1 && degree <= 4, "SH encoder: this build supports degree in [1, 4] (got %d)", degree);
    k_sh_fwd<<<wave_grid(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(inputs, outputs, n, degree, dy_dx);
    return check_launch("nsb_sh_encode_forward");
}

extern "C" int nsb_sh_encode_backward(const float *grad, const float *dy_dx, int64_t n, int32_t degree, float *grad_inputs,
                                      void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(grad && dy_dx && grad_inputs, "nsb_sh_encode_backward: NULL argument");
    NSB_REQUIRE(degree >= 1 && degree <= 4, "SH encoder: this build supports degree in [1, 4] (got %d)", degree);
    k_sh_bwd<<<wave_grid(n * 3, 256, 8), 256, 0, (cudaStream_t)stream>>>(grad, dy_dx, n, degree, grad_inputs);
    return check_launch("nsb_sh_encode_backward");
}
