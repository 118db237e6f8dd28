// The frame assembly's training noise for any range of scene nodes (include/distegnn_b200_testing_frames.h), from the
// same definition the production kernels compile (frames_noise.cuh), so that tests can restate the noisy assembly bit for
// bit and check the generator against an independent Philox.
#include <math.h>

#include "../../../include/distegnn_b200_testing_frames.h"
#include "../common.cuh"
#include "../frames_noise.cuh"

namespace degnn {

__global__ void __launch_bounds__(256) frames_noise_hook_kernel(uint64_t seed, uint32_t epoch, uint32_t sample,
                                                                int64_t first, int64_t n, float sigma_x, float sigma_v,
                                                                float* eps_x, float* eps_v, uint32_t* raw) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (uint32_t q = 0; q < 2; ++q) {
            const uint4 o = noise_raw(seed, epoch, sample, (uint32_t)(first + k), q);
            float e[3];
            noise_eps(o, q == NOISE_POS ? sigma_x : sigma_v, e);
            float* dst = (q == NOISE_POS ? eps_x : eps_v) + k * 3;
            dst[0] = e[0]; dst[1] = e[1]; dst[2] = e[2];
            if (raw) {
                uint32_t* w = raw + (k * 2 + q) * 4;
                w[0] = o.x; w[1] = o.y; w[2] = o.z; w[3] = o.w;
            }
        }
    }
}

}  // namespace degnn

extern "C" int distegnn_testing_frames_noise(uint64_t seed, uint32_t epoch, int64_t sample, int64_t first, int64_t n,
                                             float sigma_x, float sigma_v, float* eps_x, float* eps_v, uint32_t* raw,
                                             void* stream) {
    using namespace degnn;
    const int64_t lim = (int64_t)1 << 32;
    DEGNN_CHECK_ARG(sample >= 0 && sample < lim, "sample outside [0, 2^32)");
    DEGNN_CHECK_ARG(n >= 0 && first >= 0 && first <= lim - n, "node ids outside [0, 2^32)");
    DEGNN_CHECK_ARG(isfinite(sigma_x) && isfinite(sigma_v) && sigma_x >= 0.f && sigma_v >= 0.f,
                    "sigma must be finite and >= 0");
    if (n == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(eps_x && eps_v, "null pointer");
    const int64_t g = (n + 255) / 256;
    const unsigned grid = (unsigned)(g > 8 * (int64_t)sm_count() ? 8 * (int64_t)sm_count() : g);
    frames_noise_hook_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, epoch, (uint32_t)sample, first, n, sigma_x,
                                                                     sigma_v, eps_x, eps_v, raw);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
