// The frame assembly's rigid transforms for any range of sample ids (include/distegnn_b200_testing_frames.h), from the
// same definition the production kernels compile (frames_transform.cuh), so that tests can restate the transformed
// assembly bit for bit and check the generator against an independent Philox.
#include <math.h>

#include "../../../include/distegnn_b200_testing_frames.h"
#include "../common.cuh"
#include "../frames_transform.cuh"

namespace degnn {

__global__ void __launch_bounds__(256) frames_transform_hook_kernel(uint64_t seed, int64_t first, int64_t n, int rotate,
                                                                    float translate, float* R, float* t,
                                                                    uint32_t* raw) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t sample = (uint32_t)(first + k);
        Rigid T;
        rigid_of(seed, sample, rotate != 0, translate, T);
#pragma unroll
        for (int e = 0; e < 9; ++e) R[k * 9 + e] = T.r[e];
        t[k * 3] = T.t[0]; t[k * 3 + 1] = T.t[1]; t[k * 3 + 2] = T.t[2];
        if (raw) {
#pragma unroll
            for (uint32_t q = 0; q < 2; ++q) {
                const uint4 o = noise_raw(seed, 0, sample, 0, XFORM_ROT + q);
                uint32_t* w = raw + (k * 2 + q) * 4;
                w[0] = o.x; w[1] = o.y; w[2] = o.z; w[3] = o.w;
            }
        }
    }
}

}  // namespace degnn

extern "C" int distegnn_testing_frames_transform(uint64_t seed, int64_t first, int64_t n, int rotate, float translate,
                                                 float* R, float* t, uint32_t* raw, void* stream) {
    using namespace degnn;
    const int64_t lim = (int64_t)1 << 32;
    DEGNN_CHECK_ARG(n >= 0 && first >= 0 && first <= lim - n, "sample ids outside [0, 2^32)");
    DEGNN_CHECK_ARG(rotate == 0 || rotate == 1, "rotate must be 0 or 1");
    DEGNN_CHECK_ARG(isfinite(translate) && translate >= 0.f, "translate must be finite and >= 0");
    if (n == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(R && t, "null pointer");
    const int64_t g = (n + 255) / 256;
    const unsigned grid = (unsigned)(g > 8 * (int64_t)sm_count() ? 8 * (int64_t)sm_count() : g);
    frames_transform_hook_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, first, n, rotate, translate, R, t, raw);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
