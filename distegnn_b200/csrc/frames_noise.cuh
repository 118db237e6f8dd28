// Training noise of the frame assembly (csrc/frames.cu, DESIGN §22): one Gaussian vector per (seed, epoch, sample,
// scene node, stream), a pure function of those five values, so every rank and every launch that needs a node's noise
// regenerates the same bits and nothing is stored between launches.
//
//   (o0,o1,o2,o3) = Philox4x32-10(counter = (j, q, i, e), key = (lo32(s), hi32(s)))
//       j scene-local node id, q stream (0 position, 1 velocity), i sample index, e epoch, s seed
//   u_k = fp32((o_k >> 8)·2^-24 + 2^-25)      in (0, 1]: exact below 1/2, rounded to nearest even above; never 0
//   z_x, z_y = r·cospi(2u1), r·sinpi(2u1) with r = sqrt(−2 ln u0);   z_z = sqrt(−2 ln u2)·cospi(2u3)
//   ε = fp32(σ·z)                              |z| <= sqrt(50 ln 2) ≈ 5.89
//
// Accurate libm functions (the build has no fast-math) and explicit round-to-nearest products: the production kernels
// and the testing hook (csrc/testing/frames_noise.cu) compile this one definition and produce the same bits.
#pragma once
#include <curand_philox4x32_x.h>
#include <stdint.h>

namespace degnn {

enum { NOISE_POS = 0, NOISE_VEL = 1 };

// The noise of one assembly launch.  sample_ids [n_samples] (device) is each batch sample's index in the loader's sample
// list; an id outside [0, 2^32) gives NaN noise, so every noisy value of that sample is NaN.
struct FramesNoise {
    const int64_t* sample_ids;
    uint64_t seed;
    uint32_t epoch;
    float sigma_x, sigma_v;
};

__device__ __forceinline__ uint4 noise_raw(uint64_t seed, uint32_t epoch, uint32_t sample, uint32_t node, uint32_t q) {
    return curand_Philox4x32_10(make_uint4(node, q, sample, epoch), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}

__device__ __forceinline__ float noise_uniform(uint32_t o) {
    return __fadd_rn(__fmul_rn((float)(o >> 8), 0x1p-24f), 0x1p-25f);
}

// σ·z of the four words of one counter (Box–Muller, fp32).
__device__ __forceinline__ void noise_eps(uint4 o, float sigma, float eps[3]) {
    const float r01 = sqrtf(-2.f * logf(noise_uniform(o.x)));
    float s, c;
    sincospif(2.f * noise_uniform(o.y), &s, &c);
    const float r23 = sqrtf(-2.f * logf(noise_uniform(o.z)));
    const float c3 = cospif(2.f * noise_uniform(o.w));
    eps[0] = __fmul_rn(sigma, __fmul_rn(r01, c));
    eps[1] = __fmul_rn(sigma, __fmul_rn(r01, s));
    eps[2] = __fmul_rn(sigma, __fmul_rn(r23, c3));
}

// ε of scene node `node` of batch sample b in stream q.
__device__ __forceinline__ void frames_noise(const FramesNoise& nz, int b, int64_t node, uint32_t q, float eps[3]) {
    const int64_t id = __ldg(nz.sample_ids + b);
    noise_eps(noise_raw(nz.seed, nz.epoch, (uint32_t)id, (uint32_t)node, q), q == NOISE_POS ? nz.sigma_x : nz.sigma_v,
              eps);
    if (id < 0 || id > (int64_t)UINT32_MAX) eps[0] = eps[1] = eps[2] = __int_as_float(0x7fc00000);
}

}  // namespace degnn
