/*
 * distegnn_b200_testing_frames.h — the training noise of the frame assembly (csrc/frames_noise.cuh), exported by
 * libdistegnn_b200_testing.so (csrc/testing/frames_noise.cu).  NOT part of the product: only tests call it, to restate
 * distegnn_frames_assemble_noise bit for bit.
 */
#ifndef DISTEGNN_B200_TESTING_FRAMES_H
#define DISTEGNN_B200_TESTING_FRAMES_H

#include "distegnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* For scene node ids first .. first + n − 1 of sample `sample` in epoch `epoch` under `seed`: eps_x, eps_v float32 [n,3]
 * (device) receive ε of the position and velocity streams, scaled by sigma_x and sigma_v, exactly as the assembly adds
 * them; raw uint32 [n,2,4] (device, or NULL) the four Philox words of each (node, stream).  Rejects a sample outside
 * [0, 2^32), node ids outside [0, 2^32) and σ < 0 or not finite.  One launch; no allocation, no synchronisation. */
DISTEGNN_API int distegnn_testing_frames_noise(uint64_t seed, uint32_t epoch, int64_t sample, int64_t first, int64_t n,
                                               float sigma_x, float sigma_v, float *eps_x, float *eps_v, uint32_t *raw,
                                               void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_TESTING_FRAMES_H */
