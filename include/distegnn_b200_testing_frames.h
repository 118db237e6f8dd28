/*
 * distegnn_b200_testing_frames.h — the training noise and the rigid transforms of the frame assembly
 * (csrc/frames_noise.cuh, csrc/frames_transform.cuh), exported by libdistegnn_b200_testing.so (csrc/testing/frames_noise.cu,
 * csrc/testing/frames_transform.cu).  NOT part of the product: only tests call them, to restate
 * distegnn_frames_assemble_noise and distegnn_frames_assemble_transform bit for bit.
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

/* For sample ids first .. first + n − 1 under `seed`: R float32 [n,3,3] (device, row-major) and t float32 [n,3] (device)
 * receive the rotation (identity for rotate = 0) and the translation scaled by `translate`, exactly as the assembly
 * applies them; raw uint32 [n,2,4] (device, or NULL) the four Philox words of the rotation and the translation counter.
 * Rejects sample ids outside [0, 2^32), rotate other than 0 / 1 and translate < 0 or not finite.  One launch; no
 * allocation, no synchronisation. */
DISTEGNN_API int distegnn_testing_frames_transform(uint64_t seed, int64_t first, int64_t n, int rotate, float translate,
                                                   float *R, float *t, uint32_t *raw, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_TESTING_FRAMES_H */
