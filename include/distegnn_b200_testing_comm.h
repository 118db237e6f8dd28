/*
 * distegnn_b200_testing_comm.h — W ranks of the virtual-node exchange on one GPU, exported by libdistegnn_b200_testing.so
 * (csrc/testing/comm_ranks.cu).  NOT part of the product: only tests call them.
 *
 * The exchange (distegnn_allreduce_packed, distegnn_virtual_update_fwd with a communicator) runs one CTA per slot and
 * rank, and the CTAs of different ranks spin on each other's flags.  Here all W ranks run in ONE cooperative launch, so
 * every CTA of every rank is resident at once and the spinning always makes progress.  The device code is the product's
 * (csrc/comm.cuh, csrc/virtual_update_graph.cuh); what differs is the launch and the peers' segments, which are the other
 * communicators' own allocations in this process instead of CUDA-IPC mappings.
 */
#ifndef DISTEGNN_B200_TESTING_COMM_H
#define DISTEGNN_B200_TESTING_COMM_H

#include "distegnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Pause schedules of the twins: before its reduce, CTA (slot s, rank r) of call c waits
 *   DISTEGNN_PAUSE_SEEDED          hash(seed, r, s, c) mod (max_pause_ns + 1) nanoseconds;
 *   DISTEGNN_PAUSE_ONE_SLOW_RANK   max_pause_ns on rank (seed + c) mod world, 0 elsewhere: the slow rank changes with
 *                                  every call.
 * max_pause_ns = 0 is no pause. */
#define DISTEGNN_PAUSE_SEEDED 0
#define DISTEGNN_PAUSE_ONE_SLOW_RANK 1

/* Connects `world` communicators made by distegnn_comm_init in this process (one per rank 0..world-1, in any order) to
 * each other's segments, as distegnn_comm_connect lays them out.  No IPC mapping is opened, so distegnn_comm_destroy
 * closes none.  DISTEGNN_EINVAL: a world outside [1,16] or one the communicators were not made for, a duplicate or
 * missing rank, unequal max_slots, slot stride or device, a communicator that is already connected. */
DISTEGNN_API int distegnn_comm_connect_local(void *const *comms, int world);

/* *packed_ctas / *update_ctas: how many CTAs of the twins' kernels the current device holds at once (occupancy x SMs).
 * A launch of W ranks needs W x slots (W x n_graphs) <= that number, or it is refused with DISTEGNN_EINVAL. */
DISTEGNN_API int distegnn_comm_ranks_capacity(int *packed_ctas, int *update_ctas);

/* distegnn_allreduce_packed on all `world` ranks at once: comms[r] is rank r's communicator (connected), bufs[r] its
 * buffer of calls x count floats.  CTA (s, r) runs `calls` successive all-reduces of slot s of rank r; call c reduces
 * bufs[r] + c·count in place.  `schedule` and max_pause_ns choose the pauses (DISTEGNN_PAUSE_*). */
DISTEGNN_API int distegnn_allreduce_packed_ranks(void *const *comms, int world, float *const *bufs, int64_t count,
                                                 int calls, int schedule, int64_t max_pause_ns, uint64_t seed,
                                                 void *stream);

/* distegnn_virtual_update_fwd with comms[r] on all `world` ranks at once: CTA (b, r) updates graph b of rank r.  The
 * per-rank tensors are arrays of `world` pointers (Hv, G: entries NULL under FLAG_LAST); the parameters and the FLAG_INIT
 * inputs are shared.  Same argument checks as distegnn_virtual_update_fwd.  Pauses: DISTEGNN_PAUSE_SEEDED with c = 0. */
DISTEGNN_API int distegnn_virtual_update_fwd_ranks(void *const *comms, int world, int n_graphs, int A, int C, int Na,
                                                   unsigned flags, float *const *vsum, float *const *Xv,
                                                   float *const *Hv, const float *layer_params,
                                                   const float *next_layer_params, float *const *G,
                                                   const float *init_loc_mean, const float *init_hv0,
                                                   int64_t max_pause_ns, uint64_t seed, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_TESTING_COMM_H */
