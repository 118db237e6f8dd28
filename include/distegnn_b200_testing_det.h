/*
 * distegnn_b200_testing_det.h — grid-capped twins of the deterministic mode's entry points, exported by
 * libdistegnn_b200_testing.so (csrc/testing/det_capped.cu).  NOT part of the product: only tests call them.
 */
#ifndef DISTEGNN_B200_TESTING_DET_H
#define DISTEGNN_B200_TESTING_DET_H

#include "distegnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The deterministic mode's entry points (distegnn_b200.h, csrc/deterministic.cu) with their grid capped at max_ctas CTAs
 * (0 = no cap).  Same contracts and the same kernels; the results must not depend on the cap.  Tests use them to check
 * that the bits do not depend on the grid. */
DISTEGNN_API int distegnn_edge_layer_fwd_det_capped(int64_t n_nodes, int64_t n_edges, int A, int C, int Na,
                                                    unsigned flags, const int32_t *row, const int32_t *col,
                                                    const float *edge_attr_sorted, const float *x4, const float *P,
                                                    const float *Q, const float *layer_params, float *agg_m,
                                                    float *agg_x, const int32_t *n_edges_dev, void *workspace,
                                                    int64_t workspace_bytes, void *stream, int max_ctas);
DISTEGNN_API int distegnn_edge_combine_det_capped(int64_t n_nodes, int64_t n_edges, int C, const int32_t *row,
                                                  const int32_t *n_edges_dev, float *agg_m, float *agg_x, void *workspace,
                                                  int64_t workspace_bytes, void *stream, int max_ctas);
DISTEGNN_API int distegnn_virtual_layer_fwd_det_capped(int64_t n_nodes, int n_graphs, int A, int C, int Na,
                                                       unsigned flags, const int32_t *batch32, const float *x4,
                                                       const float *Hn, const float *Xv, const float *G,
                                                       const float *layer_params, float *agg_v, float *trans_v,
                                                       float *vsum, void *workspace, int64_t workspace_bytes,
                                                       void *stream, int max_ctas);
DISTEGNN_API int distegnn_vsum_combine_det_capped(int64_t n_nodes, int n_graphs, int C, unsigned flags,
                                                  const int32_t *batch32, const float *x4, float *vsum, void *workspace,
                                                  int64_t workspace_bytes, void *stream, int max_ctas);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_TESTING_DET_H */
