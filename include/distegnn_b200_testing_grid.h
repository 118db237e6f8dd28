/*
 * distegnn_b200_testing_grid.h — the grid sizing of the radius build and of the rollout's Chamfer search on the host,
 * exported by libdistegnn_b200_testing.so (csrc/testing/radius_grid.cu).  NOT part of the product: only tests call it, on machines without a device.
 */
#ifndef DISTEGNN_B200_TESTING_GRID_H
#define DISTEGNN_B200_TESTING_GRID_H

#include "distegnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Host-only: the grid distegnn_radius_graph_csr sizes for bounding-box extents ext[3] (hi - lo over the finite
 * coordinates; +inf, -inf or NaN allowed), `radius`, `n_graphs` graphs and a table of `table_cells` entries: cell edge,
 * dims[3] and ncell = dims[0]*dims[1]*dims[2] per graph (csrc/cell_grid.cuh).  No device needed. */
DISTEGNN_API int distegnn_radius_grid_size(const float *ext, float radius, int n_graphs, int64_t table_cells,
                                           float *cell, int32_t *dims, int64_t *ncell);
/* Host-only: the grid distegnn_rollout_chamfer sizes for one graph of bounding-box extents ext[3] (as above) and a budget
 * of `budget` cells per cloud (the graph's node count + 1): cell edge, dims[3] and ncell (csrc/cell_grid.cuh). */
DISTEGNN_API int distegnn_chamfer_grid_size(const float *ext, int64_t budget, float *cell, int32_t *dims,
                                            int64_t *ncell);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_TESTING_GRID_H */
