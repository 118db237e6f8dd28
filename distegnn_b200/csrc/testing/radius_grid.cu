// Host-only entry point to the radius build's grid sizing (radius_grid.cuh, include/distegnn_b200_testing_grid.h), so
// that tests without a device can check that every key fits the cell table for any extent.
#include "../../../include/distegnn_b200_testing_grid.h"
#include "../common.cuh"
#include "../radius_grid.cuh"

extern "C" int distegnn_radius_grid_size(const float* ext, float radius, int n_graphs, int64_t table_cells, float* cell,
                                         int32_t* dims, int64_t* ncell) {
    using namespace degnn;
    DEGNN_CHECK_ARG(ext && cell && dims && ncell, "null pointer");
    DEGNN_CHECK_ARG(radius > 0.f, "radius must be > 0");
    DEGNN_CHECK_ARG(table_cells >= 27 && table_cells < ((int64_t)1 << 30), "table_cells outside [27, 2^30)");
    DEGNN_CHECK_ARG(n_graphs > 0 && (int64_t)n_graphs + 1 <= table_cells, "n_graphs outside [1, table_cells - 1]");
    const RadiusGridSize s = radius_grid_size(ext, radius, n_graphs, table_cells);
    *cell = s.cell;
    for (int k = 0; k < 3; ++k) dims[k] = s.dims[k];
    *ncell = s.ncell;
    return DISTEGNN_OK;
}
