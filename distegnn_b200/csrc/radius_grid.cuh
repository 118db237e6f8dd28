// Grid sizing of the on-device radius graph (csrc/radius_csr.cu), one function for the device and the host: the build
// runs it in a single thread, and the testing library exports it (distegnn_radius_grid_size) so that the invariant below
// is checked on the CPU over normal, huge, infinite and NaN extents.
//
// Guarantee, for ANY extent (finite, overflowed to +inf, -inf for an axis without a finite node, NaN), any radius > 0
// and any n_graphs with n_graphs + 1 <= table_cells: every dim lies in [1, 1024] and n_graphs·Πdims + 1 <= table_cells,
// so every key graph·ncell + cell lies inside the dense cell table.
#pragma once
#include <float.h>
#include <stdint.h>

namespace degnn {

// First cell edge = r·(1 + 2^-10).  A node's cell index along an axis is ⌊fl(fl(x − ox) · fl(1/cell))⌋: three fp32
// roundings, each at most 2^-24 relative, of an index below 1025, so the computed index is within 3·1025·2^-24 < 1.9e-4
// cell of the exact (x − ox)/cell, and two nodes' index difference within 3.7e-4 cell of the exact one.  Two nodes
// closer than r (or admitted by the fp32 `d2 < r2`, at most ~2^-22 relative beyond r) are then less than
// 1/(1 + 2^-10) + 3.7e-4 < 0.9994 cell apart in index space: never two cells apart, so the 27-cell scan compares them.
// With the cell exactly r, pairs up to 1.5e-5 relative below r fell two cells apart far from the grid origin.
constexpr float kRadiusCellMargin = 1.0f + 1.0f / 1024.0f;
constexpr int kRadiusMaxDim = 1024;          // cells per axis

struct RadiusGridSize {
    float cell;
    int dims[3];
    int ncell;                               // dims[0]·dims[1]·dims[2] (per graph)
};

// Cells along one axis of extent `ext` for a cell edge `cell`; kRadiusMaxDim + 1 = does not fit.  An extent that is not a
// finite non-negative number (hi − lo overflowed to +inf, no finite node on the axis, NaN) gets one slab: with one cell
// along an axis every pair is compared along it, whatever the coordinates.
__host__ __device__ inline int radius_axis_cells(float ext, float cell) {
    if (!(ext >= 0.f && ext <= FLT_MAX)) return 1;
    const float q = ext / cell;
    return q < (float)kRadiusMaxDim ? (int)q + 1 : kRadiusMaxDim + 1;
}

// Cell edge r·(1 + 2^-10), grown x1.5 until the dense table of n_graphs x cells fits `table_cells` (with one spare entry
// for the scan's end marker).  If the cell overflows fp32 first (extents near FLT_MAX with more graphs than 2 cells per
// axis leave room for), one cell per graph: correct for any input, quadratic per graph, reached only by such extents.
__host__ __device__ inline RadiusGridSize radius_grid_size(const float ext[3], float radius, int n_graphs,
                                                           int64_t table_cells) {
    RadiusGridSize g;
    for (float cell = radius * kRadiusCellMargin; cell <= FLT_MAX; cell *= 1.5f) {
        bool fits = true;
        int64_t cells = n_graphs;            // < 2^31 · 1025^3 < 2^62
        for (int k = 0; k < 3; ++k) {
            g.dims[k] = radius_axis_cells(ext[k], cell);
            fits = fits && g.dims[k] <= kRadiusMaxDim;
            cells *= g.dims[k];
        }
        if (fits && cells + 1 <= table_cells) {
            g.cell = cell;
            g.ncell = g.dims[0] * g.dims[1] * g.dims[2];
            return g;
        }
    }
    g.cell = FLT_MAX;                        // with one cell per graph the edge does not matter
    g.dims[0] = g.dims[1] = g.dims[2] = 1;
    g.ncell = 1;
    return g;
}

}  // namespace degnn
