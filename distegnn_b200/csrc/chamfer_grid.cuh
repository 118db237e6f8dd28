// Grid sizing of the rollout's Chamfer search (csrc/chamfer.cu, DESIGN §20), one function for the device and the host:
// the search runs it in one thread per graph, and the testing library exports it (distegnn_chamfer_grid_size) so that
// the invariant below is checked on the CPU over normal, huge, infinite and NaN extents.
//
// Guarantee, for ANY extent (finite, overflowed to +inf, -inf for an axis without a finite node, NaN) and any budget >= 1:
// every dim lies in [1, 1024], dims[0]·dims[1]·dims[2] <= budget, and the cell edge is a normal positive fp32 number.
// A graph of n nodes gets a budget of n + 1 cells per cloud, so every key graph_base + cell lies inside the graph's part
// of the cell table.
#pragma once
#include <float.h>
#include <stdint.h>

#include "radius_grid.cuh"

namespace degnn {

constexpr float kChamferGrow = 1.25f;        // cell growth per sizing round: about one point per cell and cloud
constexpr int kChamferRingCap = 6;           // rings searched before a query scans its graph's whole cloud

// The smallest cell edge of the sequence top/1024 · 1.25^k (top = the largest finite extent; FLT_MIN if that is 0) whose
// grid has at most `budget` cells, dims capped at 1024 per axis.  No cell with the dims in range before the edge
// overflows fp32: one cell (extents near FLT_MAX on all axes).  There is no radius to start from: fixed-graph rollouts
// have none, and the search only needs a cell that holds about one point.
__host__ __device__ inline RadiusGridSize chamfer_grid_size(const float ext[3], int64_t budget) {
    float top = 0.f;
    for (int k = 0; k < 3; ++k)
        if (ext[k] >= 0.f && ext[k] <= FLT_MAX && ext[k] > top) top = ext[k];
    float cell = top / (float)kRadiusMaxDim;
    if (!(cell >= FLT_MIN)) cell = FLT_MIN;
    RadiusGridSize g;
    for (; cell <= FLT_MAX; cell *= kChamferGrow) {
        bool fits = true;
        int64_t cells = 1;                   // <= 1025^3 < 2^31
        for (int k = 0; k < 3; ++k) {
            g.dims[k] = radius_axis_cells(ext[k], cell);
            fits = fits && g.dims[k] <= kRadiusMaxDim;
            cells *= g.dims[k];
        }
        if (fits && cells <= budget) {
            g.cell = cell;
            g.ncell = (int)cells;
            return g;
        }
    }
    g.cell = FLT_MAX;
    g.dims[0] = g.dims[1] = g.dims[2] = 1;
    g.ncell = 1;
    return g;
}

}  // namespace degnn
