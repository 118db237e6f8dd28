// The uniform cell grid over a point cloud that the radius build (radius_csr.cu, DESIGN §10) and the rollout's Chamfer
// search (chamfer.cu, DESIGN §20) both build on the device: the ordered-int bounding box, the grid descriptor, the cell
// index of a point with its rounding bound, and the sizing loop.  Each exists once, here: the radius build's cell margin
// and the Chamfer search's stop rule are two readings of the same bound on `axis_cell`, and both hold only as long as
// both passes compute that index with this function.
//
// The sizing functions are `__host__ __device__`: the builds run them in one thread per grid, and the testing library
// exports them (distegnn_radius_grid_size, distegnn_chamfer_grid_size) so that their guarantees are checked on the CPU
// over normal, huge, infinite and NaN extents.
#pragma once
#include <float.h>
#include <stdint.h>

#include "common.cuh"

namespace degnn {

// ---- bounding box of the finite coordinates, in order-preserving ints so that atomicMin / atomicMax apply --------------
__device__ __forceinline__ int ordered_int(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// A bound is bounds6 = min xyz, max xyz; the empty one is (+inf x 3, -inf x 3).
// v into [lo, hi] if it is finite (an inf would stretch the grid over nothing); false if it is not
__device__ __forceinline__ bool bound_add(float& lo, float& hi, float v) {
    const bool finite = isfinite(v);
    if (finite) {
        lo = fminf(lo, v);
        hi = fmaxf(hi, v);
    }
    return finite;
}

// the warp's bound in every lane
__device__ __forceinline__ void bound_warp_reduce(float (&lo)[3], float (&hi)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = fminf(lo[d], __shfl_xor_sync(FULL, lo[d], o));
            hi[d] = fmaxf(hi[d], __shfl_xor_sync(FULL, hi[d], o));
        }
    }
}

// one thread's bound into bounds6; an axis on which it saw no finite coordinate (lo > hi) has nothing to add
__device__ __forceinline__ void bound_flush(int* bounds6, const float (&lo)[3], const float (&hi)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        if (lo[d] <= hi[d]) {
            atomicMin(bounds6 + d, ordered_int(lo[d]));
            atomicMax(bounds6 + 3 + d, ordered_int(hi[d]));
        }
    }
}

// bounds6 -> the grid origin and the extent per axis.  An axis without a finite coordinate gets origin and extent 0; a
// finite range past FLT_MAX gives an extent of +inf, which the sizing turns into one slab on that axis.
__device__ __forceinline__ void bounds_origin_extent(const int* bounds6, float (&o)[3], float (&ext)[3]) {
    for (int k = 0; k < 3; ++k) {
        o[k] = ordered_float(bounds6[k]);
        float hi = ordered_float(bounds6[3 + k]);
        if (!(o[k] <= hi)) o[k] = hi = 0.f;
        ext[k] = hi - o[k];
    }
}

// ---- the grid and the cell of a point -------------------------------------------------------------------------------
struct CellGrid {
    float ox, oy, oz, inv_cell, cell;
    int nx, ny, nz, ncell;     // ncell = nx*ny*nz
};

// Cell index along one axis, in [0, n) for any coordinate: below the origin -> 0, beyond the last cell (+inf included)
// -> n - 1, NaN -> 0.  Monotone in x, so clamping only merges end cells and only shrinks index distances.
//
// Rounding bound.  The index is ⌊u⌋ (clamped), u = fl(fl(x − o) · fl(1/cell)): three fp32 roundings, each at most 2^-24
// relative, of the exact e = (x − o)/cell, which is below 1025 inside the grid (at most 1024 cells per axis).  So
// |u − e| < 3·1025·2^-24 < 1.9e-4 cell, and the u of two points differ from their exact index difference by less than
// 3.7e-4 cell.  kRadiusCellMargin and chamfer.cu's stop rule both rest on this: a change to the expression below (an
// FMA, another clamp) has to be checked against both.
__device__ __forceinline__ int axis_cell(float x, float o, float inv_cell, int n) {
    const float q = (x - o) * inv_cell;
    return q > 0.f ? (q < (float)n ? (int)q : n - 1) : 0;
}

__device__ __forceinline__ void cell_of(const CellGrid& g, float x, float y, float z, int& ix, int& iy, int& iz) {
    ix = axis_cell(x, g.ox, g.inv_cell, g.nx);
    iy = axis_cell(y, g.oy, g.inv_cell, g.ny);
    iz = axis_cell(z, g.oz, g.inv_cell, g.nz);
}

// ---- sizing -----------------------------------------------------------------------------------------------------------
constexpr int kRadiusMaxDim = 1024;          // cells per axis

struct CellGridSize {
    float cell;
    int dims[3];
    int ncell;                               // dims[0]·dims[1]·dims[2]
};

// Cells along one axis of extent `ext` for a cell edge `cell`; kRadiusMaxDim + 1 = does not fit.  An extent that is not a
// finite non-negative number (hi − lo overflowed to +inf, no finite node on the axis, NaN) gets one slab: with one cell
// along an axis every pair is compared along it, whatever the coordinates.
__host__ __device__ inline int radius_axis_cells(float ext, float cell) {
    if (!(ext >= 0.f && ext <= FLT_MAX)) return 1;
    const float q = ext / cell;
    return q < (float)kRadiusMaxDim ? (int)q + 1 : kRadiusMaxDim + 1;
}

// The first cell edge of the sequence first_cell · growth^k (multiplied up in fp32) whose grid has at most kRadiusMaxDim
// cells per axis and at most max_cells cells.  If the edge overflows fp32 first (extents near FLT_MAX), one cell: correct
// for any input, quadratic in the points, reached only by such extents; with one cell the edge does not matter.
__host__ __device__ inline CellGridSize fit_cell_grid(const float ext[3], float first_cell, float growth,
                                                      int64_t max_cells) {
    CellGridSize g;
    for (float cell = first_cell; cell <= FLT_MAX; cell *= growth) {
        bool fits = true;
        int64_t cells = 1;                   // <= 1025^3 < 2^31
        for (int k = 0; k < 3; ++k) {
            g.dims[k] = radius_axis_cells(ext[k], cell);
            fits = fits && g.dims[k] <= kRadiusMaxDim;
            cells *= g.dims[k];
        }
        if (fits && cells <= max_cells) {
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

// The radius build's first cell edge is r·(1 + 2^-10), not r.  By the rounding bound of `axis_cell`, two nodes closer
// than r (or admitted by the fp32 `d2 < r2`, at most ~2^-22 relative beyond r) are less than 1/(1 + 2^-10) + 3.7e-4 <
// 0.9994 cell apart in index space: never two cells apart, so the 27-cell scan compares them.  With the cell exactly r,
// pairs up to 1.5e-5 relative below r fell two cells apart far from the grid origin.
constexpr float kRadiusCellMargin = 1.0f + 1.0f / 1024.0f;

// Grid of the radius build: cell edge r·(1 + 2^-10), grown x1.5 until the dense table of n_graphs x cells fits
// `table_cells` with one spare entry for the scan's end marker (n·P + 1 <= T  <=>  P <= (T − 1)/n in integers).
// Guarantee, for ANY extent (finite, overflowed to +inf, -inf for an axis without a finite node, NaN), any radius > 0
// and any n_graphs with n_graphs + 1 <= table_cells: every dim lies in [1, 1024] and n_graphs·Πdims + 1 <= table_cells,
// so every key graph·ncell + cell lies inside the dense cell table.
__host__ __device__ inline CellGridSize radius_grid_size(const float ext[3], float radius, int n_graphs,
                                                         int64_t table_cells) {
    return fit_cell_grid(ext, radius * kRadiusCellMargin, 1.5f, (table_cells - 1) / n_graphs);
}

constexpr float kChamferGrow = 1.25f;        // cell growth per sizing round: about one point per cell and cloud
constexpr int kChamferRingCap = 6;           // rings searched before a query scans its graph's whole cloud

// Grid of the Chamfer search: the smallest cell edge of the sequence top/1024 · 1.25^k (top = the largest finite extent;
// FLT_MIN if that is 0) whose grid has at most `budget` cells.  There is no radius to start from: fixed-graph rollouts
// have none, and the search only needs a cell that holds about one point.
// Guarantee, for ANY extent (as above) and any budget >= 1: every dim lies in [1, 1024], Πdims <= budget, and the cell
// edge is a normal positive fp32 number.  A graph of n nodes gets a budget of n + 1 cells per cloud, so every key
// graph_base + cell lies inside the graph's part of the cell table.
__host__ __device__ inline CellGridSize chamfer_grid_size(const float ext[3], int64_t budget) {
    float top = 0.f;
    for (int k = 0; k < 3; ++k)
        if (ext[k] >= 0.f && ext[k] <= FLT_MAX && ext[k] > top) top = ext[k];
    float cell = top / (float)kRadiusMaxDim;
    if (!(cell >= FLT_MIN)) cell = FLT_MIN;
    return fit_cell_grid(ext, cell, kChamferGrow, budget);
}

// the grid of origin o and size s
__device__ __forceinline__ CellGrid make_cell_grid(const float (&o)[3], const CellGridSize& s) {
    CellGrid g;
    g.ox = o[0]; g.oy = o[1]; g.oz = o[2];
    g.inv_cell = 1.0f / s.cell;
    g.cell = s.cell;
    g.nx = s.dims[0]; g.ny = s.dims[1]; g.nz = s.dims[2];
    g.ncell = s.ncell;
    return g;
}

}  // namespace degnn
