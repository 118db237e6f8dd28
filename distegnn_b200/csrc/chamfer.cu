// The rollout's Chamfer distance against recorded frames (DESIGN §20): for step t and graph b, with P the prediction
// and Q = targets[t] over this rank's nodes of b,
//   chamfer[t, b, 0] = Σ_{p in P} min_{q in Q} d(p, q),   chamfer[t, b, 1] = Σ_{q in Q} min_{p in P} d(q, p),
// d = target_sq_dist (rollout_err.cuh), the per-node term of distegnn_rollout_sq_err.  Exact nearest neighbours on a cell
// grid per graph, built on the device from the data every call:
//   1. init: zero the histogram, the per-graph bounds and flags, the ticket
//   2. per-graph bounding box of the finite coordinates of P ∪ Q (ordered-int atomics), and a flag for a graph with a
//      non-finite coordinate
//   3. per-graph grid (cell_grid.cuh): at most n_b + 1 cells per cloud, so graph b's cells of cloud c occupy the keys
//      c·(N + B) + lo_b + b .. + n_b (lo_b its first row): no scan over the graphs, and every key inside the table
//   4. cell key per point, and its rank in the cell (atomicAdd); 5. exclusive scan of the histogram (cub)
//   6. points scattered to start[key] + rank: each cell's points of one cloud are contiguous, in some order
//   7. one thread per point (in cell order), best = d to its matched node: rings of growing Chebyshev radius around its
//      cell in the other cloud's table until the stop rule below holds; past kChamferRingCap rings (an outlier), the
//      whole warp scans the graph's whole other cloud for it
//   8. per-graph sums of the minima, both directions at once, with the sq_err kernel's graph_chunk_sum (rollout_err.cuh)
// A minimum does not depend on the order its candidates are visited in, so the atomics' order never reaches a value.
// Every term of a sum is at most the sq_err term of its row (the matched node is a candidate), and the two sums add in
// the same fixed order (one function), so chamfer[t, b, k] <= sq_err[t, b] bit for bit.
//
// Stop rule.  For an axis with n > 1 cells the computed index of a coordinate x is min(⌊u⌋, n − 1) with u within 1.9e-4
// of the exact (x − o)/c, and two points' u within 3.7e-4 of their exact index difference (the rounding bound of
// `axis_cell`, cell_grid.cuh).  After rings 0..R, a point p not scanned has index distance >= R + 1 to the query q along
// some axis; clamping only shrinks index distances, so |u_p − u_q| > R there and |x_p − x_q| > c·(R − 3.7e-4).  Its d is
// at least the fp64 square of the fp32 difference on that axis, >= (c·(R − 3.7e-4)·(1 − 2^-24))² > (c·R·(1 − 2^-10))²
// for R >= 1.  So the search stops once best <= (c·R·(1 − 2^-10))² (R = 0: best = 0), or once the rings cover the grid:
// no point left can beat best.  An axis with one cell (extent 0, or past FLT_MAX) never separates two points.  This is
// the radius build's cell margin (kRadiusCellMargin, DESIGN §10) read the other way round.
#include <cub/device/device_scan.cuh>

#include "cell_grid.cuh"
#include "common.cuh"
#include "rollout_err.cuh"

namespace degnn {

struct ChamferGrid : CellGrid {
    int base;                  // lo_b + b: the graph's first key in either cloud's table
};

struct ChamferArgs {
    int64_t N;
    int B, steps;
    int64_t T;                 // cells per cloud table: N + B
    const float* pred;         // [N,3]
    const float* targets;      // [steps,N,3]
    const int64_t* batch;      // [N] sorted, or null (one graph)
    const int32_t* counter;    // [0] = the step
    double* chamfer;           // [steps,B,2]
    int* bounds;               // [B,6] ordered-int min xyz / max xyz
    int* flags;                // [B] non-finite coordinate seen
    ChamferGrid* grid;         // [B]
    int2* keyrank;             // [2N] (key, rank in the cell)
    int* cell_start;           // [2T + 1] histogram, then (in place) its exclusive scan
    float4* sorted;            // [2N] (x, y, z, node id) in key order: P in [0, N), Q in [N, 2N)
    double* minima;            // [2N] per-node minima: P -> Q at [0, N), Q -> P at [N, 2N)
    double* slots;             // [chunks, 2]
    unsigned* ticket;
};

__device__ __forceinline__ const float* chf_frame(const ChamferArgs& a) {   // targets[t]; row 0 outside [0, steps)
    const int t = __ldcg(a.counter);
    return a.targets + (t >= 0 && t < a.steps ? (int64_t)t * a.N * 3 : 0);
}

__global__ void chamfer_init_kernel(const ChamferArgs a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= 2 * a.T) a.cell_start[i] = 0;
    if (i < (int64_t)a.B * 6) a.bounds[i] = ordered_int(i % 6 < 3 ? INFINITY : -INFINITY);
    if (i < a.B) a.flags[i] = 0;
    if (i == 0) *a.ticket = 0;
}

constexpr int CHF_WARP_ROWS = 256;   // rows per warp of the bounds pass

// One warp per 256 rows (both clouds).  A warp whose rows lie in one graph reduces them and issues one atomic per bound;
// a warp on a graph boundary issues them per row.
__global__ void __launch_bounds__(256) chamfer_bounds_kernel(const ChamferArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t r0 = w * CHF_WARP_ROWS;
    if (r0 >= a.N) return;
    const int64_t r1 = min(a.N, r0 + CHF_WARP_ROWS);
    const float* tg = chf_frame(a);
    const int g0 = graph_id(a.batch, r0, a.B);
    const bool one = graph_id(a.batch, r1 - 1, a.B) == g0;                // batch sorted: the whole range is graph g0
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    int bad = 0;
    for (int64_t i = r0 + lane; i < r1; i += 32) {
        float l[3] = {INFINITY, INFINITY, INFINITY}, h[3] = {-INFINITY, -INFINITY, -INFINITY};
        int nf = 0;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            if (!bound_add(l[d], h[d], __ldg(a.pred + i * 3 + d))) nf = 1;
            if (!bound_add(l[d], h[d], __ldg(tg + i * 3 + d))) nf = 1;
        }
        if (one) {
#pragma unroll
            for (int d = 0; d < 3; ++d) { lo[d] = fminf(lo[d], l[d]); hi[d] = fmaxf(hi[d], h[d]); }
            bad |= nf;
        } else {
            const int b = graph_id(a.batch, i, a.B);
            bound_flush(a.bounds + (int64_t)b * 6, l, h);
            if (nf) atomicOr(a.flags + b, 1);
        }
    }
    if (!one) return;                                           // warp-uniform
    bound_warp_reduce(lo, hi);
    bad = __any_sync(FULL, bad);
    if (lane == 0) {
        bound_flush(a.bounds + (int64_t)g0 * 6, lo, hi);
        if (bad) atomicOr(a.flags + g0, 1);
    }
}

__global__ void chamfer_grid_kernel(const ChamferArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    int64_t lo, hi;
    graph_rows(a.batch, a.N, b, lo, hi);
    float o[3], ext[3];
    bounds_origin_extent(a.bounds + (int64_t)b * 6, o, ext);
    a.grid[b] = ChamferGrid{make_cell_grid(o, chamfer_grid_size(ext, hi - lo + 1)), (int)(lo + b)};
}

__device__ __forceinline__ float4 chf_point(const ChamferArgs& a, const float* tg, int64_t k, int64_t& i, int& c) {
    c = k >= a.N;
    i = k - c * a.N;
    const float* p = (c ? tg : a.pred) + i * 3;
    return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __int_as_float((int)i));
}

__global__ void __launch_bounds__(256) chamfer_keys_kernel(const ChamferArgs a) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= 2 * a.N) return;
    int64_t i;
    int c;
    const float4 p = chf_point(a, chf_frame(a), k, i, c);
    const ChamferGrid g = a.grid[graph_id(a.batch, i, a.B)];
    int ix, iy, iz;
    cell_of(g, p.x, p.y, p.z, ix, iy, iz);
    const int key = (int)(c * a.T) + g.base + (ix * g.ny + iy) * g.nz + iz;
    a.keyrank[k] = make_int2(key, atomicAdd(a.cell_start + key, 1));
}

__global__ void __launch_bounds__(256) chamfer_scatter_kernel(const ChamferArgs a) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= 2 * a.N) return;
    int64_t i;
    int c;
    const float4 p = chf_point(a, chf_frame(a), k, i, c);
    const int2 kr = a.keyrank[k];
    a.sorted[__ldg(a.cell_start + kr.x) + kr.y] = p;
}

// (c·R·(1 − 2^-10))²: no point outside rings 0..R of the query's cell is nearer (the stop rule above)
__device__ __forceinline__ double chf_ring_bound(float cell, int R) {
    const double r = (double)cell * (double)R * (1.0 - 1.0 / 1024.0);
    return r * r;
}

__global__ void __launch_bounds__(256) chamfer_search_kernel(const ChamferArgs a) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool live = s < 2 * a.N;                             // every lane reaches the warp's outlier scans below
    const float4 q = live ? a.sorted[s] : make_float4(0.f, 0.f, 0.f, 0.f);
    const int c = s >= a.N;                                    // the query's cloud; it searches the other one
    const int64_t i = __float_as_int(q.w);
    const int b = live ? graph_id(a.batch, i, a.B) : 0;
    const bool search = live && !__ldg(a.flags + b);           // a non-finite coordinate in the graph: NaN sums
    const ChamferGrid g = a.grid[b];
    const int* start = a.cell_start + (1 - c) * a.T + g.base;
    double best = INFINITY;
    auto dist = [&](const float4& v) {
        return target_sq_dist([&](int k) { return xyz(q, k); }, [&](int k) { return xyz(v, k); });
    };
    bool outlier = false;
    if (search) {
        // the matched node is a candidate: best starts at the node's sq_err term
        const float* m = (c ? a.pred : chf_frame(a)) + i * 3;
        best = dist(make_float4(__ldg(m), __ldg(m + 1), __ldg(m + 2), 0.f));
        int ix, iy, iz;
        cell_of(g, q.x, q.y, q.z, ix, iy, iz);
        const int reach = max(max(max(ix, g.nx - 1 - ix), max(iy, g.ny - 1 - iy)), max(iz, g.nz - 1 - iz));
        auto scan = [&](int k0, int k1) {                      // the points of cells k0 .. k1 − 1
            const int e = __ldg(start + k1);
            for (int p = __ldg(start + k0); p < e; ++p) best = fmin(best, dist(a.sorted[p]));
        };
        for (int R = 0;; ++R) {
            // rings 0 .. R − 1 are scanned: no point left is nearer than their bound (none scanned: 0)
            if (best <= (R > 0 ? chf_ring_bound(g.cell, R - 1) : 0.0) || R > reach) break;
            if (R > kChamferRingCap) {                         // an outlier: the graph's whole other cloud, below
                outlier = true;
                break;
            }
            for (int cx = max(ix - R, 0); cx <= min(ix + R, g.nx - 1); ++cx) {
                for (int cy = max(iy - R, 0); cy <= min(iy + R, g.ny - 1); ++cy) {
                    const int row = (cx * g.ny + cy) * g.nz;
                    if (abs(cx - ix) == R || abs(cy - iy) == R) {   // a face of the ring in x or y: its whole z range
                        scan(row + max(iz - R, 0), row + min(iz + R, g.nz - 1) + 1);
                    } else {                                   // inside: the two z faces
                        if (iz - R >= 0) scan(row + iz - R, row + iz - R + 1);
                        if (iz + R < g.nz) scan(row + iz + R, row + iz + R + 1);
                    }
                }
            }
        }
    }
    // Outliers: the whole warp scans each one's cloud, lane l taking every 32nd point, then a min over the lanes.
    for (unsigned need = __ballot_sync(FULL, outlier); need; need &= need - 1) {
        const int L = __ffs(need) - 1;
        const float4 o = make_float4(__shfl_sync(FULL, q.x, L), __shfl_sync(FULL, q.y, L), __shfl_sync(FULL, q.z, L), 0.f);
        const int* st = start;                                 // lane L's table and graph
        const int lo = __shfl_sync(FULL, __ldg(st), L);
        const int hi = __shfl_sync(FULL, __ldg(st + g.ncell), L);
        double m = INFINITY;
#pragma unroll 4
        for (int p = lo + lane; p < hi; p += 32) {
            const float4 v = a.sorted[p];
            m = fmin(m, target_sq_dist([&](int k) { return xyz(o, k); }, [&](int k) { return xyz(v, k); }));
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmin(m, __shfl_xor_sync(FULL, m, off));
        if (lane == L) best = fmin(best, m);
    }
    if (live) a.minima[c * a.N + i] = search ? best : __longlong_as_double(0x7ff8000000000000ll);
}

// distegnn_rollout_sq_err's reduction on the per-node minima, both directions at once.  The workspace is not
// initialised: the init kernel zeroes the ticket.
__global__ void __launch_bounds__(DET_RED) chamfer_sum_kernel(const ChamferArgs a) {
    const int t = __ldcg(a.counter);
    const bool keep = t >= 0 && t < a.steps;
    graph_chunk_sum<2>(a.N, a.B, a.batch, keep, a.chamfer + (keep ? (int64_t)t * a.B * 2 : 0), a.slots, a.ticket,
                       [&](int64_t k, double (&s)[2]) {
                           s[0] += __ldg(a.minima + k);
                           s[1] += __ldg(a.minima + a.N + k);
                       });
}

struct ChamferLayout {
    size_t bounds, flags, grid, keyrank, cell_start, sorted, minima, slots, ticket, tmp, tmp_bytes, total;
};

static int chamfer_layout(int64_t N, int B, ChamferLayout& L) {
    const int64_t T = N + B;
    size_t scan = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(2 * T + 1)) !=
        cudaSuccess)
        return DISTEGNN_ECUDA;
    WorkspaceCursor ws;
    L.bounds = ws.take((size_t)B * 6 * 4);
    L.flags = ws.take((size_t)B * 4);
    L.grid = ws.take((size_t)B * sizeof(ChamferGrid));
    L.keyrank = ws.take((size_t)N * 2 * sizeof(int2));
    L.cell_start = ws.take((size_t)(2 * T + 1) * 4);
    L.sorted = ws.take((size_t)N * 2 * sizeof(float4));
    L.minima = ws.take((size_t)N * 2 * 8);
    L.slots = ws.take((size_t)err_chunks(N) * 2 * 8);
    L.ticket = ws.take(4);
    L.tmp_bytes = scan;
    L.tmp = ws.take(scan);
    L.total = ws.end;
    return DISTEGNN_OK;
}

constexpr int64_t CHF_MAX_ROWS = (int64_t)1 << 29;   // N + n_graphs: the table's 2(N + B) + 1 keys stay in int32

}  // namespace degnn

extern "C" {

int distegnn_rollout_chamfer_workspace_bytes(int64_t n_nodes, int n_graphs, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(n_nodes + n_graphs <= CHF_MAX_ROWS, "n_nodes + n_graphs above 2^29");
    ChamferLayout L;
    if (int rc = chamfer_layout(n_nodes, n_graphs, L)) {
        set_error("cub temp-size query failed");
        return rc;
    }
    *bytes_host = (int64_t)L.total;
    return DISTEGNN_OK;
}

int distegnn_rollout_chamfer(int64_t n_nodes, int n_graphs, int steps, const float* pred, const float* targets,
                             const int64_t* data_batch, const int32_t* counter, double* chamfer, void* workspace,
                             int64_t workspace_bytes, void* stream_) {
    using namespace degnn;
    cudaStream_t stream = (cudaStream_t)stream_;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0 && steps >= 1, "bad size");
    DEGNN_CHECK_ARG(n_nodes + n_graphs <= CHF_MAX_ROWS, "n_nodes + n_graphs above 2^29");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    DEGNN_CHECK_ARG(counter && chamfer, "null pointer");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(pred && targets && workspace, "null pointer");
    DEGNN_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace not 16-byte aligned");
    ChamferLayout L;
    if (int rc = chamfer_layout(n_nodes, n_graphs, L)) {
        set_error("cub temp-size query failed");
        return rc;
    }
    if (workspace_bytes < (int64_t)L.total) {
        set_error("distegnn_rollout_chamfer: workspace %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)L.total);
        return DISTEGNN_EWORKSPACE;
    }
    char* ws = (char*)workspace;
    ChamferArgs a;
    a.N = n_nodes; a.B = n_graphs; a.steps = steps; a.T = n_nodes + n_graphs;
    a.pred = pred; a.targets = targets; a.batch = n_graphs > 1 ? data_batch : nullptr; a.counter = counter;
    a.chamfer = chamfer;
    a.bounds = (int*)(ws + L.bounds); a.flags = (int*)(ws + L.flags); a.grid = (ChamferGrid*)(ws + L.grid);
    a.keyrank = (int2*)(ws + L.keyrank); a.cell_start = (int*)(ws + L.cell_start); a.sorted = (float4*)(ws + L.sorted);
    a.minima = (double*)(ws + L.minima); a.slots = (double*)(ws + L.slots); a.ticket = (unsigned*)(ws + L.ticket);
    size_t tmp_bytes = L.tmp_bytes;
    const int64_t init = 2 * a.T + 1 > (int64_t)n_graphs * 6 ? 2 * a.T + 1 : (int64_t)n_graphs * 6;
    const unsigned nb2 = (unsigned)((2 * n_nodes + 255) / 256);
    const int64_t warps = (n_nodes + CHF_WARP_ROWS - 1) / CHF_WARP_ROWS;
    chamfer_init_kernel<<<(unsigned)((init + 255) / 256), 256, 0, stream>>>(a);
    chamfer_bounds_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(a);
    chamfer_grid_kernel<<<(unsigned)((n_graphs + 127) / 128), 128, 0, stream>>>(a);
    chamfer_keys_kernel<<<nb2, 256, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(ws + L.tmp, tmp_bytes, (const int32_t*)a.cell_start,
                                                        a.cell_start, (int)(2 * a.T + 1), stream);
    if (e != cudaSuccess) {
        set_error("distegnn_rollout_chamfer: cub scan failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    chamfer_scatter_kernel<<<nb2, 256, 0, stream>>>(a);
    chamfer_search_kernel<<<nb2, 256, 0, stream>>>(a);
    chamfer_sum_kernel<<<(unsigned)err_chunks(n_nodes), DET_RED, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // extern "C"
