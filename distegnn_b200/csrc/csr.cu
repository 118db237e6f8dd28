// Graph preprocessing: int64 COO (edge_index [2,E]) -> int32 CSR: the edges grouped by destination row, the rows of a
// graph contiguous and the graphs in order (DESIGN §3).
// Replaces the implicit scatter-by-edge_index[0] of unsorted_segment_sum/mean
// (reference models/FastEGNN.py:322-337).  Cached per edge_index by the Python side, so it is off the
// per-step path; the sorts are cub's radix sort (library plumbing, not a hot kernel).
//
// Row order.  Without positions the rows come in id order.  With positions (distegnn_build_csr_cells) they come in the
// order of the key (graph, cell of the destination, destination) on a cell_grid.cuh grid of about kCsrNodesPerCell nodes
// per cell: the edge kernel then visits destinations in a spatial sweep, so the neighbour rows Q[col] of the edges in
// flight are rows that nearby destinations have just read, and come from L2 instead of HBM.  Both orders are built the
// same way: the edges are stably sorted by the rank of their destination in the node order (the identity in id order),
// so the edges of a row keep the caller's relative order.  rowptr is the same in both: the exclusive prefix sum of the
// in-degrees in node-id order, which gives every node's in-degree and every graph's edge range.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "cell_grid.cuh"
#include "common.cuh"

namespace degnn {

constexpr int64_t kCsrNodesPerCell = 4;      // cell budget of the row order: about this many nodes per cell

// Ids outside [0,N) are counted into *n_invalid (the reference fails with a device-side index assert on such input) and
// clamped, so nothing downstream can index out of bounds before the host has looked at the counter.  keys[e] = the rank
// of the destination in the node order; deg[r + 1] counts the in-degree of r.
__global__ void csr_keys_kernel(const int64_t* __restrict__ edge_index, int64_t E, int64_t N,
                                const int32_t* __restrict__ rank, int32_t* keys, int32_t* vals, int32_t* deg,
                                int32_t* n_invalid) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) {
        const int64_t r = edge_index[e], c = edge_index[E + e];   // row = edge_index[0, e], col = edge_index[1, e]
        const bool bad = r < 0 || r >= N || c < 0 || c >= N;
        if (bad && n_invalid) atomicAdd(n_invalid, 1);
        const int32_t rc = (int32_t)(r < 0 ? 0 : (r >= N ? N - 1 : r));
        keys[e] = rank ? __ldg(rank + rc) : rc;
        vals[e] = (int32_t)e;
        atomicAdd(deg + rc + 1, 1);
    }
}

// After the sort, which left the sorted ranks in row: col[e'] = edge_index[1, perm[e']], row[e'] = the node of rank
// row[e'] (order == NULL: the identity).
__global__ void csr_finish_kernel(const int64_t* __restrict__ edge_index, int64_t E, int64_t N,
                                  const int32_t* __restrict__ order, const int32_t* __restrict__ perm,
                                  int32_t* __restrict__ row, int32_t* __restrict__ col) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) {
        const int64_t c = edge_index[E + perm[e]];
        col[e] = (int32_t)(c < 0 ? 0 : (c >= N ? N - 1 : c));
        if (order) row[e] = __ldg(order + row[e]);
    }
}

__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ---- node order of distegnn_build_csr_cells: bounding box, grid, (graph, cell) key per node, rank after the sort ------
__global__ void csr_bounds_kernel(const float* __restrict__ pos, int64_t N, int* bounds6) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int d = 0; d < 3; ++d) bound_add(lo[d], hi[d], __ldg(pos + i * 3 + d));
    }
    bound_warp_reduce(lo, hi);
    if ((threadIdx.x & 31) == 0) bound_flush(bounds6, lo, hi);
}

__global__ void csr_bounds_init_kernel(int* bounds6) {
    if (threadIdx.x < 6) bounds6[threadIdx.x] = ordered_int(threadIdx.x < 3 ? INFINITY : -INFINITY);
}

// one thread: the grid over the bounding box with at most `budget` cells per graph
__global__ void csr_grid_kernel(const int* bounds6, int64_t budget, CellGrid* grid) {
    float o[3], ext[3];
    bounds_origin_extent(bounds6, o, ext);
    *grid = make_cell_grid(o, chamfer_grid_size(ext, budget));
}

__global__ void csr_node_keys_kernel(const float* __restrict__ pos, const int64_t* __restrict__ batch, int64_t N, int B,
                                     const CellGrid* __restrict__ grid, int32_t* keys, int32_t* ids) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const CellGrid g = *grid;
    int ix, iy, iz;
    cell_of(g, __ldg(pos + i * 3), __ldg(pos + i * 3 + 1), __ldg(pos + i * 3 + 2), ix, iy, iz);
    keys[i] = graph_id(batch, i, B) * g.ncell + (ix * g.ny + iy) * g.nz + iz;
    ids[i] = (int32_t)i;
}

__global__ void csr_rank_kernel(const int32_t* __restrict__ order, int64_t N, int32_t* rank) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < N) rank[order[k]] = (int32_t)k;
}

__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ perm,
                                   int64_t n, int width, float* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * width) {
        int64_t r = i / width;
        int c = (int)(i - r * width);
        dst[i] = __ldg(src + (int64_t)perm[r] * width + c);
    }
}

__global__ void scatter_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ perm,
                                    int64_t n, int width, float* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * width) {
        int64_t r = i / width;
        int c = (int)(i - r * width);
        dst[(int64_t)perm[r] * width + c] = src[i];
    }
}

static int key_bits(int64_t n) {
    int b = 1;
    while (b < 31 && ((int64_t)1 << b) < n) ++b;
    return b;
}

// cells per graph of the row order, at least one: n_graphs · budget <= max(2^30, n_graphs) <= INT32_MAX, so every
// (graph, cell) key is a non-negative int32 and key_bits(n_graphs · budget) <= 31 covers them all.  The floor matters for
// n_graphs > 2^30, where the cap is 0: a budget of 0 would sort the nodes on one key bit and leave the graphs unordered.
static int64_t cell_budget(int64_t n_nodes, int n_graphs) {
    const int64_t per = n_nodes / ((int64_t)n_graphs * kCsrNodesPerCell) + 1;
    const int64_t cap = ((int64_t)1 << 30) / n_graphs;
    const int64_t budget = per < cap ? per : cap;
    return budget > 1 ? budget : 1;
}

struct CsrLayout {
    size_t keys, vals, deg, nkeys, nids, nskeys, order, rank, bounds, grid, tmp, tmp_bytes, total;
};

// The temporary storage is sized for the widest key the call can sort (31 bits); a narrower sort needs no more.
static cudaError_t csr_layout(int64_t N, int64_t E, CsrLayout& L) {
    size_t sort_e = 0, sort_n = 0, scan = 0;
    cudaError_t e = cudaSuccess;
    if (E > 0)
        e = cub::DeviceRadixSort::SortPairs(nullptr, sort_e, (const int32_t*)nullptr, (int32_t*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)E, 0, 31);
    if (e == cudaSuccess && N > 0)
        e = cub::DeviceRadixSort::SortPairs(nullptr, sort_n, (const int32_t*)nullptr, (int32_t*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)N, 0, 31);
    if (e == cudaSuccess)
        e = cub::DeviceScan::InclusiveSum(nullptr, scan, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(N + 1));
    WorkspaceCursor ws;
    L.keys = ws.take((size_t)E * 4);
    L.vals = ws.take((size_t)E * 4);
    L.deg = ws.take((size_t)(N + 1) * 4);
    L.nkeys = ws.take((size_t)N * 4);
    L.nids = ws.take((size_t)N * 4);
    L.nskeys = ws.take((size_t)N * 4);
    L.order = ws.take((size_t)N * 4);
    L.rank = ws.take((size_t)N * 4);
    L.bounds = ws.take(6 * 4);
    L.grid = ws.take(sizeof(CellGrid));
    L.tmp_bytes = sort_e > sort_n ? sort_e : sort_n;
    if (scan > L.tmp_bytes) L.tmp_bytes = scan;
    L.tmp = ws.take(L.tmp_bytes);
    L.total = ws.end + 256;              // the caller's pointer is aligned up
    return e;
}

// pos == NULL: rows in id order; else in (graph, cell, id) order of `pos` (batch may be NULL for one graph)
static int build_csr(const int64_t* edge_index, int64_t n_nodes, int64_t n_edges, const float* pos,
                     const int64_t* batch, int n_graphs, int32_t* rowptr, int32_t* row, int32_t* col, int32_t* perm,
                     void* workspace, int64_t workspace_bytes, int32_t* n_invalid, cudaStream_t stream) {
    DEGNN_CHECK_ARG(rowptr, "null rowptr");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(n_edges >= 0 && n_edges < INT32_MAX, "n_edges out of int32 range");
    DEGNN_CHECK_ARG(n_graphs >= 1, "n_graphs < 1");
    if (n_invalid) {
        fill_i32_kernel<<<1, 32, 0, stream>>>(n_invalid, 1, 0);
        DEGNN_CHECK_LAUNCH();
    }
    if (n_edges == 0) {
        int64_t n = n_nodes + 1;
        fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(rowptr, n, 0);
        DEGNN_CHECK_LAUNCH();
        return DISTEGNN_OK;
    }
    DEGNN_CHECK_ARG(edge_index && row && col && perm && workspace, "null pointer");
    DEGNN_CHECK_ARG(n_nodes > 0, "edges on an empty node set");
    int64_t need = 0;
    if (int rc = distegnn_csr_workspace_bytes(n_nodes, n_edges, &need)) return rc;
    if (workspace_bytes < need) {
        set_error("distegnn_build_csr: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    CsrLayout L;
    csr_layout(n_nodes, n_edges, L);
    char* ws = (char*)align256((uintptr_t)workspace);
    int32_t* keys = (int32_t*)(ws + L.keys);
    int32_t* vals = (int32_t*)(ws + L.vals);
    int32_t* deg = (int32_t*)(ws + L.deg);
    int32_t* order = nullptr;
    int32_t* rank = nullptr;
    void* tmp = ws + L.tmp;
    size_t tmp_bytes = L.tmp_bytes;
    const unsigned nb = (unsigned)((n_nodes + 255) / 256);
    if (pos) {
        order = (int32_t*)(ws + L.order);
        rank = (int32_t*)(ws + L.rank);
        int* bounds = (int*)(ws + L.bounds);
        CellGrid* grid = (CellGrid*)(ws + L.grid);
        const int64_t budget = cell_budget(n_nodes, n_graphs);
        csr_bounds_init_kernel<<<1, 32, 0, stream>>>(bounds);
        csr_bounds_kernel<<<nb < 1184u ? nb : 1184u, 256, 0, stream>>>(pos, n_nodes, bounds);
        csr_grid_kernel<<<1, 1, 0, stream>>>(bounds, budget, grid);
        csr_node_keys_kernel<<<nb, 256, 0, stream>>>(pos, batch, n_nodes, n_graphs, grid, (int32_t*)(ws + L.nkeys),
                                                     (int32_t*)(ws + L.nids));
        DEGNN_CHECK_LAUNCH();
        const cudaError_t e = cub::DeviceRadixSort::SortPairs(
            tmp, tmp_bytes, (const int32_t*)(ws + L.nkeys), (int32_t*)(ws + L.nskeys), (const int32_t*)(ws + L.nids), order,
            (int)n_nodes, 0, key_bits(n_graphs * budget), stream);
        if (e != cudaSuccess) {
            set_error("distegnn_build_csr: cub sort failed: %s", cudaGetErrorString(e));
            return DISTEGNN_ECUDA;
        }
        csr_rank_kernel<<<nb, 256, 0, stream>>>(order, n_nodes, rank);
    }
    fill_i32_kernel<<<(unsigned)((n_nodes + 1 + 255) / 256), 256, 0, stream>>>(deg, n_nodes + 1, 0);
    const unsigned blocks = (unsigned)((n_edges + 255) / 256);
    csr_keys_kernel<<<blocks, 256, 0, stream>>>(edge_index, n_edges, n_nodes, rank, keys, vals, deg, n_invalid);
    DEGNN_CHECK_LAUNCH();
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, (const int32_t*)keys, row, (const int32_t*)vals, perm,
                                                    (int)n_edges, 0, key_bits(n_nodes), stream);
    if (e == cudaSuccess)
        e = cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, (const int32_t*)deg, rowptr, (int)(n_nodes + 1), stream);
    if (e != cudaSuccess) {
        set_error("distegnn_build_csr: cub sort/scan failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    csr_finish_kernel<<<blocks, 256, 0, stream>>>(edge_index, n_edges, n_nodes, order, perm, row, col);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" {

int distegnn_csr_workspace_bytes(int64_t n_nodes, int64_t n_edges, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(n_edges >= 0 && n_edges < INT32_MAX, "n_edges out of int32 range");
    CsrLayout L;
    cudaError_t e = csr_layout(n_nodes, n_edges, L);
    if (e != cudaSuccess) {
        set_error("cub temp-size query failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    *bytes_host = (int64_t)L.total;
    return DISTEGNN_OK;
}

int distegnn_build_csr(const int64_t* edge_index, int64_t n_nodes, int64_t n_edges, int32_t* rowptr,
                       int32_t* row, int32_t* col, int32_t* perm, void* workspace,
                       int64_t workspace_bytes, int32_t* n_invalid, void* stream) {
    return degnn::build_csr(edge_index, n_nodes, n_edges, nullptr, nullptr, 1, rowptr, row, col, perm, workspace,
                            workspace_bytes, n_invalid, (cudaStream_t)stream);
}

int distegnn_build_csr_cells(const int64_t* edge_index, int64_t n_nodes, int64_t n_edges, const float* pos,
                             const int64_t* data_batch, int n_graphs, int32_t* rowptr, int32_t* row, int32_t* col,
                             int32_t* perm, void* workspace, int64_t workspace_bytes, int32_t* n_invalid,
                             void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(pos || n_edges == 0, "null pos");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    return build_csr(edge_index, n_nodes, n_edges, pos, data_batch, n_graphs, rowptr, row, col, perm, workspace,
                     workspace_bytes, n_invalid, (cudaStream_t)stream);
}

int distegnn_gather_rows(const float* src, const int32_t* perm, int64_t n_rows, int width, float* dst,
                         void* stream_) {
    using namespace degnn;
    if (n_rows == 0 || width == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(src && perm && dst, "null pointer");
    DEGNN_CHECK_ARG(width > 0 && n_rows > 0, "bad shape");
    int64_t n = n_rows * width;
    gather_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(src, perm, n_rows,
                                                                                      width, dst);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int distegnn_scatter_rows(const float* src, const int32_t* perm, int64_t n_rows, int width, float* dst,
                          void* stream_) {
    using namespace degnn;
    if (n_rows == 0 || width == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(src && perm && dst, "null pointer");
    DEGNN_CHECK_ARG(width > 0 && n_rows > 0, "bad shape");
    int64_t n = n_rows * width;
    scatter_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(src, perm, n_rows,
                                                                                       width, dst);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // extern "C"
