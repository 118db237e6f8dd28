// On-device radius graph, CSR out, no host round trip (SURVEY §8 f-2).
//
// Replaces the CPU `radius_graph(pos_i, r=radius, max_num_neighbors=N)` + `edge_attr = ‖Δx‖ duplicated` of the reference's
// partitioners (datasets/distribute_graphs.py:43-44, PyG / torch_cluster on the host, then an int64 edge_index that the
// model has to sort) with ONE call that takes the reference-boundary tensors (pos [N,3] fp32, data_batch int64) and leaves
// the graph in the form the edge kernels consume: int32 CSR by destination row (rowptr / row / col) and edge_attr in CSR
// order.  Everything the host used to decide is decided on the device, so the call neither synchronises nor needs the
// edge count in advance (the caller passes a CAPACITY; the true count lands in info[0], an overflow flag in info[1]):
//   1. bounding box of the finite coordinates (block reduction + ordered-int atomics)
//   2. uniform grid (radius_grid.cuh): cell size = radius·(1 + 2^-10), grown x1.5 until the dense cell table fits the
//      caller's table_cells; every key lies inside the table for any position, ±inf and NaN included
//   3. cell key per node + histogram; exclusive scan of the histogram = first position of every cell (cub)
//   4. node ids sorted by key (cub radix sort), so that a warp scans neighbouring cells together
//   5. count pass (27 cells as 9 contiguous key ranges) -> degrees -> exclusive scan = rowptr (cub)
//   6. fill pass: col, row, edge length into edge_attr columns, at rowptr offsets
// `dist < r` as torch_cluster (strict, the fp32 `d2 < r2`), j != i unless `loop`, same graph id only.  A node with a
// non-finite coordinate has an inf or NaN d2 to every node, itself included, so it gets no edges.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "radius_grid.cuh"

namespace degnn {

struct GridDev {
    float ox, oy, oz, inv_cell;
    int nx, ny, nz, ncell;     // ncell = nx*ny*nz (per graph)
};

struct RcsrArgs {
    int64_t N, capacity, table_cells;
    int B, A, loop;
    float radius;
    const float* pos;          // [N,3]
    const int64_t* batch64;    // [N] or null
    int* bounds;               // [6] ordered-int encoded min xyz / max xyz
    GridDev* grid;
    float* x4;                 // [N,4]
    int32_t* batch32;          // [N]
    int32_t* keys;             // [N]
    int32_t* ids;              // [N] 0..N-1
    int32_t* skeys;            // [N] sorted keys (unused after the sort)
    int32_t* order;            // [N] node ids in key order
    int32_t* cell_cnt;         // [table_cells + 1] histogram, then (in place) exclusive scan = cell_start
    int32_t* deg;              // [N + 1]
    int32_t* rowptr;           // [N + 1]
    int32_t* row;              // [capacity]
    int32_t* col;              // [capacity]
    float* edge_attr;          // [capacity, A] or null
    int32_t* info;             // [4]: edges found, overflow flag, cells used, reserved
};

__device__ __forceinline__ int f2ord(float f) {      // order-preserving float -> int
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void rcsr_init_kernel(const RcsrArgs a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= a.table_cells) a.cell_cnt[i] = 0;
    if (i < 3) a.bounds[i] = f2ord(INFINITY);
    if (i >= 3 && i < 6) a.bounds[i] = f2ord(-INFINITY);
    if (i < 4) a.info[i] = 0;
}

__global__ void __launch_bounds__(256) rcsr_bounds_kernel(const RcsrArgs a) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.N; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float v = __ldg(a.pos + i * 3 + d);
            if (isfinite(v)) {                            // an inf would stretch the grid over nothing
                lo[d] = fminf(lo[d], v);
                hi[d] = fmaxf(hi[d], v);
            }
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = fminf(lo[d], __shfl_xor_sync(FULL, lo[d], o));
            hi[d] = fmaxf(hi[d], __shfl_xor_sync(FULL, hi[d], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(a.bounds + d, f2ord(lo[d]));
            atomicMax(a.bounds + 3 + d, f2ord(hi[d]));
        }
    }
}

__global__ void rcsr_grid_kernel(const RcsrArgs a) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    GridDev g;
    float lo[3], ext[3];
    for (int k = 0; k < 3; ++k) {
        lo[k] = ord2f(a.bounds[k]);
        float hi = ord2f(a.bounds[3 + k]);
        if (!(lo[k] <= hi)) lo[k] = hi = 0.f;        // no finite coordinate on this axis
        ext[k] = hi - lo[k];                          // +inf if the finite range exceeds FLT_MAX: one slab on that axis
    }
    const RadiusGridSize s = radius_grid_size(ext, a.radius, a.B, a.table_cells);
    g.ox = lo[0]; g.oy = lo[1]; g.oz = lo[2];
    g.inv_cell = 1.0f / s.cell;
    g.nx = s.dims[0]; g.ny = s.dims[1]; g.nz = s.dims[2];
    g.ncell = s.ncell;
    *a.grid = g;
    a.info[2] = g.ncell * a.B;
}

// Cell index along one axis, in [0, n) for any coordinate: below the origin -> 0, beyond the last cell (+inf included)
// -> n - 1, NaN -> 0.  Monotone in x, so clamping only merges end cells, which the 27-cell scan still covers.
__device__ __forceinline__ int axis_cell(float x, float o, float inv_cell, int n) {
    const float q = (x - o) * inv_cell;
    return q > 0.f ? (q < (float)n ? (int)q : n - 1) : 0;
}

__device__ __forceinline__ void cell_of(const GridDev& g, float x, float y, float z, int& ix, int& iy, int& iz) {
    ix = axis_cell(x, g.ox, g.inv_cell, g.nx);
    iy = axis_cell(y, g.oy, g.inv_cell, g.ny);
    iz = axis_cell(z, g.oz, g.inv_cell, g.nz);
}

__global__ void __launch_bounds__(256) rcsr_keys_kernel(const RcsrArgs a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) a.deg[a.N] = 0;
    if (i >= a.N) return;
    const GridDev g = *a.grid;
    const float x = __ldg(a.pos + i * 3), y = __ldg(a.pos + i * 3 + 1), z = __ldg(a.pos + i * 3 + 2);
    *reinterpret_cast<float4*>(a.x4 + i * 4) = make_float4(x, y, z, 0.f);
    int b = 0;
    if (a.batch64) {
        const int64_t bb = a.batch64[i];
        b = (int)(bb < 0 ? 0 : (bb >= a.B ? a.B - 1 : bb));
    }
    a.batch32[i] = b;
    int ix, iy, iz;
    cell_of(g, x, y, z, ix, iy, iz);
    const int key = b * g.ncell + (ix * g.ny + iy) * g.nz + iz;
    a.keys[i] = key;
    a.ids[i] = (int32_t)i;
    atomicAdd(a.cell_cnt + key, 1);
}

template <bool FILL>
__global__ void __launch_bounds__(256) rcsr_scan_kernel(const RcsrArgs a) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.N) return;
    const GridDev g = *a.grid;
    const int i = __ldg(a.order + k);
    const float4 p = ldg4(a.x4 + (size_t)i * 4);
    const int b = __ldg(a.batch32 + i);
    int ix, iy, iz;
    cell_of(g, p.x, p.y, p.z, ix, iy, iz);
    const int gbase = b * g.ncell;
    const float r2 = a.radius * a.radius;
    int cnt = 0;
    int64_t w = FILL ? (int64_t)__ldg(a.rowptr + i) : 0;
    for (int dx = -1; dx <= 1; ++dx) {
        const int cx = ix + dx;
        if (cx < 0 || cx >= g.nx) continue;
        for (int dy = -1; dy <= 1; ++dy) {
            const int cy = iy + dy;
            if (cy < 0 || cy >= g.ny) continue;
            // the three z-neighbours are consecutive keys: one contiguous range of the sorted order
            const int z0 = max(iz - 1, 0), z1 = min(iz + 1, g.nz - 1);
            const int key0 = gbase + (cx * g.ny + cy) * g.nz + z0;
            const int s = __ldg(a.cell_cnt + key0), e = __ldg(a.cell_cnt + key0 + (z1 - z0) + 1);
            for (int q = s; q < e; ++q) {
                const int j = __ldg(a.order + q);
                if (j == i && !a.loop) continue;
                const float4 pj = ldg4(a.x4 + (size_t)j * 4);
                const float ddx = p.x - pj.x, ddy = p.y - pj.y, ddz = p.z - pj.z;
                const float d2 = edge_len2(ddx, ddy, ddz);
                if (d2 < r2) {
                    if (FILL) {
                        if (w < a.capacity) {
                            a.row[w] = i;
                            a.col[w] = j;
                            if (a.edge_attr) {
                                const float dd = sqrtf(d2);
                                for (int c = 0; c < a.A; ++c) a.edge_attr[w * a.A + c] = dd;
                            }
                        }
                        ++w;
                    } else {
                        ++cnt;
                    }
                }
            }
        }
    }
    if (!FILL) a.deg[i] = cnt;
}

__global__ void rcsr_info_kernel(const RcsrArgs a) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const int e = a.rowptr[a.N];
        a.info[0] = e;
        a.info[1] = (int64_t)e > a.capacity ? 1 : 0;
    }
}

static size_t al256(size_t x) { return (x + 255) / 256 * 256; }
static int bits_for(int64_t n) {
    int b = 1;
    while (b < 31 && ((int64_t)1 << b) < n) ++b;
    return b;
}

struct RcsrLayout {
    size_t bounds, grid, x4, batch32, keys, ids, skeys, order, cell_cnt, deg, tmp, tmp_bytes, total;
};
static int rcsr_layout(int64_t N, int64_t table_cells, RcsrLayout& L) {
    size_t sort_b = 0, scan1 = 0, scan2 = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr,
                                        (int32_t*)nullptr, (int)N, 0, bits_for(table_cells + 1)) != cudaSuccess)
        return DISTEGNN_ECUDA;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan1, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(table_cells + 1)) !=
        cudaSuccess)
        return DISTEGNN_ECUDA;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan2, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(N + 1)) != cudaSuccess)
        return DISTEGNN_ECUDA;
    size_t o = 0;
    auto put = [&](size_t& field, size_t bytes) { field = o; o += al256(bytes); };
    put(L.bounds, 6 * 4);
    put(L.grid, sizeof(GridDev));
    put(L.x4, (size_t)N * 16);
    put(L.batch32, (size_t)N * 4);
    put(L.keys, (size_t)N * 4);
    put(L.ids, (size_t)N * 4);
    put(L.skeys, (size_t)N * 4);
    put(L.order, (size_t)N * 4);
    put(L.cell_cnt, (size_t)(table_cells + 1) * 4);
    put(L.deg, (size_t)(N + 1) * 4);
    L.tmp_bytes = sort_b > scan1 ? sort_b : scan1;
    if (scan2 > L.tmp_bytes) L.tmp_bytes = scan2;
    put(L.tmp, L.tmp_bytes);
    L.total = o + 256;
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" int distegnn_radius_csr_workspace_bytes(int64_t n_nodes, int64_t table_cells, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX - 1, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(table_cells >= 27 && table_cells < ((int64_t)1 << 30), "table_cells outside [27, 2^30)");
    RcsrLayout L;
    if (int rc = rcsr_layout(n_nodes, table_cells, L)) {
        set_error("cub temp-size query failed");
        return rc;
    }
    *bytes_host = (int64_t)L.total;
    return DISTEGNN_OK;
}

extern "C" int distegnn_radius_graph_csr(int64_t n_nodes, int n_graphs, const float* pos, const int64_t* data_batch,
                                         float radius, int loop, int edge_attr_nf, int64_t capacity, int64_t table_cells,
                                         int32_t* rowptr, int32_t* row, int32_t* col, float* edge_attr, int32_t* info,
                                         void* workspace, int64_t workspace_bytes, void* stream_) {
    using namespace degnn;
    cudaStream_t stream = (cudaStream_t)stream_;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(pos && rowptr && info && workspace, "null pointer");
    DEGNN_CHECK_ARG(capacity >= 0 && capacity < INT32_MAX && (capacity == 0 || (row && col)), "bad capacity / null edge buffers");
    DEGNN_CHECK_ARG(radius > 0.f && edge_attr_nf >= 0 && edge_attr_nf <= DISTEGNN_MAX_EDGE_ATTR, "bad radius / edge_attr_nf");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    DEGNN_CHECK_ARG((int64_t)n_graphs + 1 <= table_cells, "table_cells must hold one cell per graph plus one");
    int64_t need = 0;
    if (int rc = distegnn_radius_csr_workspace_bytes(n_nodes, table_cells, &need)) return rc;
    if (workspace_bytes < need) {
        set_error("distegnn_radius_graph_csr: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    RcsrLayout L;
    rcsr_layout(n_nodes, table_cells, L);
    char* ws = (char*)(((uintptr_t)workspace + 255) / 256 * 256);
    RcsrArgs a;
    a.N = n_nodes; a.capacity = capacity; a.table_cells = table_cells; a.B = n_graphs; a.A = edge_attr_nf; a.loop = loop;
    a.radius = radius; a.pos = pos; a.batch64 = data_batch;
    a.bounds = (int*)(ws + L.bounds); a.grid = (GridDev*)(ws + L.grid); a.x4 = (float*)(ws + L.x4);
    a.batch32 = (int32_t*)(ws + L.batch32); a.keys = (int32_t*)(ws + L.keys); a.ids = (int32_t*)(ws + L.ids);
    a.skeys = (int32_t*)(ws + L.skeys); a.order = (int32_t*)(ws + L.order); a.cell_cnt = (int32_t*)(ws + L.cell_cnt);
    a.deg = (int32_t*)(ws + L.deg);
    a.rowptr = rowptr; a.row = row; a.col = col; a.edge_attr = edge_attr_nf > 0 ? edge_attr : nullptr; a.info = info;
    void* tmp = ws + L.tmp;
    size_t tmp_bytes = L.tmp_bytes;
    const unsigned nb = (unsigned)((n_nodes + 255) / 256);
    rcsr_init_kernel<<<(unsigned)((table_cells + 1 + 255) / 256), 256, 0, stream>>>(a);
    rcsr_bounds_kernel<<<nb < 1184u ? nb : 1184u, 256, 0, stream>>>(a);
    rcsr_grid_kernel<<<1, 32, 0, stream>>>(a);
    rcsr_keys_kernel<<<nb, 256, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, (const int32_t*)a.cell_cnt, a.cell_cnt,
                                                  (int)(table_cells + 1), stream);
    if (e == cudaSuccess)
        e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, (const int32_t*)a.keys, a.skeys, (const int32_t*)a.ids, a.order,
                                            (int)n_nodes, 0, bits_for(table_cells + 1), stream);
    if (e != cudaSuccess) {
        set_error("distegnn_radius_graph_csr: cub scan/sort failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    rcsr_scan_kernel<false><<<nb, 256, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, (const int32_t*)a.deg, a.rowptr, (int)(n_nodes + 1), stream);
    if (e != cudaSuccess) {
        set_error("distegnn_radius_graph_csr: cub scan failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    if (capacity > 0) rcsr_scan_kernel<true><<<nb, 256, 0, stream>>>(a);
    rcsr_info_kernel<<<1, 32, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
