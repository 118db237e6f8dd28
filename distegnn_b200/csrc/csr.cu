// Graph preprocessing: int64 COO (edge_index [2,E]) -> int32 CSR sorted (stably) by destination row.
// Replaces the implicit scatter-by-edge_index[0] of unsorted_segment_sum/mean
// (reference models/FastEGNN.py:322-337).  Cached per edge_index by the Python side, so it is off the
// per-step path; the sort itself is cub's radix sort (library plumbing, not a hot kernel).
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace degnn {

// Ids outside [0,N) are counted into *n_invalid (the reference fails with a device-side index assert on such input) and
// clamped, so nothing downstream can index out of bounds before the host has looked at the counter.
__global__ void csr_keys_kernel(const int64_t* __restrict__ edge_index, int64_t E, int64_t N, int32_t* keys,
                                int32_t* vals, int32_t* n_invalid) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) {
        const int64_t r = edge_index[e], c = edge_index[E + e];   // row = edge_index[0, e], col = edge_index[1, e]
        const bool bad = r < 0 || r >= N || c < 0 || c >= N;
        if (bad && n_invalid) atomicAdd(n_invalid, 1);
        keys[e] = (int32_t)(r < 0 ? 0 : (r >= N ? N - 1 : r));
        vals[e] = (int32_t)e;
    }
}

// After the sort: col[e'] = edge_index[1, perm[e']]; rowptr from run boundaries of the sorted rows
// (rows without edges get an empty range).
__global__ void csr_finish_kernel(const int64_t* __restrict__ edge_index, int64_t E, int64_t N,
                                  const int32_t* __restrict__ row, const int32_t* __restrict__ perm,
                                  int32_t* __restrict__ col, int32_t* __restrict__ rowptr) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) {
        const int64_t c = edge_index[E + perm[e]];
        col[e] = (int32_t)(c < 0 ? 0 : (c >= N ? N - 1 : c));
        int32_t r = row[e];
        int32_t prev = (e == 0) ? -1 : row[e - 1];
        for (int32_t k = prev + 1; k <= r; ++k) rowptr[k] = (int32_t)e;
        if (e == E - 1)
            for (int64_t k = (int64_t)r + 1; k <= N; ++k) rowptr[k] = (int32_t)E;
    }
}

__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
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

static int key_bits(int64_t n_nodes) {
    int b = 1;
    while (b < 31 && ((int64_t)1 << b) < n_nodes) ++b;
    return b;
}

static size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

static cudaError_t sort_temp_bytes(int64_t N, int64_t E, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const int32_t*)nullptr, (int32_t*)nullptr,
                                           (const int32_t*)nullptr, (int32_t*)nullptr, (int)E, 0,
                                           key_bits(N));
}

}  // namespace degnn

extern "C" {

int distegnn_csr_workspace_bytes(int64_t n_nodes, int64_t n_edges, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(n_edges >= 0 && n_edges < INT32_MAX, "n_edges out of int32 range");
    size_t tmp = 0;
    if (n_edges > 0) {
        cudaError_t e = sort_temp_bytes(n_nodes, n_edges, &tmp);
        if (e != cudaSuccess) {
            set_error("cub temp-size query failed: %s", cudaGetErrorString(e));
            return DISTEGNN_ECUDA;
        }
    }
    *bytes_host = (int64_t)(2 * align_up((size_t)n_edges * 4) + align_up(tmp) + 256);
    return DISTEGNN_OK;
}

int distegnn_build_csr(const int64_t* edge_index, int64_t n_nodes, int64_t n_edges, int32_t* rowptr,
                       int32_t* row, int32_t* col, int32_t* perm, void* workspace,
                       int64_t workspace_bytes, int32_t* n_invalid, void* stream_) {
    using namespace degnn;
    cudaStream_t stream = (cudaStream_t)stream_;
    DEGNN_CHECK_ARG(rowptr, "null rowptr");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(n_edges >= 0 && n_edges < INT32_MAX, "n_edges out of int32 range");
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
        set_error("distegnn_build_csr: workspace %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    char* ws = (char*)(((uintptr_t)workspace + 255) / 256 * 256);
    int32_t* keys = (int32_t*)ws;
    int32_t* vals = (int32_t*)(ws + align_up((size_t)n_edges * 4));
    void* tmp = ws + 2 * align_up((size_t)n_edges * 4);
    size_t tmp_bytes = 0;
    sort_temp_bytes(n_nodes, n_edges, &tmp_bytes);

    unsigned blocks = (unsigned)((n_edges + 255) / 256);
    csr_keys_kernel<<<blocks, 256, 0, stream>>>(edge_index, n_edges, n_nodes, keys, vals, n_invalid);
    DEGNN_CHECK_LAUNCH();
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, (const int32_t*)keys, row,
                                                    (const int32_t*)vals, perm, (int)n_edges, 0,
                                                    key_bits(n_nodes), stream);
    if (e != cudaSuccess) {
        set_error("distegnn_build_csr: radix sort failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    csr_finish_kernel<<<blocks, 256, 0, stream>>>(edge_index, n_edges, n_nodes, row, perm, col, rowptr);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
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
