// The METIS node partitioner (datasets/distribute_graphs.py:54-87, 151-185; DESIGN §10):
//   distegnn_csr_sorted_i64   the device half: an id-order CSR of radius_graph_csr (each row in cell-scan order) to the
//                             int64 CSR METIS takes, every row's neighbours ascending — index2ptr(sort_edge_index(ei));
//   distegnn_metis_recursive  the host half: METIS_PartGraphRecursive of the toolkit's METIS 5 (64-bit idx_t) with the
//                             reference's arguments, after the input is validated here.
#include <mutex>

#include "common.cuh"

// METIS 5 with 64-bit idx_t, as libmetis_static.a of the CUDA toolkit is built (no metis.h ships with it).
typedef int64_t metis_idx_t;
extern "C" int METIS_PartGraphRecursive(metis_idx_t* nvtxs, metis_idx_t* ncon, metis_idx_t* xadj, metis_idx_t* adjncy,
                                        metis_idx_t* vwgt, metis_idx_t* vsize, metis_idx_t* adjwgt, metis_idx_t* nparts,
                                        float* tpwgts, float* ubvec, metis_idx_t* options, metis_idx_t* edgecut,
                                        metis_idx_t* part);
static constexpr int METIS_OK_ = 1;

namespace degnn {

constexpr int SORT_WARPS = 8;           // rows per block, one warp each
constexpr int SORT_SMEM_ROW = 1024;     // a row up to this long is ranked from shared memory, a longer one from global

// One warp per row i of [0, N]: xadj[i] = min(rowptr[i], count) in int64, and the row's neighbours ascending in adjncy.
// Rows of at most 32 entries: a bitonic sort across the lanes.  Longer rows: every entry's rank is the number of entries
// below it (ties by position, so any input sorts stably), computed from a shared-memory copy of the row up to
// SORT_SMEM_ROW entries and from global memory past that.  `count` = min(*n_edges_dev, capacity), so nothing at or past
// the valid edges is read.
__global__ void __launch_bounds__(SORT_WARPS * 32) csr_sorted_i64_kernel(int64_t N, int64_t capacity,
                                                                          const int32_t* __restrict__ rowptr,
                                                                          const int32_t* __restrict__ col,
                                                                          const int32_t* n_edges_dev, int64_t* xadj,
                                                                          int64_t* adjncy) {
    __shared__ int32_t buf[SORT_WARPS][SORT_SMEM_ROW];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * SORT_WARPS + w;
    if (i > N) return;
    int64_t count = n_edges_dev ? (int64_t)__ldg(n_edges_dev) : (int64_t)__ldg(rowptr + N);
    count = max((int64_t)0, min(count, capacity));
    const int64_t b = min((int64_t)__ldg(rowptr + i), count);
    if (lane == 0) xadj[i] = b;
    if (i == N) return;
    const int64_t e = max(b, min((int64_t)__ldg(rowptr + i + 1), count));
    const int d = (int)(e - b);
    const int32_t* src = col + b;
    int64_t* dst = adjncy + b;
    if (d <= 32) {
        int v = lane < d ? __ldg(src + lane) : INT_MAX;
        for (int k = 2; k <= 32; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                const int o = __shfl_xor_sync(0xffffffffu, v, j);
                const bool up = (lane & k) == 0, low = (lane & j) == 0;
                v = (low == up) ? min(v, o) : max(v, o);
            }
        if (lane < d) dst[lane] = v;
        return;
    }
    if (d <= SORT_SMEM_ROW) {
        for (int k = lane; k < d; k += 32) buf[w][k] = __ldg(src + k);
        __syncwarp();
        src = buf[w];
    }
    for (int k = lane; k < d; k += 32) {
        const int v = src[k];
        int rank = 0;
        for (int m = 0; m < d; ++m) {
            const int u = src[m];
            rank += (u < v) | ((u == v) & (m < k));
        }
        dst[rank] = v;
    }
}

}  // namespace degnn

extern "C" {

int distegnn_csr_sorted_i64(int64_t n_nodes, int64_t n_edges, const int32_t* rowptr, const int32_t* col,
                            const int32_t* n_edges_dev, int64_t* xadj, int64_t* adjncy, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_edges >= 0, "negative size");
    DEGNN_CHECK_ARG(n_nodes < ((int64_t)1 << 31) - 1 && n_edges < ((int64_t)1 << 31), "size past int32 ids");
    DEGNN_CHECK_ARG(rowptr && xadj, "null pointer");
    DEGNN_CHECK_ARG(n_edges == 0 || (col && adjncy), "null edge pointer");
    const int64_t rows = n_nodes + 1;
    const unsigned blocks = (unsigned)((rows + SORT_WARPS - 1) / SORT_WARPS);
    csr_sorted_i64_kernel<<<blocks, SORT_WARPS * 32, 0, (cudaStream_t)stream>>>(n_nodes, n_edges, rowptr, col,
                                                                                 n_edges_dev, xadj, adjncy);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int distegnn_metis_recursive(int64_t n_nodes, const int64_t* xadj_host, const int64_t* adjncy_host, int64_t n_parts,
                             int64_t* part_host, int64_t* objval_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 1, "n_nodes must be >= 1");
    DEGNN_CHECK_ARG(xadj_host && part_host, "null pointer");
    if (n_parts < 1 || n_parts > n_nodes) {
        set_error("distegnn_metis_recursive: n_parts=%lld outside [1, n_nodes=%lld]", (long long)n_parts,
                  (long long)n_nodes);
        return DISTEGNN_EINVAL;
    }
    if (xadj_host[0] != 0) {
        set_error("distegnn_metis_recursive: xadj[0]=%lld, must be 0", (long long)xadj_host[0]);
        return DISTEGNN_EINVAL;
    }
    for (int64_t i = 0; i < n_nodes; ++i)
        if (xadj_host[i + 1] < xadj_host[i]) {
            set_error("distegnn_metis_recursive: xadj decreases at row %lld (%lld -> %lld)", (long long)i,
                      (long long)xadj_host[i], (long long)xadj_host[i + 1]);
            return DISTEGNN_EINVAL;
        }
    DEGNN_CHECK_ARG(xadj_host[n_nodes] == 0 || adjncy_host, "null adjncy with edges");
    for (int64_t i = 0; i < n_nodes; ++i)
        for (int64_t k = xadj_host[i]; k < xadj_host[i + 1]; ++k) {
            const int64_t j = adjncy_host[k];
            if (j < 0 || j >= n_nodes || j == i) {
                set_error("distegnn_metis_recursive: row %lld has neighbour %lld (%s)", (long long)i, (long long)j,
                          j == i ? "a self loop" : "outside [0, n_nodes)");
                return DISTEGNN_EINVAL;
            }
        }
    int64_t cut = 0;
    if (n_parts == 1) {                        // the reference returns zeros here without calling METIS (its 1s)
        for (int64_t i = 0; i < n_nodes; ++i) part_host[i] = 0;
    } else {
        // GKlib keeps its RNG and its error state in globals: one call at a time.
        static std::mutex mu;
        std::lock_guard<std::mutex> lock(mu);
        metis_idx_t nv = n_nodes, ncon = 1, np = n_parts;
        const int rc = METIS_PartGraphRecursive(&nv, &ncon, const_cast<metis_idx_t*>(xadj_host),
                                                const_cast<metis_idx_t*>(adjncy_host), nullptr, nullptr, nullptr, &np,
                                                nullptr, nullptr, nullptr, &cut, part_host);
        if (rc != METIS_OK_) {
            set_error("distegnn_metis_recursive: METIS_PartGraphRecursive returned %d", rc);
            return DISTEGNN_EINVAL;
        }
    }
    if (objval_host) *objval_host = cut;
    return DISTEGNN_OK;
}

}  // extern "C"
