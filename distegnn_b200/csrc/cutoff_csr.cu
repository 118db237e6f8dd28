// Edge cutoff on the device (FastEGNN's `cutoff_edges` mode): keep the shortest edges of every graph of a CSR graph.
//
// The reference rule (datasets/process_dataset.py:300-305, once per sample) sorts a graph's edges by length and keeps the
// first int(E * (1 - cutoff_rate)).  Here, for every graph b of the batch (graphs are contiguous in data_batch, so their
// candidate edges form one contiguous CSR range [es_b, ee_b)):
//   k_b   = floor((double)E_b * (1.0 - rate))                      fp64, = Python's int(E * (1 - cutoff_rate))
//   kept  = the k_b smallest candidates by (length bits, CSR position): a stable selection over candidate order
//   out   = the kept candidates as a sub-sequence of the input CSR (row order and within-row order kept), edge_attr = the
//           length in every column, rowptr_out[i] = kept candidates before rowptr_in[i]
// A segmented radix select, not a sort:
//   1. per-graph node starts (from the sorted batch) and candidate ranges, k_b, kept offsets (exclusive scan of k_b)
//   2. key pass: key[e] = bits of the fp32 length (the fill pass's arithmetic; NaN -> 0xffffffff, so it sorts last)
//   3. four 8-bit digit passes: a histogram of the current digit over the keys that still match the graph's prefix
//      (shared memory when a block's edges lie in one graph, global [B,256] atomics otherwise), then one warp per graph
//      picks the bucket holding rank k_b - 1.  Result: threshold T_b and need_b = keys equal to T_b to keep
//   4. one exclusive scan of packed (key < T_b, key == T_b) flags: an edge's output position and its tie rank at once
//   5. compaction of row / col / edge_attr and the output rowptr
// Integer counts only: the output is bitwise deterministic.
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace degnn {

constexpr int CUT_TILE = 4096;      // edges per block in the histogram pass
constexpr uint32_t NAN_KEY = 0xffffffffu;

struct CutArgs {
    int64_t N, capacity;
    int B, A;
    double keep_frac;               // 1.0 - rate, in fp64
    const float* pos;               // [N,3]
    const int64_t* batch64;         // [N] or null
    const int32_t* rowptr_in;       // [N+1]
    const int32_t* row_in;          // [capacity]
    const int32_t* col_in;          // [capacity]
    const int32_t* n_edges_in;      // [1] or null (then rowptr_in[N])
    const int32_t* overflow_in;     // [1] or null
    int32_t* rowptr_out;            // [N+1]
    int32_t* row_out;               // [capacity]
    int32_t* col_out;               // [capacity]
    float* edge_attr_out;           // [capacity, A] or null
    int32_t* info;                  // [4]
    // workspace
    int32_t* gstart;                // [B+1] first node of every graph
    int32_t* estart;                // [B+1] first candidate edge of every graph (clamped to the valid candidates)
    int32_t* kcount;                // [B+1] k_b, then (in place) the exclusive scan: first output edge of every graph
    int32_t* kb;                    // [B] k_b
    uint32_t* thr;                  // [B] prefix during the select, then the threshold T_b
    int32_t* rem;                   // [B] rank still to find among the keys matching the prefix; -1 once decided
    int32_t* need;                  // [B] keys equal to T_b to keep
    uint32_t* hist;                 // [B,256]
    uint32_t* keys;                 // [capacity]
    unsigned long long* flags;      // [capacity] (less << 32 | equal), then its exclusive scan
};

// candidates: edges below the device count, never past the capacity
__device__ __forceinline__ int64_t cut_valid(const CutArgs& a) {
    const int64_t nc = a.n_edges_in ? (int64_t)__ldg(a.n_edges_in) : (int64_t)__ldg(a.rowptr_in + a.N);
    return max((int64_t)0, min(nc, a.capacity));
}

// the graph holding candidate edge e (estart is non-decreasing; the graph found is non-empty)
__device__ __forceinline__ int graph_of_edge(const int32_t* estart, int lo, int hi, int64_t e) {
    while (lo < hi) {               // last b in [lo, hi] with estart[b] <= e
        const int mid = (lo + hi + 1) >> 1;
        if ((int64_t)__ldg(estart + mid) <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) cut_graph_starts_kernel(const CutArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= a.N; i += (int64_t)gridDim.x * blockDim.x) {
        const int prev = i == 0 ? -1 : graph_id(a.batch64, i - 1, a.B);
        const int cur = i == a.N ? a.B : graph_id(a.batch64, i, a.B);
        for (int b = prev + 1; b <= cur; ++b) a.gstart[b] = (int32_t)i;
    }
}

__global__ void __launch_bounds__(256) cut_ranges_kernel(const CutArgs a) {
    const int64_t valid = cut_valid(a);
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)a.B * 256;
         t += (int64_t)gridDim.x * blockDim.x)
        a.hist[t] = 0u;
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b <= a.B; b += gridDim.x * blockDim.x) {
        const int64_t s = min((int64_t)__ldg(a.rowptr_in + __ldg(a.gstart + b)), valid);
        a.estart[b] = (int32_t)s;
        if (b == a.B) {
            a.kcount[b] = 0;
            continue;
        }
        const int64_t e = min((int64_t)__ldg(a.rowptr_in + __ldg(a.gstart + b + 1)), valid);
        const int64_t E = e - s;
        int64_t k = (int64_t)((double)E * a.keep_frac);    // fp64, truncation = floor (non-negative)
        k = max((int64_t)0, min(k, E));
        a.kcount[b] = (int32_t)k;
        a.kb[b] = (int32_t)k;
        if (k == 0) {                                       // keep none
            a.thr[b] = 0u; a.need[b] = 0; a.rem[b] = -1;
        } else if (k == E) {                                // keep all
            a.thr[b] = NAN_KEY; a.need[b] = (int32_t)E; a.rem[b] = -1;
        } else {
            a.thr[b] = 0u; a.need[b] = 0; a.rem[b] = (int32_t)(k - 1);
        }
    }
}

__global__ void __launch_bounds__(256) cut_keys_kernel(const CutArgs a) {
    const int64_t valid = cut_valid(a);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < valid; e += (int64_t)gridDim.x * blockDim.x) {
        const int i = __ldg(a.row_in + e), j = __ldg(a.col_in + e);
        float ddx, ddy, ddz;
        edge_delta(a.pos, i, j, ddx, ddy, ddz);
        const float dd = sqrtf(edge_len2(ddx, ddy, ddz));
        a.keys[e] = isnan(dd) ? NAN_KEY : __float_as_uint(dd);     // dd >= 0: the bits order as the values
    }
}

__device__ __forceinline__ bool prefix_match(uint32_t key, uint32_t prefix, int pass) {
    if (pass == 0) return true;
    const uint32_t mask = 0xffffffffu << (32 - 8 * pass);
    return (key & mask) == (prefix & mask);
}

__global__ void __launch_bounds__(256) cut_hist_kernel(const CutArgs a, int pass) {
    __shared__ uint32_t sh[256];
    const int64_t valid = cut_valid(a);
    const int64_t t0 = (int64_t)blockIdx.x * CUT_TILE;
    if (t0 >= valid) return;
    const int64_t t1 = min(t0 + CUT_TILE, valid);
    const int shift = 24 - 8 * pass;
    const int g0 = graph_of_edge(a.estart, 0, a.B - 1, t0);
    const int g1 = graph_of_edge(a.estart, g0, a.B - 1, t1 - 1);
    if (g0 == g1) {                                    // the whole tile in one graph: privatised histogram
        if (__ldg(a.rem + g0) < 0) return;
        const uint32_t prefix = __ldg(a.thr + g0);
        sh[threadIdx.x] = 0u;
        __syncthreads();
        for (int64_t e = t0 + threadIdx.x; e < t1; e += blockDim.x) {
            const uint32_t k = __ldg(a.keys + e);
            if (prefix_match(k, prefix, pass)) atomicAdd(sh + ((k >> shift) & 255u), 1u);
        }
        __syncthreads();
        const uint32_t c = sh[threadIdx.x];
        if (c) atomicAdd(a.hist + (int64_t)g0 * 256 + threadIdx.x, c);
        return;
    }
    for (int64_t e = t0 + threadIdx.x; e < t1; e += blockDim.x) {
        const int g = graph_of_edge(a.estart, g0, g1, e);
        if (__ldg(a.rem + g) < 0) continue;
        const uint32_t k = __ldg(a.keys + e);
        if (prefix_match(k, __ldg(a.thr + g), pass)) atomicAdd(a.hist + (int64_t)g * 256 + ((k >> shift) & 255u), 1u);
    }
}

// one warp per graph: the bucket of rank rem among this pass's histogram; the histogram row is zeroed for the next pass
__global__ void __launch_bounds__(256) cut_select_kernel(const CutArgs a, int pass) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= a.B) return;
    const int b = (int)warp;
    uint32_t* h = a.hist + (int64_t)b * 256;
    uint32_t c[8];
    uint32_t s = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        c[q] = h[lane * 8 + q];
        h[lane * 8 + q] = 0u;
        s += c[q];
    }
    const int r = a.rem[b];
    if (r < 0) return;
    uint32_t incl = s;                                 // inclusive warp scan of the lane sums
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += v;
    }
    const uint32_t excl = incl - s;
    const bool mine = (uint32_t)r >= excl && (uint32_t)r < incl;
    if (!mine) return;                                 // exactly one lane holds rank r
    uint32_t cum = excl;
    int bin = lane * 8;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        if ((uint32_t)r < cum + c[q]) { bin = lane * 8 + q; break; }
        cum += c[q];
    }
    const int shift = 24 - 8 * pass;
    const uint32_t prefix = a.thr[b] | ((uint32_t)bin << shift);
    const int left = r - (int)cum;
    a.thr[b] = prefix;
    if (pass == 3) {
        a.need[b] = left + 1;
        a.rem[b] = -1;
    } else {
        a.rem[b] = left;
    }
}

__global__ void __launch_bounds__(256) cut_flags_kernel(const CutArgs a) {
    const int64_t valid = cut_valid(a);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < a.capacity; e += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long f = 0ull;
        if (e < valid) {
            const int g = graph_of_edge(a.estart, 0, a.B - 1, e);
            const uint32_t k = __ldg(a.keys + e), t = __ldg(a.thr + g);
            f = k < t ? (1ull << 32) : (k == t ? 1ull : 0ull);
        }
        a.flags[e] = f;
    }
}

// kept edges before CSR position p of graph g (p in [estart[g], estart[g+1]])
__device__ __forceinline__ int64_t kept_before(const CutArgs& a, int g, int64_t p) {
    const int64_t s = __ldg(a.estart + g), e = __ldg(a.estart + g + 1);
    const int64_t base = __ldg(a.kcount + g);
    if (p >= e) return base + __ldg(a.kb + g);
    const unsigned long long fs = a.flags[s], fp = a.flags[p];
    const int64_t less = (int64_t)((fp >> 32) - (fs >> 32));
    const int64_t eq = (int64_t)((fp & 0xffffffffull) - (fs & 0xffffffffull));
    return base + less + min(eq, (int64_t)__ldg(a.need + g));
}

__global__ void __launch_bounds__(256) cut_compact_kernel(const CutArgs a) {
    const int64_t valid = cut_valid(a);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < valid; e += (int64_t)gridDim.x * blockDim.x) {
        const int g = graph_of_edge(a.estart, 0, a.B - 1, e);
        const uint32_t k = __ldg(a.keys + e), t = __ldg(a.thr + g);
        if (k > t) continue;
        const int64_t s = __ldg(a.estart + g);
        const unsigned long long fs = a.flags[s], fe = a.flags[e];
        const int64_t eq = (int64_t)((fe & 0xffffffffull) - (fs & 0xffffffffull));
        const int64_t nd = __ldg(a.need + g);
        if (k == t && eq >= nd) continue;
        const int64_t less = (int64_t)((fe >> 32) - (fs >> 32));
        const int64_t w = __ldg(a.kcount + g) + less + min(eq, nd);
        a.row_out[w] = __ldg(a.row_in + e);
        a.col_out[w] = __ldg(a.col_in + e);
        if (a.edge_attr_out) {
            const float dd = k == NAN_KEY ? __uint_as_float(0x7fc00000u) : __uint_as_float(k);
            for (int c = 0; c < a.A; ++c) a.edge_attr_out[w * a.A + c] = dd;
        }
    }
}

__global__ void __launch_bounds__(256) cut_rowptr_kernel(const CutArgs a) {
    const int64_t valid = cut_valid(a);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= a.N; i += (int64_t)gridDim.x * blockDim.x) {
        if (i == a.N) {
            a.rowptr_out[i] = __ldg(a.kcount + a.B);
            const int64_t nc = a.n_edges_in ? (int64_t)__ldg(a.n_edges_in) : (int64_t)__ldg(a.rowptr_in + a.N);
            a.info[0] = __ldg(a.kcount + a.B);
            a.info[1] = (nc > a.capacity || (a.overflow_in && __ldg(a.overflow_in) != 0)) ? 1 : 0;
            a.info[2] = (int32_t)nc;
            a.info[3] = 0;
            continue;
        }
        const int g = graph_id(a.batch64, i, a.B);
        const int64_t s = __ldg(a.estart + g), e = __ldg(a.estart + g + 1);
        const int64_t p = min(max(min((int64_t)__ldg(a.rowptr_in + i), valid), s), e);
        a.rowptr_out[i] = (int32_t)kept_before(a, g, p);
    }
}

struct CutLayout {
    size_t gstart, estart, kcount, kb, thr, rem, need, hist, keys, flags, tmp, tmp_bytes, total;
};
static int cut_layout(int64_t N, int B, int64_t capacity, CutLayout& L) {
    size_t scan1 = 0, scan2 = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan1, (int32_t*)nullptr, (int32_t*)nullptr, B + 1) != cudaSuccess)
        return DISTEGNN_ECUDA;
    if (capacity > 0 && cub::DeviceScan::ExclusiveSum(nullptr, scan2, (unsigned long long*)nullptr,
                                                      (unsigned long long*)nullptr, (int)capacity) != cudaSuccess)
        return DISTEGNN_ECUDA;
    WorkspaceCursor ws;
    L.gstart = ws.take((size_t)(B + 1) * 4);
    L.estart = ws.take((size_t)(B + 1) * 4);
    L.kcount = ws.take((size_t)(B + 1) * 4);
    L.kb = ws.take((size_t)B * 4);
    L.thr = ws.take((size_t)B * 4);
    L.rem = ws.take((size_t)B * 4);
    L.need = ws.take((size_t)B * 4);
    L.hist = ws.take((size_t)B * 256 * 4);
    L.keys = ws.take((size_t)capacity * 4);
    L.flags = ws.take((size_t)capacity * 8);
    L.tmp_bytes = scan1 > scan2 ? scan1 : scan2;
    L.tmp = ws.take(L.tmp_bytes);
    L.total = ws.end + 256;              // the caller's pointer is aligned up
    (void)N;
    return DISTEGNN_OK;
}

static unsigned cut_grid(int64_t n) {
    const int64_t cap = 8 * (int64_t)sm_count();
    const int64_t g = (n + 255) / 256;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace degnn

extern "C" int distegnn_cutoff_csr_workspace_bytes(int64_t n_nodes, int n_graphs, int64_t capacity, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_nodes < INT32_MAX - 1, "n_nodes out of int32 range");
    DEGNN_CHECK_ARG(n_graphs > 0 && n_graphs < (1 << 24), "n_graphs outside [1, 2^24)");
    DEGNN_CHECK_ARG(capacity >= 0 && capacity < INT32_MAX, "capacity out of int32 range");
    CutLayout L;
    if (int rc = cut_layout(n_nodes, n_graphs, capacity, L)) {
        set_error("cub temp-size query failed");
        return rc;
    }
    *bytes_host = (int64_t)L.total;
    return DISTEGNN_OK;
}

extern "C" int distegnn_cutoff_csr(int64_t n_nodes, int n_graphs, const float* pos, const int64_t* data_batch,
                                   double cutoff_rate, int edge_attr_nf, const int32_t* rowptr_in, const int32_t* row_in,
                                   const int32_t* col_in, const int32_t* n_edges_in, int64_t capacity,
                                   const int32_t* overflow_in, int32_t* rowptr_out, int32_t* row_out, int32_t* col_out,
                                   float* edge_attr_out, int32_t* info, void* workspace, int64_t workspace_bytes,
                                   void* stream_) {
    using namespace degnn;
    cudaStream_t stream = (cudaStream_t)stream_;
    DEGNN_CHECK_ARG(cutoff_rate >= 0.0 && cutoff_rate <= 1.0, "cutoff_rate must lie in [0, 1] (and not be NaN)");
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(edge_attr_nf >= 0 && edge_attr_nf <= DISTEGNN_MAX_EDGE_ATTR, "bad edge_attr_nf");
    DEGNN_CHECK_ARG(pos && rowptr_in && rowptr_out && info && workspace, "null pointer");
    DEGNN_CHECK_ARG(capacity >= 0 && capacity < INT32_MAX, "capacity out of int32 range");
    DEGNN_CHECK_ARG(capacity == 0 || (row_in && col_in && row_out && col_out && (edge_attr_nf == 0 || edge_attr_out)),
                    "null pointer (edge buffers)");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    // our own buffers alone (a lower bound, known without the cub temp-size query), then the exact size
    int64_t need = (int64_t)(n_graphs + 1) * 12 + (int64_t)n_graphs * (16 + 256 * 4) + capacity * 12;
    if (workspace_bytes < need) {
        set_error("distegnn_cutoff_csr: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    if (int rc = distegnn_cutoff_csr_workspace_bytes(n_nodes, n_graphs, capacity, &need)) return rc;
    if (workspace_bytes < need) {
        set_error("distegnn_cutoff_csr: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    CutLayout L;
    cut_layout(n_nodes, n_graphs, capacity, L);
    char* ws = (char*)align256((uintptr_t)workspace);
    CutArgs a;
    a.N = n_nodes; a.capacity = capacity; a.B = n_graphs; a.A = edge_attr_nf; a.keep_frac = 1.0 - cutoff_rate;
    a.pos = pos; a.batch64 = n_graphs > 1 ? data_batch : nullptr;
    a.rowptr_in = rowptr_in; a.row_in = row_in; a.col_in = col_in; a.n_edges_in = n_edges_in; a.overflow_in = overflow_in;
    a.rowptr_out = rowptr_out; a.row_out = row_out; a.col_out = col_out;
    a.edge_attr_out = edge_attr_nf > 0 ? edge_attr_out : nullptr; a.info = info;
    a.gstart = (int32_t*)(ws + L.gstart); a.estart = (int32_t*)(ws + L.estart); a.kcount = (int32_t*)(ws + L.kcount);
    a.kb = (int32_t*)(ws + L.kb); a.thr = (uint32_t*)(ws + L.thr); a.rem = (int32_t*)(ws + L.rem);
    a.need = (int32_t*)(ws + L.need); a.hist = (uint32_t*)(ws + L.hist); a.keys = (uint32_t*)(ws + L.keys);
    a.flags = (unsigned long long*)(ws + L.flags);
    void* tmp = ws + L.tmp;
    size_t tmp_bytes = L.tmp_bytes;
    const unsigned gn = cut_grid(n_nodes + 1), gb = cut_grid((int64_t)n_graphs * 256);
    cut_graph_starts_kernel<<<gn, 256, 0, stream>>>(a);
    cut_ranges_kernel<<<gb, 256, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, a.kcount, a.kcount, n_graphs + 1, stream);
    if (e != cudaSuccess) {
        set_error("distegnn_cutoff_csr: cub scan failed: %s", cudaGetErrorString(e));
        return DISTEGNN_ECUDA;
    }
    if (capacity > 0) {
        const unsigned ge = cut_grid(capacity);
        const unsigned tiles = (unsigned)((capacity + CUT_TILE - 1) / CUT_TILE);
        const unsigned sel = (unsigned)(((int64_t)n_graphs * 32 + 255) / 256);
        cut_keys_kernel<<<ge, 256, 0, stream>>>(a);
        for (int pass = 0; pass < 4; ++pass) {
            cut_hist_kernel<<<tiles, 256, 0, stream>>>(a, pass);
            cut_select_kernel<<<sel, 256, 0, stream>>>(a, pass);
        }
        cut_flags_kernel<<<ge, 256, 0, stream>>>(a);
        DEGNN_CHECK_LAUNCH();
        e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, a.flags, a.flags, (int)capacity, stream);
        if (e != cudaSuccess) {
            set_error("distegnn_cutoff_csr: cub scan failed: %s", cudaGetErrorString(e));
            return DISTEGNN_ECUDA;
        }
        cut_compact_kernel<<<ge, 256, 0, stream>>>(a);
    }
    cut_rowptr_kernel<<<gn, 256, 0, stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
