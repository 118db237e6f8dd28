// Deterministic mode (det.cuh, DESIGN §17): workspace sizing, the two combine passes, and the fixed-order rollout centroid;
// with the centroid's reduction, the rollout's per-step error against recorded targets (DESIGN §19), fixed-order always.
// Each output element of these kernels is computed by one thread in an order fixed by the input sizes, so their grids do
// not enter the result.
#include "common.cuh"
#include "det.cuh"

namespace degnn {

int det_check_workspace(int64_t n_nodes, int64_t n_edges, int C, const void* ws, int64_t ws_bytes, const char* who) {
    DEGNN_CHECK_ARG(ws, "null deterministic workspace");
    DEGNN_CHECK_ARG(((uintptr_t)ws & 15) == 0, "deterministic workspace not 16-byte aligned");
    const int64_t need = det_vsum_bytes(n_nodes, C) + (n_edges >= 0 ? det_edge_bytes(n_edges) : 0);
    if (ws_bytes < need) {
        set_error("%s: workspace %lld < %lld bytes", who, (long long)ws_bytes, (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    return DISTEGNN_OK;
}

template <typename I>
__device__ int64_t lower_bound_dev(const I* v, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)__ldg(v + mid) < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// One warp per 16-edge slice; the slice that holds a row's first edge and whose last run goes on into the next slice adds
// the slots of the row's later slices to the row, in slice order.  Lane l: agg_m columns 2l, 2l+1; lanes 0..2: agg_x.
__global__ void __launch_bounds__(256) edge_combine_det_kernel(int64_t E, const int32_t* E_dev, const int32_t* row,
                                                               const float* slots, float* agg_m, float* agg_x) {
    const int lane = threadIdx.x & 31;
    const int64_t nE = E_dev ? min((int64_t)__ldg(E_dev), E) : E;
    const int64_t n_slices = (nE + 15) / 16;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < n_slices; s += warps) {
        const int r = __ldg(row + min(16 * s + 15, nE - 1));
        if (16 * (s + 1) >= nE || __ldg(row + 16 * (s + 1)) != r) continue;     // the slice's last run ends in it
        if (s > 0 && __ldg(row + 16 * s - 1) == r) continue;                     // the row started before the slice
        float2 m = make_float2(0.f, 0.f);
        float x = 0.f;
        if (agg_m) m = *reinterpret_cast<const float2*>(agg_m + (size_t)r * H + 2 * lane);
        if (lane < 3) x = agg_x[(size_t)r * 4 + lane];
        for (int64_t s2 = s + 1; 16 * s2 < nE && __ldg(row + 16 * s2) == r; ++s2) {
            const float* sl = slots + s2 * DET_EDGE_SLOT;
            if (agg_m) {
                m.x += sl[2 * lane];
                m.y += sl[2 * lane + 1];
            }
            if (lane < 3) x += sl[H + lane];
        }
        if (agg_m) *reinterpret_cast<float2*>(agg_m + (size_t)r * H + 2 * lane) = m;
        if (lane < 3) agg_x[(size_t)r * 4 + lane] = x;
    }
}

constexpr int DET_RED = 256;   // threads of the per-graph reductions: part of the summation order

// Σ over rows [lo, hi) of v(i) (NV components) in a fixed order: thread t takes rows lo + t, lo + t + DET_RED, ..., then a
// fixed tree over the threads.  Result in red[k][0].
template <typename T, int NV, typename F>
__device__ void det_row_sum(int64_t lo, int64_t hi, F v, T (*red)[DET_RED]) {
    const int t = threadIdx.x;
    T s[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) s[k] = T(0);
    for (int64_t i = lo + t; i < hi; i += DET_RED) v(i, s);
#pragma unroll
    for (int k = 0; k < NV; ++k) red[k][t] = s[k];
    for (int o = DET_RED / 2; o > 0; o >>= 1) {
        __syncthreads();
        if (t < o)
#pragma unroll
            for (int k = 0; k < NV; ++k) red[k][t] += red[k][t + o];
    }
    __syncthreads();
}

// One thread per vsum chunk (the real<->virtual kernel's chunks, det.cuh): Σx of the chunk's nodes in node order per graph,
// stored to vsum[g, 0:3] for a graph that starts in the chunk, else to the chunk's slot (entries 0..2 of a slot are not
// used by the real<->virtual kernel).
__global__ void __launch_bounds__(256) chunk_xsum_det_kernel(int64_t N, int C, int shift, const int32_t* batch,
                                                             const float* x4, float* slots, float* vsum) {
    const int K = 4 + 3 * C + H * C;
    const int64_t per = (int64_t)det_nodes_per_tile(C) << shift;      // nodes per chunk
    const int64_t chunks = (N + per - 1) / per;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n0 = c * per, n1 = min(N, n0 + per);
        const int cont = (n0 > 0 && __ldg(batch + n0 - 1) == __ldg(batch + n0)) ? __ldg(batch + n0) : -1;
        int cur = __ldg(batch + n0);
        float sx = 0.f, sy = 0.f, sz = 0.f;
        auto flush = [&]() {
            float* dst = cur == cont ? slots + c * K : vsum + (size_t)cur * K;
            dst[0] = sx; dst[1] = sy; dst[2] = sz;
        };
        for (int64_t i = n0; i < n1; ++i) {
            const int gr = __ldg(batch + i);
            if (gr != cur) {
                flush();
                cur = gr;
                sx = sy = sz = 0.f;
            }
            const float4 v = ldg4(x4 + i * 4);
            sx += v.x; sy += v.y; sz += v.z;
        }
        flush();
    }
}

// Block (b, part): graph b's rows [lo, hi) by binary search of the sorted batch; entries part·256 + t < n_entries of
// vsum[b] (entry 3 excepted) += the slots of chunks chunk(lo)+1 .. chunk(hi−1), in chunk order; vsum[b, 3] = hi − lo.
__global__ void __launch_bounds__(256) vsum_combine_det_kernel(int64_t N, int C, int shift, int n_entries,
                                                               const int32_t* batch, const float* slots, float* vsum) {
    const int K = 4 + 3 * C + H * C;
    const int b = blockIdx.x, i = blockIdx.y * blockDim.x + threadIdx.x;
    const int64_t lo = lower_bound_dev(batch, N, b), hi = lower_bound_dev(batch, N, (int64_t)b + 1);
    float* dst = vsum + (size_t)b * K;
    if (i == 3) dst[3] = (float)(hi - lo);
    if (i >= n_entries || i == 3 || hi == lo) return;
    const int64_t per = (int64_t)det_nodes_per_tile(C) << shift;
    const int64_t c0 = lo / per, c1 = (hi - 1) / per;
    const float* sl = slots + i;
    float acc = dst[i];
    int64_t c = c0 + 1;
    for (; c + 8 <= c1 + 1; c += 8) {           // eight independent loads in flight, added in chunk order
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __ldg(sl + (c + k) * K);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc += v[k];
    }
    for (; c <= c1; ++c) acc += __ldg(sl + c * K);
    dst[i] = acc;
}

// sums[b] += (Σx, Σy, Σz, count) over the rows of graph b, in fp64 and a fixed order (one block per graph)
__global__ void __launch_bounds__(DET_RED) centroid_det_kernel(int64_t N, int B, const float* pos, const int64_t* batch,
                                                               double* sums) {
    __shared__ double red[3][DET_RED];
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        const int64_t lo = batch ? lower_bound_dev(batch, N, b) : 0;
        const int64_t hi = batch ? lower_bound_dev(batch, N, (int64_t)b + 1) : N;
        det_row_sum<double, 3>(lo, hi, [&](int64_t i, double (&s)[3]) {
            s[0] += (double)__ldg(pos + i * 3); s[1] += (double)__ldg(pos + i * 3 + 1); s[2] += (double)__ldg(pos + i * 3 + 2);
        }, red);
        if (threadIdx.x < 3) sums[(size_t)b * 4 + threadIdx.x] += red[threadIdx.x][0];
        if (threadIdx.x == 3) sums[(size_t)b * 4 + 3] += (double)(hi - lo);
        __syncthreads();
    }
}

// The per-step error of a rollout against recorded targets (distegnn_rollout_sq_err).  Block c takes the rows [c·CH,
// (c+1)·CH) and sums Σ_d (pred − target)² (fp32 differences, fp64 squares and sums) over each graph's rows in the chunk
// with det_row_sum, the centroid's reduction.  A graph's first chunk stores its partial to sq_err[t, b], each later chunk
// to its own slot; the last block to finish adds every graph's slots in chunk order.  So the order depends on N and the
// graph sizes alone, and every value is a plain store (a rerun step overwrites its row).
constexpr int64_t SQERR_CHUNK = 2048;   // rows per block: part of the summation order

__global__ void __launch_bounds__(DET_RED) rollout_sq_err_kernel(int64_t N, int B, int steps, const float* pred,
                                                                 const float* targets, const int64_t* batch,
                                                                 const int32_t* counter, double* sq_err, double* slots,
                                                                 unsigned* ticket) {
    __shared__ double red[1][DET_RED];
    __shared__ bool last;
    const int t = __ldcg(counter);             // this step: the advance moves the counter on after this launch
    const bool keep = t >= 0 && t < steps;
    const int64_t c = blockIdx.x, r0 = c * SQERR_CHUNK, r1 = min(N, r0 + SQERR_CHUNK);
    const float* tg = targets + (keep ? (int64_t)t * N * 3 : 0);
    double* out = sq_err + (keep ? (int64_t)t * B : 0);
    for (int64_t i = r0; keep && i < r1;) {    // the graphs of the chunk, one after the other (batch sorted)
        const int64_t b = batch ? __ldg(batch + i) : 0;
        const int64_t j = batch ? i + lower_bound_dev(batch + i, r1 - i, b + 1) : r1;
        det_row_sum<double, 1>(i, j, [&](int64_t k, double (&s)[1]) {
            const float dx = __fsub_rn(__ldg(pred + k * 3), __ldg(tg + k * 3));
            const float dy = __fsub_rn(__ldg(pred + k * 3 + 1), __ldg(tg + k * 3 + 1));
            const float dz = __fsub_rn(__ldg(pred + k * 3 + 2), __ldg(tg + k * 3 + 2));
            s[0] += ((double)dx * dx + (double)dy * dy) + (double)dz * dz;
        }, red);
        if (threadIdx.x == 0 && b >= 0 && b < B) {
            const bool first = i > r0 || r0 == 0 || (batch && __ldg(batch + r0 - 1) != b);   // starts in this chunk
            if (first) out[b] = red[0][0];
            else slots[c] = red[0][0];
        }
        __syncthreads();
        i = j;
    }
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (threadIdx.x == 0) *ticket = 0;
    if (!keep) return;
    for (int b = threadIdx.x; b < B; b += DET_RED) {
        const int64_t lo = batch ? lower_bound_dev(batch, N, b) : 0;
        const int64_t hi = batch ? lower_bound_dev(batch, N, (int64_t)b + 1) : N;
        double acc = 0.0;
        if (hi > lo) {
            acc = __ldcg(out + b);
            int64_t k = lo / SQERR_CHUNK + 1;
            const int64_t k1 = (hi - 1) / SQERR_CHUNK;
            for (; k + 8 <= k1 + 1; k += 8) {  // eight independent loads in flight, added in chunk order
                double v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = __ldcg(slots + k + u);
#pragma unroll
                for (int u = 0; u < 8; ++u) acc += v[u];
            }
            for (; k <= k1; ++k) acc += __ldcg(slots + k);
        }
        out[b] = acc;
    }
}

static int64_t sq_err_chunks(int64_t N) { return (N + SQERR_CHUNK - 1) / SQERR_CHUNK; }
static int64_t sq_err_workspace(int64_t N) { return det_align(sq_err_chunks(N) * 8) + 256; }

static unsigned det_blocks(int64_t units, int64_t per_sm, int max_ctas) {
    const int64_t cap = per_sm * sm_count();
    return (unsigned)det_grid(units < 1 ? 1 : (units > cap ? cap : units), max_ctas);
}

int edge_combine_det(int64_t n_nodes, int64_t n_edges, int C, const int32_t* row, const int32_t* n_edges_dev,
                     float* agg_m, float* agg_x, void* workspace, int64_t workspace_bytes, void* stream, int max_ctas) {
    if (int rc = check_dims(0, C, 0)) return rc;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_edges >= 0, "negative size");
    if (n_edges == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(row && agg_x, "null pointer");
    if (int rc = det_check_workspace(n_nodes, n_edges, C, workspace, workspace_bytes, "distegnn_edge_combine_det"))
        return rc;
    edge_combine_det_kernel<<<det_blocks(((n_edges + 15) / 16 + 7) / 8, 4, max_ctas), 256, 0, (cudaStream_t)stream>>>(
        n_edges, n_edges_dev, row, det_edge_slots(workspace, n_nodes, C), agg_m, agg_x);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int vsum_combine_det(int64_t n_nodes, int n_graphs, int C, unsigned flags, const int32_t* batch32, const float* x4,
                     float* vsum, void* workspace, int64_t workspace_bytes, void* stream, int max_ctas) {
    if (int rc = check_dims(0, C, 0)) return rc;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(vsum && (n_nodes == 0 || (batch32 && x4)), "null pointer");
    if (int rc = det_check_workspace(n_nodes, -1, C, workspace, workspace_bytes, "distegnn_vsum_combine_det")) return rc;
    const int shift = det_chunk_shift(n_nodes, C);
    // INIT: only Σx (no real<->virtual kernel ran); LAST: that kernel wrote only the Σ ΔX·φ_X entries 4 .. 4+3C
    const int n_entries = (flags & DISTEGNN_FLAG_INIT) ? 3 : (flags & DISTEGNN_FLAG_LAST) ? 4 + 3 * C : det_K(C);
    float* slots = det_vsum_slots(workspace);
    if (n_nodes > 0) {
        chunk_xsum_det_kernel<<<det_blocks((det_chunks(n_nodes, C) + 255) / 256, 4, max_ctas), 256, 0,
                                (cudaStream_t)stream>>>(n_nodes, C, shift, batch32, x4, slots, vsum);
        DEGNN_CHECK_LAUNCH();
    }
    const dim3 grid((unsigned)n_graphs, (unsigned)((n_entries + 255) / 256));
    vsum_combine_det_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(n_nodes, C, shift, n_entries, batch32, slots, vsum);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" {

int distegnn_deterministic_workspace_bytes(int64_t n_nodes, int64_t edge_capacity, int C, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0 && edge_capacity >= 0, "negative size");
    if (int rc = check_dims(0, C, 0)) return rc;
    *bytes_host = det_vsum_bytes(n_nodes, C) + det_edge_bytes(edge_capacity);
    return DISTEGNN_OK;
}

int distegnn_edge_combine_det(int64_t n_nodes, int64_t n_edges, int C, const int32_t* row, const int32_t* n_edges_dev,
                              float* agg_m, float* agg_x, void* workspace, int64_t workspace_bytes, void* stream) {
    return degnn::edge_combine_det(n_nodes, n_edges, C, row, n_edges_dev, agg_m, agg_x, workspace, workspace_bytes,
                                   stream, 0);
}

int distegnn_vsum_combine_det(int64_t n_nodes, int n_graphs, int C, unsigned flags, const int32_t* batch32,
                              const float* x4, float* vsum, void* workspace, int64_t workspace_bytes, void* stream) {
    return degnn::vsum_combine_det(n_nodes, n_graphs, C, flags, batch32, x4, vsum, workspace, workspace_bytes, stream, 0);
}

int distegnn_rollout_centroid_det(int64_t n_nodes, int n_graphs, const float* pos, const int64_t* data_batch,
                                  double* sums, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(pos && sums, "null pointer");
    centroid_det_kernel<<<det_blocks(n_graphs, 8, 0), DET_RED, 0, (cudaStream_t)stream>>>(n_nodes, n_graphs, pos,
                                                                                       data_batch, sums);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int distegnn_rollout_sq_err_workspace_bytes(int64_t n_nodes, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0, "negative size");
    *bytes_host = sq_err_workspace(n_nodes);
    return DISTEGNN_OK;
}

int distegnn_rollout_sq_err(int64_t n_nodes, int n_graphs, int steps, const float* pred, const float* targets,
                            const int64_t* data_batch, const int32_t* counter, double* sq_err, void* workspace,
                            int64_t workspace_bytes, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0 && steps >= 1, "bad size");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    DEGNN_CHECK_ARG(counter && sq_err, "null pointer");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(pred && targets && workspace, "null pointer");
    DEGNN_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace not 16-byte aligned");
    if (workspace_bytes < sq_err_workspace(n_nodes)) {
        set_error("distegnn_rollout_sq_err: workspace %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)sq_err_workspace(n_nodes));
        return DISTEGNN_EWORKSPACE;
    }
    double* slots = reinterpret_cast<double*>(workspace);
    unsigned* ticket = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(workspace) + det_align(sq_err_chunks(n_nodes) * 8));
    rollout_sq_err_kernel<<<(unsigned)sq_err_chunks(n_nodes), DET_RED, 0, (cudaStream_t)stream>>>(
        n_nodes, n_graphs, steps, pred, targets, data_batch, counter, sq_err, slots, ticket);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // extern "C"
