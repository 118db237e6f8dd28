// What the rollout's errors against recorded targets share (DESIGN §19, §20): the per-node distance, and the fixed-order
// per-graph sum over chunks of rows that adds it up.  distegnn_rollout_sq_err (rollout_err.cu) and
// distegnn_rollout_chamfer (chamfer.cu) both take their per-graph sums through `graph_chunk_sum`, so a sum of per-node
// minima of `target_sq_dist` is never above the sum of its matched terms: the two add in one order because they are one
// function.  Its row reduction, `det_row_sum`, is also the deterministic rollout centroid's (deterministic.cu).
#pragma once

#include "common.cuh"

namespace degnn {

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

// rows [lo, hi) of graph b in a sorted data_batch (lo <= hi for any batch); every row without a batch (one graph)
__device__ __forceinline__ void graph_rows(const int64_t* batch, int64_t N, int64_t b, int64_t& lo, int64_t& hi) {
    lo = batch ? lower_bound_dev(batch, N, b) : 0;
    hi = batch ? lower_bound_dev(batch, N, b + 1) : N;
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

constexpr int64_t SQERR_CHUNK = 2048;   // rows per block of the error sums: part of the summation order
inline int64_t err_chunks(int64_t N) { return (N + SQERR_CHUNK - 1) / SQERR_CHUNK; }

// out[b·NV + k] = Σ over the rows of graph b of component k of `term` (term(i, s) adds row i's NV components to s), for
// every graph b < B, by a grid of err_chunks(N) blocks of DET_RED threads.  Block c takes the rows [c·CH, (c+1)·CH) and
// sums each graph's rows in the chunk (batch sorted; found by a binary search inside the chunk) with det_row_sum.  A
// graph's first chunk stores its partial to out, each later chunk to its own slot (slots: [chunks, NV]); the last block
// to finish adds every graph's slots in chunk order.  So the order depends on N and the graph sizes alone, and every
// value is a plain store (a rerun overwrites).  `ticket` must be 0 at the launch; the last block leaves it 0.
// !keep: nothing is written but the ticket.
template <int NV, typename F>
__device__ __forceinline__ void graph_chunk_sum(int64_t N, int B, const int64_t* batch, bool keep, double* out,
                                                double* slots, unsigned* ticket, F term) {
    __shared__ double red[NV][DET_RED];
    __shared__ bool last;
    const int64_t c = blockIdx.x, r0 = c * SQERR_CHUNK, r1 = min(N, r0 + SQERR_CHUNK);
    for (int64_t i = r0; keep && i < r1;) {    // the graphs of the chunk, one after the other
        const int64_t b = batch ? __ldg(batch + i) : 0;
        const int64_t j = batch ? i + lower_bound_dev(batch + i, r1 - i, b + 1) : r1;
        det_row_sum<double, NV>(i, j, term, red);
        if (threadIdx.x == 0 && b >= 0 && b < B) {
            const bool first = i > r0 || r0 == 0 || (batch && __ldg(batch + r0 - 1) != b);   // starts in this chunk
            double* dst = first ? out + b * NV : slots + c * NV;
#pragma unroll
            for (int k = 0; k < NV; ++k) dst[k] = red[k][0];
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
    for (int u = threadIdx.x; u < NV * B; u += DET_RED) {
        const int b = u / NV, d = u % NV;
        int64_t lo, hi;
        graph_rows(batch, N, b, lo, hi);
        double acc = 0.0;
        if (hi > lo) {
            acc = __ldcg(out + u);
            int64_t k = lo / SQERR_CHUNK + 1;
            const int64_t k1 = (hi - 1) / SQERR_CHUNK;
            for (; k + 8 <= k1 + 1; k += 8) {  // eight independent loads in flight, added in chunk order
                double v[8];
#pragma unroll
                for (int w = 0; w < 8; ++w) v[w] = __ldcg(slots + (k + w) * NV + d);
#pragma unroll
                for (int w = 0; w < 8; ++w) acc += v[w];
            }
            for (; k <= k1; ++k) acc += __ldcg(slots + k * NV + d);
        }
        out[u] = acc;
    }
}

// d(u, v) = ‖u − v‖² of the rollout's errors: the differences in fp32 (round to nearest), their squares (exact) and the
// sum in fp64, in this order.  u(k), v(k) return coordinate k (0, 1, 2) of the two points, read in the order x, y, z.
// fl(a − b) = −fl(b − a), so d(u, v) and d(v, u) have the same bits.
template <typename U, typename V>
__device__ __forceinline__ double target_sq_dist(U u, V v) {
    const float dx = __fsub_rn(u(0), v(0));
    const float dy = __fsub_rn(u(1), v(1));
    const float dz = __fsub_rn(u(2), v(2));
    return ((double)dx * dx + (double)dy * dy) + (double)dz * dz;
}

// coordinate k of a point held in registers
__device__ __forceinline__ float xyz(const float4& p, int k) { return k == 0 ? p.x : (k == 1 ? p.y : p.z); }

}  // namespace degnn
