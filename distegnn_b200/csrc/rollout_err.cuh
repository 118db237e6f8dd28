// What the rollout's errors against recorded targets share (DESIGN §19, §20): the per-node distance, and the fixed-order
// per-graph reduction of the deterministic rollout centroid that sums it.  distegnn_rollout_sq_err (deterministic.cu)
// and distegnn_rollout_chamfer (chamfer.cu) both take their per-graph sums through det_row_sum over the same chunks of
// SQERR_CHUNK rows, so that a sum of per-node minima of `target_sq_dist` is never above the sum of its matched terms.
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
