// Lloyd iterations of the k-means node partitioner on the device (SURVEY §8 f-2).
//
// Reference: datasets/distribute_graphs.py:118-143, 188-198 — `KMeans(n_clusters=P, random_state=0, n_init="auto")
// .fit_predict(pos)` (sklearn, host) assigns every node of the big graph to one of P partitions.  The O(N·P·iterations)
// part runs here; the k-means++ seeding stays sklearn's own (`kmeans_plusplus`, which reproduces `random_state=0`) on the
// caller's side.  One call enqueues `iters` Lloyd iterations with sklearn's stopping rules evaluated ON THE DEVICE
// (`_kmeans_single_lloyd`): stop when no label changed (strict convergence) or when the squared centre shift falls to
// `tol` — then one more assignment pass so that labels match the final centres; iterations enqueued after convergence
// are no-ops.  state[0]: 0 running, 1 final assignment pending, 2 done; state[1]: iterations done; state[2]: labels
// changed in the last pass.  Cluster sums are accumulated in float64 (order-independent to ~1e-16).
//
// Points have D coordinates: D = 3 for node positions (distegnn_kmeans_lloyd, the k-means partitioner) and D = P <= 16
// for the spectral partitioner's embedding (distegnn_kmeans_lloyd_d, which also returns the inertia sklearn compares
// its n_init runs by).  The D = 3 instantiation keeps the three-term distance expression of the positions' path.
#include "common.cuh"

namespace degnn {

constexpr int KM_MAXK = 64;
constexpr int KM_MAXD = DISTEGNN_KMEANS_MAX_DIM;
constexpr int KM_THREADS = 256;
constexpr int KM_INERTIA_THREADS = 1024;

struct KmArgs {
    int64_t N;
    int K;
    int D;
    float tol;
    const float* pos;       // [N,D]
    float* centers;         // [K,D]
    int32_t* labels;        // [N] (in: previous labels, −1 initially)
    double* sums;           // [K,D+1] Σx_0 .. Σx_{D-1}, count   (zero on entry to every pass)
    int32_t* state;         // [4]
    double* inertia;        // [1] or NULL
};

// squared distance of point `x` to centre k; DT = 3: the positions' expression, DT = 0: D coordinates in order
template <int DT>
__device__ __forceinline__ float km_dist(const float* x, const float* sc, int k, int D) {
    if constexpr (DT == 3) {
        const float dx = x[0] - sc[3 * k], dy = x[1] - sc[3 * k + 1], dz = x[2] - sc[3 * k + 2];
        return dx * dx + dy * dy + dz * dz;
    } else {
        float d = 0.f;
#pragma unroll
        for (int c = 0; c < KM_MAXD; ++c)
            if (c < D) {
                const float t = x[c] - sc[k * D + c];
                d = __fmaf_rn(t, t, d);
            }
        return d;
    }
}

template <int DT>
__device__ __forceinline__ void km_load(const float* pos, int64_t i, int D, float (&x)[KM_MAXD]) {
    if constexpr (DT == 3) {
        x[0] = __ldg(pos + i * 3); x[1] = __ldg(pos + i * 3 + 1); x[2] = __ldg(pos + i * 3 + 2);
    } else {
#pragma unroll
        for (int c = 0; c < KM_MAXD; ++c)
            if (c < D) x[c] = __ldg(pos + i * D + c);
    }
}

template <int DT>
__global__ void __launch_bounds__(KM_THREADS) kmeans_assign_kernel(const KmArgs a) {
    constexpr int DMAX = DT == 3 ? 3 : KM_MAXD;             // the positions' path keeps its small footprint
    __shared__ float sc[KM_MAXK * DMAX];
    __shared__ double ssum[KM_MAXK * (DMAX + 1)];
    __shared__ int schanged;
    const int st = a.state[0];
    if (st == 2) return;
    const int tid = threadIdx.x, K = a.K, D = DT == 3 ? 3 : a.D, W = D + 1;
    for (int i = tid; i < K * D; i += KM_THREADS) sc[i] = a.centers[i];
    for (int i = tid; i < K * W; i += KM_THREADS) ssum[i] = 0.0;
    if (tid == 0) schanged = 0;
    __syncthreads();
    int changed = 0;
    for (int64_t i = (int64_t)blockIdx.x * KM_THREADS + tid; i < a.N; i += (int64_t)gridDim.x * KM_THREADS) {
        float x[KM_MAXD];
        km_load<DT>(a.pos, i, D, x);
        float best = INFINITY;
        int bk = 0;
        for (int k = 0; k < K; ++k) {
            const float d = km_dist<DT>(x, sc, k, D);
            if (d < best) { best = d; bk = k; }          // first minimum wins, as argmin
        }
        if (a.labels[i] != bk) {
            ++changed;
            a.labels[i] = bk;
        }
        if (st == 0) {
#pragma unroll
            for (int c = 0; c < KM_MAXD; ++c)
                if (c < D) atomicAdd(ssum + W * bk + c, (double)x[c]);
            atomicAdd(ssum + W * bk + D, 1.0);
        }
    }
    if (changed) atomicAdd(&schanged, changed);
    __syncthreads();
    if (st == 0)
        for (int i = tid; i < K * W; i += KM_THREADS)
            if (ssum[i] != 0.0) atomicAdd(a.sums + i, ssum[i]);
    if (tid == 0 && schanged) atomicAdd(a.state + 2, schanged);
}

__global__ void kmeans_update_kernel(const KmArgs a) {
    __shared__ float shift[KM_MAXK];
    const int st = a.state[0];
    if (st == 2) return;
    const int k = threadIdx.x, D = a.D, W = D + 1;
    if (st == 1) {                                        // the final assignment has run
        if (k == 0) a.state[0] = 2;
        return;
    }
    float s = 0.f;
    if (k < a.K) {
        const double n = a.sums[W * k + D];
        if (n > 0.0) {                                    // an empty cluster keeps its centre
            for (int c = 0; c < D; ++c) {
                const float cc = (float)(a.sums[W * k + c] / n);
                const float dc = cc - a.centers[D * k + c];
                s += dc * dc;
                a.centers[D * k + c] = cc;
            }
        }
        for (int c = 0; c < W; ++c) a.sums[W * k + c] = 0.0;
    }
    if (k < KM_MAXK) shift[k] = s;
    __syncthreads();
    if (k == 0) {
        float tot = 0.f;
        for (int i = 0; i < a.K; ++i) tot += shift[i];
        a.state[1] += 1;
        if (a.state[2] == 0) a.state[0] = 2;              // strict convergence: labels already match the centres
        else if (tot <= a.tol) a.state[0] = 1;            // converged by tolerance: one more assignment pass
        a.state[2] = 0;
    }
}

// Σ_i ‖x_i − c_{label_i}‖² once the iterations are done: one CTA, thread t takes rows t, t + 1024, ... in order, then a
// fixed shuffle tree and the warps in order — the same bits on every call and GPU
__global__ void __launch_bounds__(KM_INERTIA_THREADS) kmeans_inertia_kernel(const KmArgs a) {
    __shared__ double red[KM_INERTIA_THREADS / 32];
    if (a.state[0] != 2) return;
    const int tid = threadIdx.x, D = a.D;
    double acc = 0.0;
    for (int64_t i = tid; i < a.N; i += KM_INERTIA_THREADS) {
        float x[KM_MAXD];
        km_load<0>(a.pos, i, D, x);
        acc += (double)km_dist<0>(x, a.centers, a.labels[i], D);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
    if ((tid & 31) == 0) red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
        double v = 0.0;
        for (int w = 0; w < KM_INERTIA_THREADS / 32; ++w) v += red[w];
        a.inertia[0] = v;
    }
}

static int kmeans_run(const KmArgs& a, int iters, cudaStream_t st) {
    int64_t blocks = (a.N + KM_THREADS * 4 - 1) / (KM_THREADS * 4);
    if (blocks > 8 * sm_count()) blocks = 8 * sm_count();
    for (int it = 0; it < iters; ++it) {
        if (a.D == 3) kmeans_assign_kernel<3><<<(unsigned)blocks, KM_THREADS, 0, st>>>(a);
        else kmeans_assign_kernel<0><<<(unsigned)blocks, KM_THREADS, 0, st>>>(a);
        kmeans_update_kernel<<<1, KM_MAXK, 0, st>>>(a);
    }
    if (a.inertia) kmeans_inertia_kernel<<<1, KM_INERTIA_THREADS, 0, st>>>(a);
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" int distegnn_kmeans_lloyd_d(int64_t n_nodes, int n_clusters, int dim, const float* pos, float* centers,
                                       int32_t* labels, double* sums, int32_t* state, float tol, int iters,
                                       double* inertia, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes > 0 && pos && centers && labels && sums && state, "null pointer / bad size");
    DEGNN_CHECK_ARG(n_clusters >= 1 && n_clusters <= KM_MAXK, "n_clusters outside [1,64]");
    DEGNN_CHECK_ARG(dim >= 1 && dim <= KM_MAXD, "dim outside [1,16]");
    DEGNN_CHECK_ARG(iters >= 1 && tol >= 0.f, "bad iteration count / tolerance");
    KmArgs a;
    a.N = n_nodes; a.K = n_clusters; a.D = dim; a.tol = tol; a.pos = pos; a.centers = centers; a.labels = labels;
    a.sums = sums; a.state = state; a.inertia = inertia;
    kmeans_run(a, iters, (cudaStream_t)stream);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_kmeans_lloyd(int64_t n_nodes, int n_clusters, const float* pos, float* centers, int32_t* labels,
                                     double* sums, int32_t* state, float tol, int iters, void* stream) {
    return distegnn_kmeans_lloyd_d(n_nodes, n_clusters, 3, pos, centers, labels, sums, state, tol, iters, nullptr, stream);
}
