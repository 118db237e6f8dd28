// Lloyd iterations of the k-means node partitioner on the device (SURVEY §8 f-2).
//
// Reference: datasets/distribute_graphs.py:118-143, 188-198 — `KMeans(n_clusters=P, random_state=0, n_init="auto")
// .fit_predict(pos)` (sklearn, host) assigns every node of the big graph to one of P partitions.  The O(N·P·iterations)
// part runs here; the k-means++ seeding stays sklearn's own (`kmeans_plusplus`, which reproduces `random_state=0`) on the
// caller's side.  One call enqueues `iters` Lloyd iterations with sklearn's stopping rules evaluated ON THE DEVICE
// (`_kmeans_single_lloyd`): stop when no label changed (strict convergence) or when the squared centre shift falls to
// `tol` — then one more assignment pass so that labels match the final centres; iterations enqueued after convergence
// are no-ops.  state[0]: 0 running, 1 final assignment pending, 2 done; state[1]: iterations done; state[2]: labels
// changed in the last pass.  Cluster sums are accumulated in float64 (order-independent to ~1e-16).  The update step
// is sklearn's M-step (`_k_means_common.pyx`): empty clusters are relocated to the points farthest from their centres,
// then every centre is fp32(sum)·fp32(1/count) — so on data whose sums are exact the centres are sklearn's bit for bit.
// No extra device memory and no host synchronisation: the relocation runs inside the update launch when a count is 0.
//
// Points have D coordinates: D = 3 for node positions (distegnn_kmeans_lloyd, the k-means partitioner) and D = P <= 16
// for the spectral partitioner's embedding (distegnn_kmeans_lloyd_d, which also returns the inertia sklearn compares
// its n_init runs by).  The D = 3 instantiation keeps the three-term distance expression of the positions' path.
#include "common.cuh"

namespace degnn {

constexpr int KM_MAXK = 64;
constexpr int KM_MAXD = DISTEGNN_KMEANS_MAX_DIM;
constexpr int KM_THREADS = 256;
constexpr int KM_UPDATE_THREADS = 1024;
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

// (d, i) comes before (d', i') in the relocation order: larger distance first, then lower index
__device__ __forceinline__ bool km_before(float d, int64_t i, float d2, int64_t i2) {
    return d > d2 || (d == d2 && i < i2);
}

// sklearn's `_relocate_empty_clusters_dense`, between the assignment and the averaging: with distances
// d_i = ‖x_i − c_old[label_i]‖² to the centres the assignment used, the e-th empty cluster (ascending id) takes the e-th
// point in the order (d descending, index ascending): its sums become that point and count 1, and the point's own
// cluster loses it.  Labels are not changed.  Nothing moves when every d_i is 0.  One CTA, one pass over the points per
// empty cluster, each pass finding the next point after the previous one in that order — empty clusters are rare, and
// the launch costs only the count check otherwise.
template <int DT>
__device__ void km_relocate(const KmArgs& a, const float* sc, const int* empty, int n_empty) {
    __shared__ float rd[KM_UPDATE_THREADS / 32];
    __shared__ long long ri[KM_UPDATE_THREADS / 32];
    __shared__ float pick_d;
    __shared__ long long pick_i;
    const int tid = threadIdx.x, D = DT == 3 ? 3 : a.D, W = D + 1;
    float pd = INFINITY;
    int64_t pi = -1;
    for (int e = 0; e < n_empty; ++e) {
        float bd = -1.f;
        int64_t bi = -1;
        for (int64_t i = tid; i < a.N; i += KM_UPDATE_THREADS) {
            float x[KM_MAXD];
            km_load<DT>(a.pos, i, D, x);
            const float d = km_dist<DT>(x, sc, a.labels[i], D);
            if (km_before(pd, pi, d, i) && (bi < 0 || km_before(d, i, bd, bi))) { bd = d; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(FULL, bd, o);
            const long long oi = __shfl_xor_sync(FULL, (long long)bi, o);
            if (oi >= 0 && (bi < 0 || km_before(od, oi, bd, bi))) { bd = od; bi = oi; }
        }
        if ((tid & 31) == 0) { rd[tid >> 5] = bd; ri[tid >> 5] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < KM_UPDATE_THREADS / 32; ++w)
                if (ri[w] >= 0 && (bi < 0 || km_before(rd[w], ri[w], bd, bi))) { bd = rd[w]; bi = ri[w]; }
            pick_d = bd; pick_i = bi;
            if (bi >= 0 && !(e == 0 && bd == 0.f)) {       // the farthest point sits on its centre: nothing moves
                const int knew = empty[e], kold = a.labels[bi];
                float x[KM_MAXD];
                km_load<DT>(a.pos, bi, D, x);
                for (int c = 0; c < D; ++c) {
                    a.sums[W * kold + c] -= (double)x[c];
                    a.sums[W * knew + c] = (double)x[c];
                }
                a.sums[W * kold + D] -= 1.0;
                a.sums[W * knew + D] = 1.0;
            }
        }
        __syncthreads();
        pd = pick_d; pi = pick_i;
        if (pi < 0 || (e == 0 && pd == 0.f)) return;      // fewer points than empty clusters: the rest stay empty
    }
}

// sklearn's `_average_centers` and `_center_shift`: centre = fp32(sum) · fp32(1/count), the product rounded once (the
// fp64 sums hold the fp32 sums exactly wherever those are exact); a cluster still empty after the relocation (every
// point on its centre, or a relocated point that was alone in its cluster) takes the centre of the first largest
// cluster m — as sklearn fills its buffer in cluster order, that is m's mean when m < k and m's plain sum otherwise.
template <int DT>
__global__ void __launch_bounds__(KM_UPDATE_THREADS) kmeans_update_kernel(const KmArgs a) {
    __shared__ float sc[KM_MAXK * KM_MAXD];
    __shared__ float shift[KM_MAXK];
    __shared__ int empty[KM_MAXK];
    __shared__ int n_empty, amax;
    const int st = a.state[0];
    if (st == 2) return;
    const int tid = threadIdx.x, K = a.K, D = a.D, W = D + 1;
    if (st == 1) {                                        // the final assignment has run
        if (tid == 0) a.state[0] = 2;
        return;
    }
    for (int i = tid; i < K * D; i += KM_UPDATE_THREADS) sc[i] = a.centers[i];
    if (tid == 0) {
        int n = 0;
        for (int k = 0; k < K; ++k)
            if (a.sums[W * k + D] == 0.0) empty[n++] = k;
        n_empty = n;
    }
    __syncthreads();
    if (n_empty) km_relocate<DT>(a, sc, empty, n_empty);
    if (tid == 0) {
        int m = 0;
        for (int k = 1; k < K; ++k)
            if (a.sums[W * k + D] > a.sums[W * m + D]) m = k;
        amax = m;
    }
    __syncthreads();
    float cc[KM_MAXD];
    if (tid < K) {
        const int k = tid, m = amax;
        const double n = a.sums[W * k + D];
        const int src = n > 0.0 ? k : m;
        const bool mean = n > 0.0 || m < k;
        const double alpha = (double)(float)(1.0 / a.sums[W * src + D]);
#pragma unroll
        for (int c = 0; c < KM_MAXD; ++c)
            if (c < D) cc[c] = mean ? (float)(a.sums[W * src + c] * alpha) : (float)a.sums[W * src + c];
    }
    __syncthreads();                                      // every thread has read the sums it needs
    if (tid < K) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < KM_MAXD; ++c)
            if (c < D) {
                const float dc = cc[c] - sc[D * tid + c];
                s += dc * dc;
                a.centers[D * tid + c] = cc[c];
            }
        for (int c = 0; c < W; ++c) a.sums[W * tid + c] = 0.0;
        shift[tid] = s;
    }
    __syncthreads();
    if (tid == 0) {
        float tot = 0.f;
        for (int i = 0; i < K; ++i) tot += shift[i];
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
        if (a.D == 3) {
            kmeans_assign_kernel<3><<<(unsigned)blocks, KM_THREADS, 0, st>>>(a);
            kmeans_update_kernel<3><<<1, KM_UPDATE_THREADS, 0, st>>>(a);
        } else {
            kmeans_assign_kernel<0><<<(unsigned)blocks, KM_THREADS, 0, st>>>(a);
            kmeans_update_kernel<0><<<1, KM_UPDATE_THREADS, 0, st>>>(a);
        }
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
