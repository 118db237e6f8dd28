// Matrix-free operator of the spectral node partitioner (datasets/distribute_graphs.py:90-115, 201-223: sklearn's
// SpectralClustering with an RBF affinity).  The reference forms the dense N×N affinity; here every product recomputes
// it from the positions, so memory stays O(N·k).
//
//   Y = s ⊙ ( A_off · (s ⊙ X) ),   A_ij = 2^(−γ₂ ‖x_i − x_j‖²) for j ≠ i, A_ii = 0,   γ₂ = γ·log₂e
//
// With s = d^−½ this is S·X, S = D^−½ (A − I) D^−½; with X = 1 and s = 1 it is the degree vector d.  Every entry is one
// fp32 ex2 of an fp32 squared distance of the caller's (centred) positions — the same bits for (i,j) and (j,i), since
// x_j − x_i = −(x_i − x_j) exactly.  A query row sums one 128-column tile in fp32 (at most 128 terms), adds that partial
// to fp64 accumulators, tile after tile in ascending order; column tiles are split over a grid dimension whose size is
// a function of N alone, and a second kernel adds the splits in ascending order.  No atomics: the same input gives the
// same bits on every call, stream and GPU.
//
// Also here: the tall-skinny fp64 products of the eigensolver (Gram matrices U·Vᵀ and combinations Cᵀ·U of vectors
// stored one after the other), with a fixed summation order for the same reason.
#include "common.cuh"

namespace degnn {

constexpr int SP_ROWS = 128;          // query rows per CTA, one per thread
constexpr int SP_COLS = 128;          // columns per shared-memory tile = terms per fp32 partial sum
constexpr int SP_TARGET_CTAS = 1024;  // column splits are chosen so that row tiles × splits reaches this (N only)
constexpr int GR_THREADS = 256;
constexpr int64_t GR_CHUNK = 8192;    // rows per Gram partial (fixed: the summation order depends on n only)

struct SpSplit {
    int64_t tiles;      // row tiles = column tiles
    int64_t per;        // column tiles per split
    int64_t splits;
};

static SpSplit sp_split(int64_t n) {
    SpSplit s;
    s.tiles = (n + SP_COLS - 1) / SP_COLS;
    int64_t want = (SP_TARGET_CTAS + s.tiles - 1) / s.tiles;
    if (want > s.tiles) want = s.tiles;
    if (want < 1) want = 1;
    s.per = (s.tiles + want - 1) / want;
    s.splits = (s.tiles + s.per - 1) / s.per;
    return s;
}

__device__ __forceinline__ float ex2f(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <int K, bool DIAG>
__device__ __forceinline__ void sp_tile(const float4* sp, const float* sw, float xi, float yi, float zi, float g2,
                                        int self, float (&f)[K]) {
#pragma unroll 4
    for (int jj = 0; jj < SP_COLS; ++jj) {
        const float4 p = sp[jj];
        const float dx = xi - p.x, dy = yi - p.y, dz = zi - p.z;
        const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
        float a = ex2f(-g2 * d2);
        if (DIAG && jj == self) a = 0.f;                       // the self term, excluded exactly
#pragma unroll
        for (int c = 0; c < K; ++c) f[c] = __fmaf_rn(a, sw[jj * K + c], f[c]);
    }
}

// grid (row tiles, splits); part[split][i][c]
template <int K>
__global__ void __launch_bounds__(SP_ROWS) spectral_apply_kernel(int64_t n, const float* __restrict__ pos, float g2,
                                                                 const double* __restrict__ scale,
                                                                 const double* __restrict__ x, double* __restrict__ part,
                                                                 int64_t per) {
    __shared__ float4 sp[SP_COLS];
    __shared__ __align__(16) float sw[SP_COLS * K];
    const int tid = threadIdx.x;
    const int64_t i = (int64_t)blockIdx.x * SP_ROWS + tid;
    const bool valid = i < n;
    const float xi = valid ? pos[3 * i] : 0.f, yi = valid ? pos[3 * i + 1] : 0.f, zi = valid ? pos[3 * i + 2] : 0.f;
    double acc[K];
#pragma unroll
    for (int c = 0; c < K; ++c) acc[c] = 0.0;
    const int64_t tiles = (n + SP_COLS - 1) / SP_COLS;
    const int64_t t0 = (int64_t)blockIdx.y * per;
    const int64_t t1 = t0 + per < tiles ? t0 + per : tiles;
    for (int64_t t = t0; t < t1; ++t) {
        const int64_t j = t * SP_COLS + tid;
        __syncthreads();
        if (j < n) {
            sp[tid] = make_float4(pos[3 * j], pos[3 * j + 1], pos[3 * j + 2], 0.f);
            const double sj = scale ? scale[j] : 1.0;
#pragma unroll
            for (int c = 0; c < K; ++c) sw[tid * K + c] = (float)(x ? sj * x[j * K + c] : sj);
        } else {                                               // padding columns: weight 0, a finite entry
            sp[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int c = 0; c < K; ++c) sw[tid * K + c] = 0.f;
        }
        __syncthreads();
        float f[K];
#pragma unroll
        for (int c = 0; c < K; ++c) f[c] = 0.f;
        if (t == (int64_t)blockIdx.x) sp_tile<K, true>(sp, sw, xi, yi, zi, g2, tid, f);
        else sp_tile<K, false>(sp, sw, xi, yi, zi, g2, tid, f);
#pragma unroll
        for (int c = 0; c < K; ++c) acc[c] += (double)f[c];
    }
    if (valid) {
        double* o = part + ((int64_t)blockIdx.y * n + i) * K;
#pragma unroll
        for (int c = 0; c < K; ++c) o[c] = acc[c];
    }
}

// y[i][c] = s_i · Σ_split part[split][i][c], splits in ascending order
__global__ void spectral_finish_kernel(int64_t n, int k, int64_t splits, const double* __restrict__ scale,
                                       const double* __restrict__ part, double* __restrict__ y) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * k) return;
    double v = 0.0;
    for (int64_t s = 0; s < splits; ++s) v += part[s * n * k + e];
    y[e] = scale ? scale[e / k] * v : v;
}

// Gram partials: ws[chunk][p][q] = Σ_{r in chunk} U[p][r]·V[q][r], grid (chunks, a); a fixed shuffle tree per warp and
// the warps in ascending order
__global__ void __launch_bounds__(GR_THREADS) spectral_gram_kernel(int64_t n, int a, int b, const double* __restrict__ U,
                                                                  const double* __restrict__ V, double* __restrict__ ws) {
    __shared__ double red[GR_THREADS / 32][16];
    const int p = blockIdx.y, tid = threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.x * GR_CHUNK;
    const int64_t r1 = r0 + GR_CHUNK < n ? r0 + GR_CHUNK : n;
    double acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = 0.0;
    const double* u = U + (int64_t)p * n;
    for (int64_t r = r0 + tid; r < r1; r += GR_THREADS) {
        const double ur = u[r];
#pragma unroll
        for (int q = 0; q < 16; ++q)
            if (q < b) acc[q] = fma(ur, V[(int64_t)q * n + r], acc[q]);
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        double v = acc[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        acc[q] = v;
    }
    const int w = tid >> 5, l = tid & 31;
    if (l == 0)
#pragma unroll
        for (int q = 0; q < 16; ++q) red[w][q] = acc[q];
    __syncthreads();
    if (tid < b) {
        double v = 0.0;
        for (int i = 0; i < GR_THREADS / 32; ++i) v += red[i][tid];
        ws[((int64_t)blockIdx.x * a + p) * b + tid] = v;
    }
}

__global__ void spectral_gram_finish_kernel(int a, int b, int64_t chunks, const double* __restrict__ ws,
                                            double* __restrict__ G) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a * b) return;
    double v = 0.0;
    for (int64_t c = 0; c < chunks; ++c) v += ws[c * a * b + e];
    G[e] = v;
}

// Y[q][r] = (subtract ? Y[q][r] : 0) ∓ Σ_p C[p][q]·U[p][r], p ascending
__global__ void spectral_combine_kernel(int64_t n, int a, int b, const double* __restrict__ U,
                                        const double* __restrict__ Cm, double* __restrict__ Y, int subtract) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = 0.0;
    for (int p = 0; p < a; ++p) {
        const double ur = U[(int64_t)p * n + r];
#pragma unroll
        for (int q = 0; q < 16; ++q)
            if (q < b) acc[q] = fma(__ldg(Cm + p * b + q), ur, acc[q]);
    }
#pragma unroll
    for (int q = 0; q < 16; ++q)
        if (q < b) {
            double* o = Y + (int64_t)q * n + r;
            *o = subtract ? *o - acc[q] : acc[q];
        }
}

template <int K>
static void launch_apply(int64_t n, const float* pos, float g2, const double* scale, const double* x, double* part,
                         const SpSplit& s, cudaStream_t st) {
    spectral_apply_kernel<K><<<dim3((unsigned)s.tiles, (unsigned)s.splits), SP_ROWS, 0, st>>>(n, pos, g2, scale, x, part,
                                                                                              s.per);
}

}  // namespace degnn

using namespace degnn;

extern "C" int distegnn_spectral_workspace_bytes(int64_t n_nodes, int k, int a, int64_t* bytes_host) {
    DEGNN_CHECK_ARG(bytes_host && n_nodes > 0, "null pointer / bad size");
    DEGNN_CHECK_ARG(k >= 1 && k <= DISTEGNN_SPECTRAL_MAX_K && a >= 1, "k outside [1,16] or a < 1");
    DEGNN_CHECK_ARG(n_nodes <= (int64_t)SP_COLS * 65535 * 16, "n_nodes too large");
    const SpSplit s = sp_split(n_nodes);
    const int64_t chunks = (n_nodes + GR_CHUNK - 1) / GR_CHUNK;
    const int64_t apply = s.splits * n_nodes * k * 8, gram = chunks * a * k * 8;
    *bytes_host = align256((size_t)(apply > gram ? apply : gram));
    return DISTEGNN_OK;
}

extern "C" int distegnn_spectral_apply(int64_t n_nodes, int k, const float* pos, float gamma_log2e, const double* scale,
                                       const double* x, double* y, void* workspace, int64_t workspace_bytes,
                                       void* stream) {
    DEGNN_CHECK_ARG(n_nodes > 0 && pos && y && workspace, "null pointer / bad size");
    DEGNN_CHECK_ARG(k >= 1 && k <= DISTEGNN_SPECTRAL_MAX_K, "k outside [1,16]");
    DEGNN_CHECK_ARG(x || k == 1, "x == NULL (all ones) needs k == 1");
    DEGNN_CHECK_ARG(gamma_log2e >= 0.f && gamma_log2e < INFINITY, "gamma_log2e must be finite and >= 0");
    int64_t need = 0;
    const int rc = distegnn_spectral_workspace_bytes(n_nodes, k, 1, &need);
    if (rc != DISTEGNN_OK) return rc;
    DEGNN_CHECK_ARG(workspace_bytes >= need, "workspace too small (distegnn_spectral_workspace_bytes)");
    const SpSplit s = sp_split(n_nodes);
    cudaStream_t st = (cudaStream_t)stream;
    double* part = (double*)workspace;
    switch (k) {
#define SP_CASE(KK) case KK: launch_apply<KK>(n_nodes, pos, gamma_log2e, scale, x, part, s, st); break;
        SP_CASE(1) SP_CASE(2) SP_CASE(3) SP_CASE(4) SP_CASE(5) SP_CASE(6) SP_CASE(7) SP_CASE(8)
        SP_CASE(9) SP_CASE(10) SP_CASE(11) SP_CASE(12) SP_CASE(13) SP_CASE(14) SP_CASE(15) SP_CASE(16)
#undef SP_CASE
    }
    const int64_t tot = n_nodes * k;
    spectral_finish_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(n_nodes, k, s.splits, scale, part, y);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_spectral_gram(int64_t n_nodes, int a, int b, const double* u, const double* v, double* g,
                                      void* workspace, int64_t workspace_bytes, void* stream) {
    DEGNN_CHECK_ARG(n_nodes > 0 && u && v && g && workspace, "null pointer / bad size");
    DEGNN_CHECK_ARG(a >= 1 && a <= 65535 && b >= 1 && b <= DISTEGNN_SPECTRAL_MAX_K, "a outside [1,65535] or b outside [1,16]");
    int64_t need = 0;
    const int rc = distegnn_spectral_workspace_bytes(n_nodes, b, a, &need);
    if (rc != DISTEGNN_OK) return rc;
    DEGNN_CHECK_ARG(workspace_bytes >= need, "workspace too small (distegnn_spectral_workspace_bytes)");
    const int64_t chunks = (n_nodes + GR_CHUNK - 1) / GR_CHUNK;
    cudaStream_t st = (cudaStream_t)stream;
    spectral_gram_kernel<<<dim3((unsigned)chunks, (unsigned)a), GR_THREADS, 0, st>>>(n_nodes, a, b, u, v,
                                                                                     (double*)workspace);
    spectral_gram_finish_kernel<<<(a * b + 255) / 256, 256, 0, st>>>(a, b, chunks, (const double*)workspace, g);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_spectral_combine(int64_t n_nodes, int a, int b, const double* u, const double* c, double* y,
                                         int subtract, void* stream) {
    DEGNN_CHECK_ARG(n_nodes > 0 && u && c && y, "null pointer / bad size");
    DEGNN_CHECK_ARG(a >= 1 && b >= 1 && b <= DISTEGNN_SPECTRAL_MAX_K, "a < 1 or b outside [1,16]");
    DEGNN_CHECK_ARG(subtract == 0 || subtract == 1, "subtract must be 0 or 1");
    spectral_combine_kernel<<<(unsigned)((n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n_nodes, a, b, u, c, y,
                                                                                                  subtract);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
