// Loss side of the training step (SURVEY §8 f-3): node-count weighted MSE + MMD regulariser on the virtual coordinates,
// with the per-step scalar collectives folded into ONE packed SUM all-reduce.
//
// Reference: utils/train.py:98-147 — `loss(loc_pred, loc_target)` (MSE), two scalar all-reduces (total node count :104,
// logged loss :109) and an all_gather consistency check of `loc_mean` (:52-61) per step, then a Python loop over the
// graphs of the batch with `randperm` sampling, two `cdist` kernels (:11-14) per graph and ~20 small ATen launches each.
//
// Here (fp32).  Every sum is a chain per thread, a tree over the block (block_sum: 5 shuffle levels in a warp, 3 over
// the 8 warps) and one atomicAdd per block into a global accumulator, in no fixed order:
//   SSE         ⌈6144/256⌉ = 24 fmaf per thread of a node block, the tree, one atomicAdd per block of 2048 nodes
//   l_vv, l_rv  ⌈C²/256⌉ and ⌈S·C/256⌉ terms per thread, the tree, one atomicAdd per graph
//   ∂/∂Xv       the C + S pair terms of an entry, added by shared-memory atomicAdd
// so a sum Σ of positive terms is within γ_n·Σ, γ_n = n·u/(1 − n·u), u = 2⁻²⁴: n ≈ 2 + 24 + 8 + node_blocks + 2 for
// the SSE (489 node blocks at 1M nodes), n ≈ ⌈S·C/256⌉ + 8 + B for l_vv and l_rv, and an entry of ∂/∂Xv is within
// γ_{C+S−1}·Σ|term| plus each term's own roundings (tests/test_loss_kernel.py derives its bounds from this).
// n_r is converted to float, which is exact up to 2^24 nodes per rank.
//   distegnn_loss_partials   one launch: Σ(pred−target)² over the rank's nodes folded straight into the packed vector
//                            [n_r, n_r·MSE_r, loc_mean of this rank in its slot], and per graph l_vv = Σ k(V_c,V_c'),
//                            l_rv = Σ k(R_s,V_c), k(x,y) = exp(−‖x−y‖/(2σ²)) (distance NOT squared, :12-13), together with
//                            the un-weighted gradient of (l_vv/B/C² − 2·l_rv/B/S/C) w.r.t. the virtual coordinates
//   (caller)                 ONE all-reduce (SUM) of the packed vector: total node count, logged loss and every rank's
//                            loc_mean (each rank fills only its own slot) arrive together
//   distegnn_loss_finalize   one launch: coef = world·n_r/Σn (:110); loss = coef·(MSE + weight·MMD) / accumulation_steps;
//                            the gradients d loss/d pred [N,3] and d loss/d Xv [B,3,C] (the forward of a fused loss already
//                            knows them); logged loss; max deviation of the ranks' loc_mean from rank 0's
// Stepped (the *_steps entry points, DESIGN §26): K steps of a rollout in the same two launches, step t = blockIdx.y.
// Every block of step t runs the one-step arithmetic on step t's slices; the packed vector carries one n_r·MSE_r per
// step, [n_r, n_r·MSE_0 .. n_r·MSE_{K−1}, loc_mean slots], so K = 1 is the one-step layout and gives its bits; the
// finalize scales every step's gradient by coef/K and adds the K scalars in step order.
#include "common.cuh"

namespace degnn {

constexpr int LOSS_THREADS = 256;
constexpr int LOSS_NODES_PER_CTA = 2048;

struct LossArgs {
    int64_t N;
    int K, B, C, S, world, rank;
    float sigma, weight, inv_accum, inv_steps;
    const float* pred;        // [K,N,3]
    const float* target;      // [K,N,3]
    const float* Xv;          // [K,B,3,C]
    const float* loc_mean;    // [B,3] or null
    const int64_t* graph_ptr; // [B+1] first node of every graph (data_batch is sorted)
    const int32_t* samples;   // [K,B,S] local node indices drawn for the MMD (−1 = none), train.py:128-129
    float* acc;               // [K,3]: Σ_b l_vv, Σ_b l_rv, n_r·MSE_r    (zeroed by the caller)
    float* packed;            // [1 + K + world·3B]                      (zeroed by the caller)
    float* gV_raw;            // [K,B,3,C] gradient of (l_vv/B/C² − 2 l_rv/B/S/C) w.r.t. Xv
    float* g_pred;            // [K,N,3]
    float* g_Xv;              // [K,B,3,C]
    float* out;               // [4]: loss, logged loss, MMD term, max |loc_mean_r − loc_mean_0|
    float* out_steps;         // [2K] or null: logged loss and MMD term of every step
};

__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x < LOSS_THREADS / 32) s = sh[threadIdx.x];
    if (w == 0) {
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
    }
    return s;   // valid in thread 0
}

// blocks [0, node_blocks): squared error; blocks [node_blocks, node_blocks + B): MMD of graph b; blockIdx.y: the step
__global__ void __launch_bounds__(LOSS_THREADS) loss_partials_kernel(const LossArgs a, int node_blocks) {
    __shared__ float sh[LOSS_THREADS / 32];
    __shared__ float sV[3 * DISTEGNN_MAX_CHANNELS];
    __shared__ float sG[3 * DISTEGNN_MAX_CHANNELS];
    const int tid = threadIdx.x, t = blockIdx.y;
    const float* target = a.target + (size_t)t * a.N * 3;
    float* acc = a.acc + 3 * t;
    if ((int)blockIdx.x < node_blocks) {
        const float* pred = a.pred + (size_t)t * a.N * 3;
        const int64_t e0 = (int64_t)blockIdx.x * LOSS_NODES_PER_CTA * 3;
        const int64_t e1 = min(e0 + (int64_t)LOSS_NODES_PER_CTA * 3, a.N * 3);
        float s = 0.f;
        for (int64_t i = e0 + tid; i < e1; i += LOSS_THREADS) {
            const float d = __ldg(pred + i) - __ldg(target + i);
            s = fmaf(d, d, s);
        }
        s = block_sum(s, sh);
        if (tid == 0) {
            // n_r · MSE_r = n_r · sse / (3 n_r) = sse / 3: the rank's term of the logged loss before the division by Σn
            atomicAdd(a.packed + 1 + t, s * (1.0f / 3.0f));
            atomicAdd(acc + 2, s * (1.0f / 3.0f));
            if (blockIdx.x == 0 && t == 0) {
                a.packed[0] = (float)a.N;
                if (a.loc_mean)
                    for (int i = 0; i < 3 * a.B; ++i) a.packed[1 + a.K + (size_t)a.rank * 3 * a.B + i] = a.loc_mean[i];
            }
        }
        return;
    }
    const int b = blockIdx.x - node_blocks, C = a.C, S = a.S;
    const float inv2s2 = 1.0f / (2.0f * a.sigma * a.sigma);
    const int32_t* samples = a.samples + (size_t)t * a.B * S;
    if (tid < 3 * C) {
        sV[tid] = a.Xv[((size_t)t * a.B + b) * 3 * C + tid];     // [3][C]
        sG[tid] = 0.f;
    }
    __syncthreads();
    const float wvv = 1.0f / ((float)a.B * C * C), wrv = 2.0f / ((float)a.B * S * C);
    float lvv = 0.f, lrv = 0.f;
    // virtual-virtual: ordered pairs (c, c'); the gradient w.r.t. V_c collects both orders: 2·∂k(V_c,V_c')/∂V_c
    for (int p = tid; p < C * C; p += LOSS_THREADS) {
        const int c = p / C, d = p - c * C;
        const float dx = sV[c] - sV[d], dy = sV[C + c] - sV[C + d], dz = sV[2 * C + c] - sV[2 * C + d];
        const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
        const float k = expf(-dist * inv2s2);
        lvv += k;
        if (dist > 0.f) {                            // cdist's backward is 0 at coincident points
            const float g = -2.0f * wvv * k * inv2s2 / dist;
            atomicAdd(sG + c, g * dx);
            atomicAdd(sG + C + c, g * dy);
            atomicAdd(sG + 2 * C + c, g * dz);
        }
    }
    // sampled real nodes vs virtual: pairs (s, c)
    const int64_t n0 = a.graph_ptr[b];
    for (int p = tid; p < S * C; p += LOSS_THREADS) {
        const int s = p / C, c = p - s * C;
        const int li = samples[(size_t)b * S + s];
        if (li < 0) continue;
        const float* r = target + (size_t)(n0 + li) * 3;
        const float dx = sV[c] - __ldg(r), dy = sV[C + c] - __ldg(r + 1), dz = sV[2 * C + c] - __ldg(r + 2);
        const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
        const float k = expf(-dist * inv2s2);
        lrv += k;
        if (dist > 0.f) {
            const float g = wrv * k * inv2s2 / dist;     // −wrv · ∂k/∂V_c
            atomicAdd(sG + c, g * dx);
            atomicAdd(sG + C + c, g * dy);
            atomicAdd(sG + 2 * C + c, g * dz);
        }
    }
    lvv = block_sum(lvv, sh);
    lrv = block_sum(lrv, sh);
    __syncthreads();
    if (tid == 0) {
        atomicAdd(acc + 0, lvv);
        atomicAdd(acc + 1, lrv);
    }
    if (tid < 3 * C) a.gV_raw[((size_t)t * a.B + b) * 3 * C + tid] = sG[tid];
}

__device__ __forceinline__ float step_mmd(const LossArgs& a, int t) {                   // :142-145
    return a.acc[3 * t] / ((float)a.B * a.C * a.C) - 2.0f * a.acc[3 * t + 1] / ((float)a.B * a.S * a.C);
}

// after the all-reduce of `packed`: scalars (block (0, 0)) and the gradients (all blocks; blockIdx.y: the step)
__global__ void __launch_bounds__(LOSS_THREADS) loss_finalize_kernel(const LossArgs a) {
    const int tid = threadIdx.x, C = a.C, t = blockIdx.y;
    const float n_r = (float)a.N, n_tot = a.packed[0];
    const float share = n_r / n_tot;                                    // node_cnt / total_node_cnt, train.py:105
    const float coef = (float)a.world * share * a.inv_accum;            // :110 (DDP averages, the reference wants the sum), :150
    const float coef_t = coef * a.inv_steps;                            // the mean over the steps (K = 1: coef exactly)
    if (blockIdx.x == 0) {
        if (tid == 0 && t == 0) {
            // ℓ_t = coef·(MSE_t + weight·MMD_t), added in step order from step 0's value (K = 1: the one-step bits)
            float loss = 0.f, logged = 0.f, mmd = 0.f;
            for (int s = 0; s < a.K; ++s) {
                const float mse_s = n_r > 0.f ? a.acc[3 * s + 2] / n_r : 0.f;
                const float mmd_s = step_mmd(a, s);
                const float l_s = coef * (mse_s + a.weight * mmd_s);
                const float logged_s = a.packed[1 + s] / n_tot;         // Σ_r n_r/Σn · MSE_r  (:106-108)
                loss = s ? loss + l_s : l_s;
                logged = s ? logged + logged_s : logged_s;
                mmd = s ? mmd + mmd_s : mmd_s;
                if (a.out_steps) {
                    a.out_steps[s] = logged_s;
                    a.out_steps[a.K + s] = mmd_s;
                }
            }
            a.out[0] = loss * a.inv_steps;
            a.out[1] = logged * a.inv_steps;
            a.out[2] = mmd * a.inv_steps;
            const float* lm = a.packed + 1 + a.K;
            float dev = 0.f;
            if (a.loc_mean)
                for (int r = 1; r < a.world; ++r)
                    for (int i = 0; i < 3 * a.B; ++i)
                        dev = fmaxf(dev, fabsf(lm[(size_t)r * 3 * a.B + i] - lm[i]));
            a.out[3] = dev;
        }
        const float cV = coef_t * a.weight;
        const size_t o = (size_t)t * a.B * 3 * C;
        for (int i = tid; i < a.B * 3 * C; i += LOSS_THREADS) a.g_Xv[o + i] = cV * a.gV_raw[o + i];
    }
    const float cp = n_r > 0.f ? coef_t * 2.0f / (3.0f * n_r) : 0.f;    // d MSE / d pred = 2 (pred − target) / (3 n_r)
    const size_t o = (size_t)t * a.N * 3;
    const int64_t e0 = (int64_t)blockIdx.x * LOSS_NODES_PER_CTA * 3;
    const int64_t e1 = min(e0 + (int64_t)LOSS_NODES_PER_CTA * 3, a.N * 3);
    for (int64_t i = e0 + tid; i < e1; i += LOSS_THREADS)
        a.g_pred[o + i] = cp * (__ldg(a.pred + o + i) - __ldg(a.target + o + i));
}

}  // namespace degnn

static int loss_fill(degnn::LossArgs& a, int steps, int64_t n_nodes, int n_graphs, int C, int S, int world, int rank,
                     float sigma, float weight, int accumulation_steps, const float* pred, const float* target,
                     const float* Xv, const float* loc_mean, const int64_t* graph_ptr, const int32_t* samples, float* acc,
                     float* packed, float* gV_raw) {
    using namespace degnn;
    DEGNN_CHECK_ARG(steps >= 1 && steps <= 65535, "steps out of range [1, 65535]");
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(C >= 1 && C <= DISTEGNN_MAX_CHANNELS, "virtual_channels out of range");
    DEGNN_CHECK_ARG(S >= 1 && world >= 1 && rank >= 0 && rank < world && accumulation_steps >= 1, "bad argument");
    DEGNN_CHECK_ARG(sigma > 0.f, "sigma must be positive");
    DEGNN_CHECK_ARG((n_nodes == 0 || (pred && target)) && Xv && graph_ptr && samples && acc && packed && gV_raw,
                    "null pointer");
    a.N = n_nodes; a.K = steps; a.B = n_graphs; a.C = C; a.S = S; a.world = world; a.rank = rank;
    a.sigma = sigma; a.weight = weight; a.inv_accum = 1.0f / (float)accumulation_steps; a.inv_steps = 1.0f / (float)steps;
    a.pred = pred; a.target = target; a.Xv = Xv; a.loc_mean = loc_mean; a.graph_ptr = graph_ptr; a.samples = samples;
    a.acc = acc; a.packed = packed; a.gV_raw = gV_raw; a.g_pred = nullptr; a.g_Xv = nullptr; a.out = nullptr;
    a.out_steps = nullptr;
    return DISTEGNN_OK;
}

static int node_blocks_of(int64_t n_nodes) {
    const int nb = (int)((n_nodes + degnn::LOSS_NODES_PER_CTA - 1) / degnn::LOSS_NODES_PER_CTA);
    return nb < 1 ? 1 : nb;                                             // block 0 also writes n_r and the loc_mean slot
}

extern "C" int distegnn_loss_packed_floats_steps(int steps, int n_graphs, int world) {
    return 1 + steps + world * 3 * n_graphs;
}

extern "C" int distegnn_loss_packed_floats(int n_graphs, int world) {
    return distegnn_loss_packed_floats_steps(1, n_graphs, world);
}

extern "C" int distegnn_loss_partials_steps(int steps, int64_t n_nodes, int n_graphs, int C, int S, int world, int rank,
                                            float sigma, const float* pred, const float* target, const float* Xv,
                                            const float* loc_mean, const int64_t* graph_ptr, const int32_t* samples,
                                            float* acc, float* packed, float* gV_raw, void* stream) {
    using namespace degnn;
    LossArgs a;
    if (int rc = loss_fill(a, steps, n_nodes, n_graphs, C, S, world, rank, sigma, 0.f, 1, pred, target, Xv, loc_mean,
                           graph_ptr, samples, acc, packed, gV_raw))
        return rc;
    const int node_blocks = node_blocks_of(n_nodes);
    loss_partials_kernel<<<dim3((unsigned)(node_blocks + n_graphs), (unsigned)steps), LOSS_THREADS, 0,
                           (cudaStream_t)stream>>>(a, node_blocks);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_loss_partials(int64_t n_nodes, int n_graphs, int C, int S, int world, int rank, float sigma,
                                      const float* pred, const float* target, const float* Xv, const float* loc_mean,
                                      const int64_t* graph_ptr, const int32_t* samples, float* acc, float* packed,
                                      float* gV_raw, void* stream) {
    return distegnn_loss_partials_steps(1, n_nodes, n_graphs, C, S, world, rank, sigma, pred, target, Xv, loc_mean,
                                        graph_ptr, samples, acc, packed, gV_raw, stream);
}

extern "C" int distegnn_loss_finalize_steps(int steps, int64_t n_nodes, int n_graphs, int C, int S, int world, int rank,
                                            float sigma, float weight, int accumulation_steps, const float* pred,
                                            const float* target, const float* loc_mean, const float* acc,
                                            const float* packed, const float* gV_raw, float* g_pred, float* g_Xv,
                                            float* out, float* out_steps, void* stream) {
    using namespace degnn;
    LossArgs a;
    static const int64_t dummy_ptr = 0;
    static const int32_t dummy_smp = 0;
    if (int rc = loss_fill(a, steps, n_nodes, n_graphs, C, S, world, rank, sigma, weight, accumulation_steps, pred,
                           target, gV_raw /*unused Xv slot*/, loc_mean, &dummy_ptr, &dummy_smp, const_cast<float*>(acc),
                           const_cast<float*>(packed), const_cast<float*>(gV_raw)))
        return rc;
    DEGNN_CHECK_ARG((n_nodes == 0 || g_pred) && g_Xv && out, "null output pointer");
    a.g_pred = g_pred; a.g_Xv = g_Xv; a.out = out; a.out_steps = out_steps;
    loss_finalize_kernel<<<dim3((unsigned)node_blocks_of(n_nodes), (unsigned)steps), LOSS_THREADS, 0,
                           (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_loss_finalize(int64_t n_nodes, int n_graphs, int C, int S, int world, int rank, float sigma,
                                      float weight, int accumulation_steps, const float* pred, const float* target,
                                      const float* loc_mean, const float* acc, const float* packed, const float* gV_raw,
                                      float* g_pred, float* g_Xv, float* out, void* stream) {
    return distegnn_loss_finalize_steps(1, n_nodes, n_graphs, C, S, world, rank, sigma, weight, accumulation_steps, pred,
                                        target, loc_mean, acc, packed, gV_raw, g_pred, g_Xv, out, nullptr, stream);
}
