// Virtual-node update, fused with the cross-partition SUM all-reduce of the packed statistics (one CTA per graph).
//
// Reference: the global halves of coord_model_virtual / node_model_virtual and the next layer's m_X
// (models/FastEGNN.py:199, 229-233, 258-264) behind weighted_average_reduce (:310-319), which the reference runs as 6 NCCL
// calls + host syncs per layer.  Here the CTA of graph b first all-reduces vsum[b,:] over NVLink peer memory (comm.cuh;
// skipped for a single partition), then computes from the summed statistics
//   n = max(vsum[b,3],1);  Xv += vsum[b,4:4+3C]/n;  Hv += MLP_hv([Hv; vsum[b,4+3C:]/n])
//   x̄ = vsum[b,0:3]/n;  m_X = (Xv−x̄)ᵀ(Xv−x̄);  G_next = W1v_V·Hv + W1v_M·m_X + b1v (next layer's)
// and leaves vsum either holding the summed statistics (training path keeps them) or zeroed for the next layer's
// accumulation (FLAG_ZERO_VSUM: no memset launch between layers).
#include "virtual_update.cuh"

namespace degnn {

template <bool SYNC>
__global__ void __launch_bounds__(VU_THREADS) virtual_update_kernel(const VUpdArgs a, const CommDev cd) {
    const int b = blockIdx.x;
    const NoPause pause;
#include "virtual_update_graph.cuh"
}

}  // namespace degnn

extern "C" int distegnn_virtual_update_fwd(int n_graphs, int A, int C, int Na, unsigned flags, float* vsum, float* Xv,
                                           float* Hv, const float* layer_params, const float* next_layer_params,
                                           float* G, const float* init_loc_mean, const float* init_hv0, void* comm,
                                           void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_graphs == 0) return DISTEGNN_OK;
    VUpdArgs a;
    if (int rc = virtual_update_args(__func__, n_graphs, A, C, Na, flags, vsum, Xv, Hv, layer_params, next_layer_params,
                                     G, init_loc_mean, init_hv0, &a))
        return rc;
    if (comm) {
        const CommHost* c = (const CommHost*)comm;
        DEGNN_CHECK_ARG(c->connected, "comm not connected (distegnn_comm_connect)");
        DEGNN_CHECK_ARG(n_graphs <= c->dev.max_slots && a.K <= c->dev.stride,
                        "comm capacity (max_slots, slot_floats) too small for [n_graphs, K]");
        virtual_update_kernel<true><<<(unsigned)n_graphs, VU_THREADS, 0, (cudaStream_t)stream>>>(a, c->dev);
    } else {
        CommDev none;
        none.world = 1; none.rank = 0;
        virtual_update_kernel<false><<<(unsigned)n_graphs, VU_THREADS, 0, (cudaStream_t)stream>>>(a, none);
    }
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

// =====================================================================================================================
// Backward of the virtual-node update (SURVEY §8 f-1; in the reference: autograd through models/FastEGNN.py:193-199,
// 222-234, 258-264).  One CTA per graph, everything recomputed from vsum / Xv / Hv; replaces torch recompute + autograd
// (a dozen cuBLAS / elementwise launches per layer on [B,C,64] tensors).  The node count n = vsum[b,3] is a constant of
// the graph (the reference divides by detached counts), so g_vsum[b,3] = 0.
// =====================================================================================================================
namespace degnn {

struct VUpdBwdArgs {
    int B, C, K;
    unsigned flags;
    const float* vsum; const float* Xv; const float* Hv;
    const float* m1; const float* mb1; const float* m2; const float* mb2;
    const float* nv1v; const float* nv1m; const float* nvb1;
    const float* g_Xn; const float* g_Hn; const float* g_G;     // upstream (g_Hn / g_G null with FLAG_LAST)
    float* g_vsum; float* g_Xv; float* g_Hv;                    // written
    float* d_m1; float* d_mb1; float* d_m2; float* d_mb2;       // accumulated (this layer's block)
    float* d_nv1v; float* d_nv1m; float* d_nvb1;                // accumulated (next layer's block)
};

__global__ void __launch_bounds__(NTHREADS) virtual_update_bwd_kernel(const VUpdBwdArgs a) {
    constexpr int MC = DISTEGNN_MAX_CHANNELS;
    __shared__ float sX[3 * MC], sZ[3 * MC], sM[MC * MC], sgM[MC * MC], sgZ[3 * MC];
    __shared__ float sHv[MC * H], sAg[MC * H], sZ1[MC * H], sT[MC * H], sHn[MC * H], sgG[MC * H], sgH[MC * H], sgz[MC * H];
    const int b = blockIdx.x, tid = threadIdx.x, C = a.C, K = a.K;
    const float* vs = a.vsum + (size_t)b * K;
    float* gv = a.g_vsum + (size_t)b * K;
    const bool init = a.flags & DISTEGNN_FLAG_INIT, last = a.flags & DISTEGNN_FLAG_LAST;
    const float inv = 1.0f / fmaxf(vs[3], 1.0f);
    for (int i = tid; i < K; i += NTHREADS) gv[i] = 0.f;
    if (last) {                                                 // X' = Xv + S/n only
        __syncthreads();
        if (tid < 3 * C) {
            const float g = a.g_Xn ? a.g_Xn[(size_t)b * 3 * C + tid] : 0.f;
            a.g_Xv[(size_t)b * 3 * C + tid] = g;
            gv[4 + tid] = g * inv;
        }
        return;
    }
    // ---- recompute the forward quantities -------------------------------------------------------------------------------
    if (tid < 3 * C) {
        float x = a.Xv[(size_t)b * 3 * C + tid];
        if (!init) x += vs[4 + tid] * inv;
        sX[tid] = x;
        sZ[tid] = x - vs[tid / C] * inv;
    }
    for (int i = tid; i < C * H; i += NTHREADS) {
        sHv[i] = a.Hv[(size_t)b * C * H + i];
        sAg[i] = init ? 0.f : vs[4 + 3 * C + i] * inv;
        sgG[i] = a.g_G ? a.g_G[(size_t)b * C * H + i] : 0.f;
    }
    __syncthreads();
    if (tid < C * C) {
        const int i = tid / C, j = tid - i * C;
        sM[tid] = sZ[i] * sZ[j] + sZ[C + i] * sZ[C + j] + sZ[2 * C + i] * sZ[2 * C + j];
    }
    if (!init) {
        for (int i = tid; i < C * H; i += NTHREADS) {
            const int c = i / H, n = i - c * H;
            float s = __ldg(a.mb1 + n);
#pragma unroll 16
            for (int k = 0; k < H; ++k) s = fmaf(sHv[c * H + k], __ldg(a.m1 + k * H + n), s);
#pragma unroll 16
            for (int k = 0; k < H; ++k) s = fmaf(sAg[c * H + k], __ldg(a.m1 + (H + k) * H + n), s);
            sZ1[i] = s;
            sT[i] = silu(s);
        }
        __syncthreads();
        for (int i = tid; i < C * H; i += NTHREADS) {
            const int c = i / H, n = i - c * H;
            float s = __ldg(a.mb2 + n);
#pragma unroll 16
            for (int k = 0; k < H; ++k) s = fmaf(sT[c * H + k], __ldg(a.m2 + k * H + n), s);
            sHn[i] = sHv[i] + s;
        }
    } else {
        for (int i = tid; i < C * H; i += NTHREADS) sHn[i] = sHv[i];
    }
    __syncthreads();
    // ---- G = Hn·V1V + m_Xᵀ·V1M + b: parameter gradients, g_Hn, g_mX --------------------------------------------------------
    for (int i = tid; i < H * H; i += NTHREADS) {               // d V1V[k][n] += Σ_c Hn[c][k]·g_G[c][n]
        const int k = i / H, n = i - k * H;
        float s = 0.f;
        for (int c = 0; c < C; ++c) s = fmaf(sHn[c * H + k], sgG[c * H + n], s);
        atomicAdd(a.d_nv1v + i, s);
    }
    for (int i = tid; i < C * H; i += NTHREADS) {               // d V1M[j][n] += Σ_c m_X[j][c]·g_G[c][n]
        const int j = i / H, n = i - j * H;
        float s = 0.f;
        for (int c = 0; c < C; ++c) s = fmaf(sM[j * C + c], sgG[c * H + n], s);
        atomicAdd(a.d_nv1m + i, s);
    }
    if (tid < H) {
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += sgG[c * H + tid];
        atomicAdd(a.d_nvb1 + tid, s);
    }
    for (int i = tid; i < C * H; i += NTHREADS) {               // g_Hn[c][k] = upstream + Σ_n g_G[c][n]·V1V[k][n]
        const int c = i / H, k = i - c * H;
        float s = a.g_Hn ? a.g_Hn[(size_t)b * C * H + i] : 0.f;
#pragma unroll 16
        for (int n = 0; n < H; ++n) s = fmaf(sgG[c * H + n], __ldg(a.nv1v + k * H + n), s);
        sgH[i] = s;
    }
    if (tid < C * C) {                                          // g_mX[j][c] = Σ_n g_G[c][n]·V1M[j][n]
        const int j = tid / C, c = tid - j * C;
        float s = 0.f;
        for (int n = 0; n < H; ++n) s = fmaf(sgG[c * H + n], __ldg(a.nv1m + j * H + n), s);
        sgM[tid] = s;
    }
    __syncthreads();
    if (tid < 3 * C) {                                          // m_X = ZᵀZ: g_Z[d][i] = Σ_j (g_mX[i][j] + g_mX[j][i])·Z[d][j]
        const int d = tid / C, i = tid - d * C;
        float s = 0.f;
        for (int j = 0; j < C; ++j) s = fmaf(sgM[i * C + j] + sgM[j * C + i], sZ[d * C + j], s);
        sgZ[tid] = s;
    }
    __syncthreads();
    if (tid < 3 * C) {                                          // Z = X' − x̄, X' = Xv (+ S/n)
        const float g = (a.g_Xn ? a.g_Xn[(size_t)b * 3 * C + tid] : 0.f) + sgZ[tid];
        a.g_Xv[(size_t)b * 3 * C + tid] = g;
        if (!init) gv[4 + tid] = g * inv;
    }
    if (tid < 3) {                                              // x̄ = vsum[0:3]/n
        float s = 0.f;
        for (int i = 0; i < C; ++i) s += sgZ[tid * C + i];
        gv[tid] = -s * inv;
    }
    if (init) {                                                 // Hn = Hv
        for (int i = tid; i < C * H; i += NTHREADS) a.g_Hv[(size_t)b * C * H + i] = sgH[i];
        return;
    }
    // ---- Hn = Hv + SiLU([Hv | agg]·M1 + b1)·M2 + b2 ---------------------------------------------------------------------------
    for (int i = tid; i < H * H; i += NTHREADS) {               // d M2[k][n] += Σ_c t[c][k]·g_Hn[c][n]
        const int k = i / H, n = i - k * H;
        float s = 0.f;
        for (int c = 0; c < C; ++c) s = fmaf(sT[c * H + k], sgH[c * H + n], s);
        atomicAdd(a.d_m2 + i, s);
    }
    if (tid < H) {
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += sgH[c * H + tid];
        atomicAdd(a.d_mb2 + tid, s);
    }
    for (int i = tid; i < C * H; i += NTHREADS) {               // g_z[c][k] = (Σ_n g_Hn[c][n]·M2[k][n])·SiLU'(z)
        const int c = i / H, k = i - c * H;
        float s = 0.f;
#pragma unroll 16
        for (int n = 0; n < H; ++n) s = fmaf(sgH[c * H + n], __ldg(a.m2 + k * H + n), s);
        const float z = sZ1[i], e = __expf(-z), sg = 1.0f / (1.0f + e);
        sgz[i] = s * sg * fmaf(z, 1.0f - sg, 1.0f);
    }
    __syncthreads();
    for (int i = tid; i < 2 * H * H; i += NTHREADS) {           // d M1[k][n] += Σ_c cat[c][k]·g_z[c][n]
        const int k = i / H, n = i - k * H;
        const float* src = k < H ? sHv + k : sAg + (k - H);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s = fmaf(src[c * H], sgz[c * H + n], s);
        atomicAdd(a.d_m1 + i, s);
    }
    if (tid < H) {
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += sgz[c * H + tid];
        atomicAdd(a.d_mb1 + tid, s);
    }
    for (int i = tid; i < 2 * C * H; i += NTHREADS) {           // g_cat[c][k] = Σ_n g_z[c][n]·M1[k][n]
        const int c = i / (2 * H), k = i - c * 2 * H;
        float s = 0.f;
#pragma unroll 16
        for (int n = 0; n < H; ++n) s = fmaf(sgz[c * H + n], __ldg(a.m1 + k * H + n), s);
        if (k < H) a.g_Hv[(size_t)b * C * H + c * H + k] = sgH[c * H + k] + s;      // residual + first half of the concatenation
        else gv[4 + 3 * C + c * H + (k - H)] = s * inv;                              // agg = vsum[4+3C:]/n
    }
}

}  // namespace degnn

extern "C" int distegnn_virtual_update_bwd(int n_graphs, int A, int C, int Na, unsigned flags, const float* vsum,
                                           const float* Xv, const float* Hv, const float* layer_params,
                                           const float* next_layer_params, const float* g_Xn, const float* g_Hn,
                                           const float* g_G, float* g_vsum, float* g_Xv, float* g_Hv, float* g_layer_params,
                                           float* g_next_layer_params, void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_graphs == 0) return DISTEGNN_OK;
    const bool last = flags & DISTEGNN_FLAG_LAST, init = flags & DISTEGNN_FLAG_INIT;
    DEGNN_CHECK_ARG(n_graphs > 0 && vsum && Xv && g_vsum && g_Xv, "null pointer / bad size");
    DEGNN_CHECK_ARG(last || (Hv && g_Hv && next_layer_params && g_next_layer_params), "null pointer (non-last)");
    DEGNN_CHECK_ARG(last || init || (layer_params && g_layer_params), "null layer_params (regular layer)");
    DEGNN_CHECK_ARG(!(flags & DISTEGNN_FLAG_INIT_CENTROID), "FLAG_INIT_CENTROID is for inference (no gradient through x̄)");
    Layout L = make_layout(A, C, Na);
    VUpdBwdArgs a;
    a.B = n_graphs; a.C = C; a.K = 4 + 3 * C + H * C; a.flags = flags;
    a.vsum = vsum; a.Xv = Xv; a.Hv = Hv;
    const float* lp = layer_params;
    a.m1 = lp ? lp + L.off[DISTEGNN_P_M_W1] : nullptr; a.mb1 = lp ? lp + L.off[DISTEGNN_P_M_B1] : nullptr;
    a.m2 = lp ? lp + L.off[DISTEGNN_P_M_W2] : nullptr; a.mb2 = lp ? lp + L.off[DISTEGNN_P_M_B2] : nullptr;
    const float* nx = next_layer_params;
    a.nv1v = nx ? nx + L.off[DISTEGNN_P_V_W1V] : nullptr; a.nv1m = nx ? nx + L.off[DISTEGNN_P_V_W1M] : nullptr;
    a.nvb1 = nx ? nx + L.off[DISTEGNN_P_V_B1] : nullptr;
    a.g_Xn = g_Xn; a.g_Hn = g_Hn; a.g_G = g_G; a.g_vsum = g_vsum; a.g_Xv = g_Xv; a.g_Hv = g_Hv;
    float* d = g_layer_params;
    a.d_m1 = d ? d + L.off[DISTEGNN_P_M_W1] : nullptr; a.d_mb1 = d ? d + L.off[DISTEGNN_P_M_B1] : nullptr;
    a.d_m2 = d ? d + L.off[DISTEGNN_P_M_W2] : nullptr; a.d_mb2 = d ? d + L.off[DISTEGNN_P_M_B2] : nullptr;
    float* dn = g_next_layer_params;
    a.d_nv1v = dn ? dn + L.off[DISTEGNN_P_V_W1V] : nullptr; a.d_nv1m = dn ? dn + L.off[DISTEGNN_P_V_W1M] : nullptr;
    a.d_nvb1 = dn ? dn + L.off[DISTEGNN_P_V_B1] : nullptr;
    virtual_update_bwd_kernel<<<(unsigned)n_graphs, NTHREADS, 0, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
