// Backward of the per-node stage and of the embedding prologue (SURVEY §8 f-1) — hand-written, fp32 FMA tile GEMMs.
//
// Forward (distegnn_node_layer_fwd; reference models/FastEGNN.py:177-183 coord tail, 203-217 node_model, plus the next
// layer's first-layer projections that this implementation evaluates per node):
//   φ_v = L_W3·SiLU(h·L_W + L_B) + L_B3                 x' = x + agg_x/deg + trans_v + φ_v·vel
//   z = [h | agg_m/deg | agg_v | attr]·N_W1 + N_B1     h' = h + SiLU(z)·N_W2 + N_B2
//   P' = h'·W1A' + B1',  Q' = h'·W1B',  Hn' = h'·W1H'   (the NEXT layer's blocks)
// Backward, per tile of 128 nodes (everything recomputed from the N-sized tensors the forward keeps; 5 tiles of shared
// memory; the eight 64x64 weight gradients accumulate in registers over all tiles of a CTA and are flushed once):
//   g_h' += g_P'·W1A'ᵀ + g_Q'·W1B'ᵀ + g_Hn'·W1H'ᵀ        g_z = (g_h'·N_W2ᵀ) ⊙ SiLU'(z)
//   [g_h | g_agg_m·deg | g_agg_v | ·] = g_z·N_W1ᵀ         g_u = (g_x'·vel)·L_W3 ⊙ SiLU'(u),  g_h += g_u·L_Wᵀ + g_h'
//   g_x = g_trans_v = g_x',  g_agg_x = g_x'/deg
// The embedding prologue (FastEGNN.py:302 + layer-0 projections) is the same first line followed by
// g_W_emb = featᵀ·g_h0, g_b_emb = Σ g_h0 (distegnn_embed_bwd).  Replaces torch recompute + autograd on cuBLAS.
#include <string.h>

#include "bwd_common.cuh"
#include "common.cuh"

namespace degnn {

struct NodeBwdArgs {
    int64_t N;
    int Na;
    unsigned flags;
    const int32_t* rowptr;
    const float* h; const float* vel; const float* attr; const float* agg_m; const float* agg_v;
    // upstream gradients
    const float* g_xn;      // [N,3]  w.r.t. x' (direct part)
    const float* g_vsum;    // [B,K] or null: gradient of the packed statistics; [b,0:3] is Σ_i x'_i, i.e. adds to g_x'
    const int32_t* batch;   // [N] graph id per node (with g_vsum)
    int K;
    const float* g_hn;      // [N,64] w.r.t. h'  (null: zero)
    const float* g_P; const float* g_Q; const float* g_Hn;   // [N,64] w.r.t. the next layer's projections (null: zero)
    // parameters (this layer / next layer), k-major
    const float* lw; const float* lb; const float* lw3;
    const float* n1; const float* nb1; const float* n2; const float* nb2;
    const float* xa; const float* xb; const float* xh;          // next: E_W1A, E_W1B, V_W1H
    // outputs
    float* g_h; float* g_x; float* g_agg_x; float* g_trans_v; float* g_agg_m; float* g_agg_v;
    float* d_lw; float* d_lb; float* d_lw3; float* d_lb3;
    float* d_n1; float* d_nb1; float* d_n2; float* d_nb2;
    float* d_xa; float* d_xb1; float* d_xb; float* d_xh;        // next layer's block: E_W1A, E_B1, E_W1B, V_W1H
};

// Gradients with respect to the model's inputs (the kInputs instantiations; the <false> ones are the weights-only kernels)
struct InputGradArgs {
    // node stage, ACCUMULATED over the layers: g_vel += φ_v·g_x',  g_attr += g_z·N_W1[3H:3H+Na]ᵀ (not with FLAG_LAST)
    float* g_vel; float* g_attr;
    const float* lb3;        // L_B3 (φ_v's bias)
    // embedding prologue, WRITTEN: g_feat = g_h0·emb_wtᵀ,  g_loc = g_x0 + g_vsum0[batch, 0:3] (Σx of the initial x̄)
    float* g_feat; float* g_loc;
    const float* emb_wt; const int32_t* batch; const float* g_x0; const float* g_vsum0;
    int K;
};

constexpr int NB_TILE = TILE_M * LDA;                            // floats per tile
constexpr int NB_SMEM_BYTES = 5 * NB_TILE * 4 + 2 * TILE_M * 4 + 64;

// acc[i][j] += Σ_n As[ty+16i][n] · W[4tx+j][n]   (As · Wᵀ, W k-major [64][64] in global memory / L1)
__device__ __forceinline__ void gemm_tile_gt(float (&acc)[8][4], const float* As, const float* __restrict__ Wg, int ty, int tx) {
#pragma unroll 2
    for (int n4 = 0; n4 < 16; ++n4) {
        float4 w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = ldg4(Wg + (4 * tx + j) * H + 4 * n4);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 a = *reinterpret_cast<const float4*>(As + (ty + 16 * i) * LDA + 4 * n4);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                acc[i][j] = fmaf(a.x, w[j].x, fmaf(a.y, w[j].y, fmaf(a.z, w[j].z, fmaf(a.w, w[j].w, acc[i][j]))));
        }
    }
}
__device__ __forceinline__ void store_acc(float* T, const float (&acc)[8][4], int ty, int tx) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
        *reinterpret_cast<float4*>(T + (ty + 16 * i) * LDA + 4 * tx) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}
__device__ __forceinline__ void zero44(float (&a)[4][4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) a[i][j] = 0.f;
}
// column sum of a tile over its 128 rows (threads 0..63, one column each)
__device__ __forceinline__ float colsum(const float* T, int col) {
    float s = 0.f;
#pragma unroll 8
    for (int r = 0; r < TILE_M; ++r) s += T[r * LDA + col];
    return s;
}
// g_hn (acc) += g_P·XAᵀ + g_Q·XBᵀ + g_Hn·XHᵀ with the projections' weight / bias gradients; Thn = the h' tile, TA scratch
__device__ __forceinline__ void proj_backward(float (&acc)[8][4], const NodeBwdArgs& a, int64_t n0, int nvalid, float* TA,
                                              const float* Thn, float (&wxa)[4][4], float (&wxb)[4][4], float (&wxh)[4][4],
                                              float& bx, int tid, int ty, int tx) {
    const float* gs[3] = {a.g_P, a.g_Q, a.g_Hn};
    const float* ws[3] = {a.xa, a.xb, a.xh};
#pragma unroll
    for (int m = 0; m < 3; ++m) {
        __syncthreads();
        load_a_tile(TA, gs[m] + (size_t)n0 * H, nvalid, nullptr, tid);
        __syncthreads();
        gemm_tile_gt(acc, TA, ws[m], ty, tx);
        if (m == 0) {
            wgrad_tile(wxa, TA, Thn, tid);
            if (tid < H) bx += colsum(TA, tid);
        } else if (m == 1) {
            wgrad_tile(wxb, TA, Thn, tid);
        } else {
            wgrad_tile(wxh, TA, Thn, tid);
        }
    }
}

template <bool kInputs>
__global__ void __launch_bounds__(NTHREADS, 1) node_layer_bwd_kernel(const NodeBwdArgs a, const InputGradArgs in) {
    extern __shared__ __align__(16) float nb_smem[];
    float* TA = nb_smem;                 // operand tile (h, agg_m/deg, agg_v, upstream gradients)
    float* TZ = TA + NB_TILE;            // z, later u
    float* TT = TZ + NB_TILE;            // t = SiLU(z), later s = SiLU(u)
    float* THN = TT + NB_TILE;           // h'
    float* TG = THN + NB_TILE;           // gradient tile (g_h', g_z, g_u)
    float* sinv = TG + NB_TILE;          // [128] 1/max(deg,1)
    float* sgphi = sinv + TILE_M;        // [128] g_φv = g_x'·vel
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const bool last = a.flags & DISTEGNN_FLAG_LAST;
    const int Na = a.Na;

    float wN1a[4][4], wN1b[4][4], wN1c[4][4], wN2[4][4], wLW[4][4], wXA[4][4], wXB[4][4], wXH[4][4];
    zero44(wN1a); zero44(wN1b); zero44(wN1c); zero44(wN2); zero44(wLW); zero44(wXA); zero44(wXB); zero44(wXH);
    float bN1 = 0.f, bN2 = 0.f, bL = 0.f, bX = 0.f, dW3 = 0.f, dB3 = 0.f;       // per-column accumulators (tid < 64)

    const int64_t num_tiles = (a.N + TILE_M - 1) / TILE_M;
    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int64_t n0 = tile * TILE_M;
        const int nvalid = (int)min((int64_t)TILE_M, a.N - n0);
        __syncthreads();
        if (tid < TILE_M) {
            float inv = 0.f, gp = 0.f;
            float4 gx = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tid < nvalid) {
                const size_t node = (size_t)(n0 + tid);
                inv = 1.0f / (float)max(__ldg(a.rowptr + node + 1) - __ldg(a.rowptr + node), 1);
                gx = make_float4(__ldg(a.g_xn + node * 3), __ldg(a.g_xn + node * 3 + 1), __ldg(a.g_xn + node * 3 + 2), 0.f);
                if (a.g_vsum) {                                   // x' also feeds the per-graph Σ x' of the next layer
                    const float* gv = a.g_vsum + (size_t)__ldg(a.batch + node) * a.K;
                    gx.x += __ldg(gv); gx.y += __ldg(gv + 1); gx.z += __ldg(gv + 2);
                }
                gp = gx.x * __ldg(a.vel + node * 3) + gx.y * __ldg(a.vel + node * 3 + 1) + gx.z * __ldg(a.vel + node * 3 + 2);
                // coordinate path: x' = x + agg_x/deg + trans_v + φ_v·vel
                a.g_x[node * 3] = gx.x; a.g_x[node * 3 + 1] = gx.y; a.g_x[node * 3 + 2] = gx.z;
                *reinterpret_cast<float4*>(a.g_trans_v + node * 4) = gx;
                *reinterpret_cast<float4*>(a.g_agg_x + node * 4) = make_float4(gx.x * inv, gx.y * inv, gx.z * inv, 0.f);
            }
            sinv[tid] = inv;
            sgphi[tid] = gp;
        }
        float accH[8][4];                                         // g_h of the tile, built up over the three paths
        zero_acc(accH);

        if (!last) {
            // ---- recompute z, t = SiLU(z), h' ---------------------------------------------------------------------
            float acc[8][4];
            zero_acc(acc);
            const float* srcs[3] = {a.h, a.agg_m, a.agg_v};
#pragma unroll
            for (int m = 0; m < 3; ++m) {
                __syncthreads();
                load_a_tile(TA, srcs[m] + (size_t)n0 * H, nvalid, m == 1 ? sinv : nullptr, tid);
                __syncthreads();
                gemm_tile_g(acc, TA, a.n1 + (size_t)m * H * H, ty, tx);
            }
            {
                const float4 b = ldg4(a.nb1 + 4 * tx);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = ty + 16 * i;
                    float4 z = make_float4(acc[i][0] + b.x, acc[i][1] + b.y, acc[i][2] + b.z, acc[i][3] + b.w);
                    if (r < nvalid)
                        for (int k = 0; k < Na; ++k)
                            z = fma4(__ldg(a.attr + (size_t)(n0 + r) * Na + k), ldg4(a.n1 + (size_t)(3 * H + k) * H + 4 * tx), z);
                    *reinterpret_cast<float4*>(TZ + r * LDA + 4 * tx) = z;
                    *reinterpret_cast<float4*>(TT + r * LDA + 4 * tx) = silu4(z);
                }
            }
            __syncthreads();
            zero_acc(acc);
            gemm_tile_g(acc, TT, a.n2, ty, tx);
            {
                // h' = h + t·N_W2 + N_B2: the activation the next layer's projection weights see
                const float4 b2 = ldg4(a.nb2 + 4 * tx);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = ty + 16 * i;
                    float4 hv = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (r < nvalid) hv = ldg4(a.h + (size_t)(n0 + r) * H + 4 * tx);
                    *reinterpret_cast<float4*>(THN + r * LDA + 4 * tx) =
                        make_float4(hv.x + acc[i][0] + b2.x, hv.y + acc[i][1] + b2.y, hv.z + acc[i][2] + b2.z, hv.w + acc[i][3] + b2.w);
                }
            }
            // ---- g_h' = upstream + projections' data gradients; their weight gradients need the h' tile -----------
            float accG[8][4];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = ty + 16 * i;
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
                if (a.g_hn && r < nvalid) g = ldg4(a.g_hn + (size_t)(n0 + r) * H + 4 * tx);
                accG[i][0] = g.x; accG[i][1] = g.y; accG[i][2] = g.z; accG[i][3] = g.w;
            }
            if (a.g_P) proj_backward(accG, a, n0, nvalid, TA, THN, wXA, wXB, wXH, bX, tid, ty, tx);
            __syncthreads();
            store_acc(TG, accG, ty, tx);                          // TG = g_h'
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) accH[i][j] = accG[i][j];      // residual path: h' = h + ...
            __syncthreads();
            // ---- node MLP layer 2: g_t = g_h'·N_W2ᵀ, g_N_W2 += tᵀ·g_h', g_N_B2 += Σ g_h' ---------------------------
            wgrad_tile(wN2, TG, TT, tid);
            if (tid < H) bN2 += colsum(TG, tid);
            zero_acc(acc);
            gemm_tile_gt(acc, TG, a.n2, ty, tx);
            __syncthreads();
#pragma unroll
            for (int i = 0; i < 8; ++i) {                         // g_z = g_t ⊙ SiLU'(z) -> TG
                const int r = ty + 16 * i;
                const float4 z = *reinterpret_cast<const float4*>(TZ + r * LDA + 4 * tx);
                *reinterpret_cast<float4*>(TG + r * LDA + 4 * tx) =
                    make_float4(acc[i][0] * dsilu(z.x), acc[i][1] * dsilu(z.y), acc[i][2] * dsilu(z.z), acc[i][3] * dsilu(z.w));
            }
            __syncthreads();
            if (tid < H) {
                bN1 += colsum(TG, tid);
                for (int k = 0; k < Na; ++k) {                    // attr rows of N_W1: Σ_rows attr[row][k]·g_z[row][n]
                    float s = 0.f;
                    for (int r = 0; r < nvalid; ++r) s = fmaf(__ldg(a.attr + (size_t)(n0 + r) * Na + k), TG[r * LDA + tid], s);
                    atomicAdd(a.d_n1 + (size_t)(3 * H + k) * H + tid, s);
                }
            }
            if constexpr (kInputs) {                              // g_attr[r][k] += Σ_n g_z[r][n]·N_W1[3H+k][n]
                const int r = tid & (TILE_M - 1);
                if (in.g_attr && r < nvalid) {
                    for (int k = tid / TILE_M; k < Na; k += NTHREADS / TILE_M) {
                        const float* w = a.n1 + (size_t)(3 * H + k) * H;
                        float s = 0.f;
#pragma unroll 16
                        for (int n = 0; n < H; ++n) s = fmaf(TG[r * LDA + n], __ldg(w + n), s);
                        in.g_attr[(size_t)(n0 + r) * Na + k] += s;
                    }
                }
            }
            // ---- node MLP layer 1: [g_h | g_agg_m·deg | g_agg_v] = g_z·N_W1ᵀ, weight gradients per 64-row block --------
            gemm_tile_gt(accH, TG, a.n1, ty, tx);                 // block 0 lands in g_h
            __syncthreads();
            load_a_tile(TA, a.h + (size_t)n0 * H, nvalid, nullptr, tid);
            __syncthreads();
            wgrad_tile(wN1a, TG, TA, tid);
#pragma unroll
            for (int m = 1; m < 3; ++m) {
                zero_acc(acc);
                gemm_tile_gt(acc, TG, a.n1 + (size_t)m * H * H, ty, tx);
                float* dst = m == 1 ? a.g_agg_m : a.g_agg_v;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = ty + 16 * i;
                    if (r < nvalid) {
                        const float s = m == 1 ? sinv[r] : 1.0f;  // agg_m enters as agg_m/deg
                        *reinterpret_cast<float4*>(dst + (size_t)(n0 + r) * H + 4 * tx) =
                            make_float4(acc[i][0] * s, acc[i][1] * s, acc[i][2] * s, acc[i][3] * s);
                    }
                }
                __syncthreads();
                load_a_tile(TA, (m == 1 ? a.agg_m : a.agg_v) + (size_t)n0 * H, nvalid, m == 1 ? sinv : nullptr, tid);
                __syncthreads();
                if (m == 1) wgrad_tile(wN1b, TG, TA, tid);
                else wgrad_tile(wN1c, TG, TA, tid);
            }
        }
        // ---- velocity head: u = h·L_W + L_B, s = SiLU(u), φ_v = s·L_W3 + L_B3; g_φv = g_x'·vel ------------------------
        {
            float acc[8][4];
            __syncthreads();
            load_a_tile(TA, a.h + (size_t)n0 * H, nvalid, nullptr, tid);
            __syncthreads();
            zero_acc(acc);
            gemm_tile_g(acc, TA, a.lw, ty, tx);
            const float4 b = ldg4(a.lb + 4 * tx), w3 = ldg4(a.lw3 + 4 * tx);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = ty + 16 * i;
                const float gp = sgphi[r];
                const float4 u = make_float4(acc[i][0] + b.x, acc[i][1] + b.y, acc[i][2] + b.z, acc[i][3] + b.w);
                const float4 s = silu4(u);
                *reinterpret_cast<float4*>(TT + r * LDA + 4 * tx) = make_float4(s.x * gp, s.y * gp, s.z * gp, s.w * gp);   // for g_L_W3
                *reinterpret_cast<float4*>(TG + r * LDA + 4 * tx) =
                    make_float4(gp * w3.x * dsilu(u.x), gp * w3.y * dsilu(u.y), gp * w3.z * dsilu(u.z), gp * w3.w * dsilu(u.w));
            }
            if constexpr (kInputs) {                              // g_vel += φ_v·g_x'; φ_v summed over the 16 tx lanes
                if (in.g_vel) {
                    const float b3 = __ldg(in.lb3);
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int r = ty + 16 * i;
                        const float4 s = silu4(make_float4(acc[i][0] + b.x, acc[i][1] + b.y, acc[i][2] + b.z, acc[i][3] + b.w));
                        float p = s.x * w3.x + s.y * w3.y + s.z * w3.z + s.w * w3.w;
                        p += __shfl_xor_sync(FULL, p, 8);
                        p += __shfl_xor_sync(FULL, p, 4);
                        p += __shfl_xor_sync(FULL, p, 2);
                        p += __shfl_xor_sync(FULL, p, 1);
                        if (tx == 0 && r < nvalid) {
                            const size_t node = (size_t)(n0 + r);
                            float gx[3] = {__ldg(a.g_xn + node * 3), __ldg(a.g_xn + node * 3 + 1), __ldg(a.g_xn + node * 3 + 2)};
                            if (a.g_vsum) {
                                const float* gv = a.g_vsum + (size_t)__ldg(a.batch + node) * a.K;
                                gx[0] += __ldg(gv); gx[1] += __ldg(gv + 1); gx[2] += __ldg(gv + 2);
                            }
                            const float phi = p + b3;
                            for (int d = 0; d < 3; ++d) in.g_vel[node * 3 + d] += phi * gx[d];
                        }
                    }
                }
            }
            __syncthreads();
            if (tid < H) {
                dW3 += colsum(TT, tid);
                bL += colsum(TG, tid);
            }
            if (tid == 0) {
                float s = 0.f;
                for (int r = 0; r < nvalid; ++r) s += sgphi[r];
                dB3 += s;
            }
            wgrad_tile(wLW, TG, TA, tid);
            gemm_tile_gt(accH, TG, a.lw, ty, tx);                 // g_h += g_u·L_Wᵀ
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = ty + 16 * i;
            if (r < nvalid)
                *reinterpret_cast<float4*>(a.g_h + (size_t)(n0 + r) * H + 4 * tx) =
                    make_float4(accH[i][0], accH[i][1], accH[i][2], accH[i][3]);
        }
    }
    // ---- flush the per-CTA parameter gradients -----------------------------------------------------------------------
    wgrad_flush(a.d_lw, wLW, tid);
    if (tid < H) {
        atomicAdd(a.d_lb + tid, bL);
        atomicAdd(a.d_lw3 + tid, dW3);
    }
    if (tid == 0) atomicAdd(a.d_lb3, dB3);
    if (!last) {
        wgrad_flush(a.d_n1, wN1a, tid);
        wgrad_flush(a.d_n1 + (size_t)H * H, wN1b, tid);
        wgrad_flush(a.d_n1 + (size_t)2 * H * H, wN1c, tid);
        wgrad_flush(a.d_n2, wN2, tid);
        if (tid < H) {
            atomicAdd(a.d_nb1 + tid, bN1);
            atomicAdd(a.d_nb2 + tid, bN2);
        }
        if (a.g_P) {
            wgrad_flush(a.d_xa, wXA, tid);
            wgrad_flush(a.d_xb, wXB, tid);
            wgrad_flush(a.d_xh, wXH, tid);
            if (tid < H) atomicAdd(a.d_xb1 + tid, bX);
        }
    }
}

// ---- embedding prologue backward: g_h0 = g_h + projections; g_W_emb = featᵀ·g_h0, g_b_emb = Σ g_h0 -----------------
struct EmbedBwdArgs {
    NodeBwdArgs nb;          // uses: N, h (= h0), g_hn (= g_h), g_P, g_Q, g_Hn, xa, xb, xh, d_xa, d_xb1, d_xb, d_xh
    int F;
    const float* feat;       // [N,F]
    float* d_wt;             // [F][64]
    float* d_b;              // [64]
};

template <bool kInputs>
__global__ void __launch_bounds__(NTHREADS, 1) embed_bwd_kernel(const EmbedBwdArgs e, const InputGradArgs in) {
    extern __shared__ __align__(16) float nb_smem[];
    const NodeBwdArgs& a = e.nb;
    float* TA = nb_smem;
    float* THN = TA + NB_TILE;
    float* TG = THN + NB_TILE;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    float wXA[4][4], wXB[4][4], wXH[4][4];
    zero44(wXA); zero44(wXB); zero44(wXH);
    float bX = 0.f, bE = 0.f;
    float dwt[DISTEGNN_MAX_NODE_FEAT];
#pragma unroll
    for (int k = 0; k < DISTEGNN_MAX_NODE_FEAT; ++k) dwt[k] = 0.f;
    const int64_t num_tiles = (a.N + TILE_M - 1) / TILE_M;
    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int64_t n0 = tile * TILE_M;
        const int nvalid = (int)min((int64_t)TILE_M, a.N - n0);
        __syncthreads();
        load_a_tile(THN, a.h + (size_t)n0 * H, nvalid, nullptr, tid);
        float accG[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = ty + 16 * i;
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
            if (a.g_hn && r < nvalid) g = ldg4(a.g_hn + (size_t)(n0 + r) * H + 4 * tx);
            accG[i][0] = g.x; accG[i][1] = g.y; accG[i][2] = g.z; accG[i][3] = g.w;
        }
        proj_backward(accG, a, n0, nvalid, TA, THN, wXA, wXB, wXH, bX, tid, ty, tx);
        __syncthreads();
        store_acc(TG, accG, ty, tx);
        __syncthreads();
        if constexpr (kInputs) {
            const int r = tid & (TILE_M - 1);
            if (in.g_feat && r < nvalid) {                        // g_feat[r][k] = Σ_n g_h0[r][n]·emb_wt[k][n]
                for (int k = tid / TILE_M; k < e.F; k += NTHREADS / TILE_M) {
                    const float* w = in.emb_wt + (size_t)k * H;
                    float s = 0.f;
#pragma unroll 16
                    for (int n = 0; n < H; ++n) s = fmaf(TG[r * LDA + n], __ldg(w + n), s);
                    in.g_feat[(size_t)(n0 + r) * e.F + k] = s;
                }
            }
            if (in.g_loc && tid < nvalid) {                       // layer 0's x is node_loc; Σx feeds the initial x̄
                const size_t node = (size_t)(n0 + tid);
                const float* gv = in.g_vsum0 ? in.g_vsum0 + (size_t)__ldg(in.batch + node) * in.K : nullptr;
                for (int d = 0; d < 3; ++d) in.g_loc[node * 3 + d] = __ldg(in.g_x0 + node * 3 + d) + (gv ? __ldg(gv + d) : 0.f);
            }
        }
        if (tid < H) {
            bE += colsum(TG, tid);
            for (int r = 0; r < nvalid; ++r) {
                const float g = TG[r * LDA + tid];
#pragma unroll
                for (int k = 0; k < DISTEGNN_MAX_NODE_FEAT; ++k)
                    if (k < e.F) dwt[k] = fmaf(__ldg(e.feat + (size_t)(n0 + r) * e.F + k), g, dwt[k]);
            }
        }
    }
    wgrad_flush(a.d_xa, wXA, tid);
    wgrad_flush(a.d_xb, wXB, tid);
    wgrad_flush(a.d_xh, wXH, tid);
    if (tid < H) {
        atomicAdd(a.d_xb1 + tid, bX);
        atomicAdd(e.d_b + tid, bE);
#pragma unroll
        for (int k = 0; k < DISTEGNN_MAX_NODE_FEAT; ++k)
            if (k < e.F) atomicAdd(e.d_wt + (size_t)k * H + tid, dwt[k]);
    }
}

static int node_layer_bwd_launch(int64_t n_nodes, int A, int C, int Na, unsigned flags, const int32_t* rowptr,
                                 const float* h, const float* node_vel, const float* node_attr, const float* agg_m,
                                 const float* agg_v, const float* layer_params, const float* next_layer_params,
                                 const float* g_x_out, const float* g_vsum, const int32_t* batch32, const float* g_h_out,
                                 const float* g_P, const float* g_Q, const float* g_Hn, float* g_h, float* g_x, float* g_agg_x,
                                 float* g_trans_v, float* g_agg_m, float* g_agg_v, float* g_layer_params,
                                 float* g_next_layer_params, float* g_node_vel, float* g_node_attr, void* stream) {
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    const bool last = flags & DISTEGNN_FLAG_LAST;
    DEGNN_CHECK_ARG(n_nodes > 0, "bad size");
    DEGNN_CHECK_ARG(rowptr && h && node_vel && layer_params && g_x_out && g_h && g_x && g_agg_x && g_trans_v && g_layer_params,
                    "null pointer");
    DEGNN_CHECK_ARG(Na == 0 || node_attr || last, "null node_attr with node_attr_nf > 0");
    DEGNN_CHECK_ARG(last || (agg_m && agg_v && g_agg_m && g_agg_v), "null pointer (non-last layer)");
    DEGNN_CHECK_ARG(!g_P || (g_Q && g_Hn && next_layer_params && g_next_layer_params),
                    "g_P needs g_Q, g_Hn and the next layer's parameter / gradient blocks");
    Layout L = make_layout(A, C, Na);
    NodeBwdArgs a;
    a.N = n_nodes; a.Na = Na; a.flags = flags; a.rowptr = rowptr;
    a.h = h; a.vel = node_vel; a.attr = node_attr; a.agg_m = agg_m; a.agg_v = agg_v;
    DEGNN_CHECK_ARG(!g_vsum || batch32, "g_vsum needs batch32");
    a.g_xn = g_x_out; a.g_vsum = g_vsum; a.batch = batch32; a.K = 4 + 3 * C + H * C;
    a.g_hn = last ? nullptr : g_h_out; a.g_P = last ? nullptr : g_P; a.g_Q = g_Q; a.g_Hn = g_Hn;
    const float* lp = layer_params;
    a.lw = lp + L.off[DISTEGNN_P_L_W]; a.lb = lp + L.off[DISTEGNN_P_L_B]; a.lw3 = lp + L.off[DISTEGNN_P_L_W3];
    a.n1 = lp + L.off[DISTEGNN_P_N_W1]; a.nb1 = lp + L.off[DISTEGNN_P_N_B1]; a.n2 = lp + L.off[DISTEGNN_P_N_W2];
    a.nb2 = lp + L.off[DISTEGNN_P_N_B2];
    const float* nx = next_layer_params;
    a.xa = nx ? nx + L.off[DISTEGNN_P_E_W1A] : nullptr;
    a.xb = nx ? nx + L.off[DISTEGNN_P_E_W1B] : nullptr;
    a.xh = nx ? nx + L.off[DISTEGNN_P_V_W1H] : nullptr;
    a.g_h = g_h; a.g_x = g_x; a.g_agg_x = g_agg_x; a.g_trans_v = g_trans_v; a.g_agg_m = g_agg_m; a.g_agg_v = g_agg_v;
    float* d = g_layer_params;
    a.d_lw = d + L.off[DISTEGNN_P_L_W]; a.d_lb = d + L.off[DISTEGNN_P_L_B]; a.d_lw3 = d + L.off[DISTEGNN_P_L_W3];
    a.d_lb3 = d + L.off[DISTEGNN_P_L_B3];
    a.d_n1 = d + L.off[DISTEGNN_P_N_W1]; a.d_nb1 = d + L.off[DISTEGNN_P_N_B1]; a.d_n2 = d + L.off[DISTEGNN_P_N_W2];
    a.d_nb2 = d + L.off[DISTEGNN_P_N_B2];
    float* dn = g_next_layer_params;
    a.d_xa = dn ? dn + L.off[DISTEGNN_P_E_W1A] : nullptr;
    a.d_xb1 = dn ? dn + L.off[DISTEGNN_P_E_B1] : nullptr;
    a.d_xb = dn ? dn + L.off[DISTEGNN_P_E_W1B] : nullptr;
    a.d_xh = dn ? dn + L.off[DISTEGNN_P_V_W1H] : nullptr;
    InputGradArgs in;
    memset(&in, 0, sizeof(in));
    in.g_vel = g_node_vel;
    in.g_attr = (Na > 0 && !last) ? g_node_attr : nullptr;       // the last layer has no node MLP: no attr term
    in.lb3 = lp + L.off[DISTEGNN_P_L_B3];
    const bool inputs = in.g_vel || in.g_attr;
    const void* kernel = inputs ? (const void*)node_layer_bwd_kernel<true> : (const void*)node_layer_bwd_kernel<false>;
    ensure_dynamic_smem(kernel, (int)NB_SMEM_BYTES);
    const int64_t tiles = (n_nodes + TILE_M - 1) / TILE_M;
    int64_t grid = sm_count();
    if (grid > tiles) grid = tiles;
    if (inputs)
        node_layer_bwd_kernel<true><<<(unsigned)grid, NTHREADS, NB_SMEM_BYTES, (cudaStream_t)stream>>>(a, in);
    else
        node_layer_bwd_kernel<false><<<(unsigned)grid, NTHREADS, NB_SMEM_BYTES, (cudaStream_t)stream>>>(a, in);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

static int embed_bwd_launch(int64_t n_nodes, int F, int A, int C, int Na, const float* node_feat, const float* h0,
                            const float* layer0_params, const float* g_h, const float* g_P, const float* g_Q,
                            const float* g_Hn, float* g_emb_wt, float* g_emb_b, float* g_layer0_params, const float* emb_wt,
                            const int32_t* batch32, const float* g_x0, const float* g_vsum0, float* g_node_feat,
                            float* g_node_loc, void* stream) {
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && F >= 1 && F <= DISTEGNN_MAX_NODE_FEAT, "bad size");
    DEGNN_CHECK_ARG(node_feat && h0 && layer0_params && g_P && g_Q && g_Hn && g_emb_wt && g_emb_b && g_layer0_params,
                    "null pointer");
    DEGNN_CHECK_ARG(!g_node_feat || emb_wt, "g_node_feat needs emb_wt");
    DEGNN_CHECK_ARG(!g_node_loc || g_x0, "g_node_loc needs g_x0");
    DEGNN_CHECK_ARG(!g_node_loc || !g_vsum0 || batch32, "g_vsum0 needs batch32");
    Layout L = make_layout(A, C, Na);
    EmbedBwdArgs e;
    memset(&e, 0, sizeof(e));
    e.nb.N = n_nodes; e.nb.h = h0; e.nb.g_hn = g_h; e.nb.g_P = g_P; e.nb.g_Q = g_Q; e.nb.g_Hn = g_Hn;
    e.nb.xa = layer0_params + L.off[DISTEGNN_P_E_W1A];
    e.nb.xb = layer0_params + L.off[DISTEGNN_P_E_W1B];
    e.nb.xh = layer0_params + L.off[DISTEGNN_P_V_W1H];
    e.nb.d_xa = g_layer0_params + L.off[DISTEGNN_P_E_W1A];
    e.nb.d_xb1 = g_layer0_params + L.off[DISTEGNN_P_E_B1];
    e.nb.d_xb = g_layer0_params + L.off[DISTEGNN_P_E_W1B];
    e.nb.d_xh = g_layer0_params + L.off[DISTEGNN_P_V_W1H];
    e.F = F; e.feat = node_feat; e.d_wt = g_emb_wt; e.d_b = g_emb_b;
    InputGradArgs in;
    memset(&in, 0, sizeof(in));
    in.g_feat = g_node_feat; in.g_loc = g_node_loc; in.emb_wt = emb_wt; in.batch = batch32; in.g_x0 = g_x0;
    in.g_vsum0 = g_vsum0; in.K = 4 + 3 * C + H * C;
    const bool inputs = g_node_feat || g_node_loc;
    const int smem = 3 * NB_TILE * 4;
    const void* kernel = inputs ? (const void*)embed_bwd_kernel<true> : (const void*)embed_bwd_kernel<false>;
    ensure_dynamic_smem(kernel, smem);
    const int64_t tiles = (n_nodes + TILE_M - 1) / TILE_M;
    int64_t grid = sm_count();
    if (grid > tiles) grid = tiles;
    if (inputs)
        embed_bwd_kernel<true><<<(unsigned)grid, NTHREADS, smem, (cudaStream_t)stream>>>(e, in);
    else
        embed_bwd_kernel<false><<<(unsigned)grid, NTHREADS, smem, (cudaStream_t)stream>>>(e, in);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" int distegnn_node_layer_bwd(int64_t n_nodes, int A, int C, int Na, unsigned flags, const int32_t* rowptr,
                                       const float* h, const float* node_vel, const float* node_attr, const float* agg_m,
                                       const float* agg_v, const float* layer_params, const float* next_layer_params,
                                       const float* g_x_out, const float* g_vsum, const int32_t* batch32, const float* g_h_out,
                                       const float* g_P, const float* g_Q, const float* g_Hn, float* g_h, float* g_x, float* g_agg_x, float* g_trans_v,
                                       float* g_agg_m, float* g_agg_v, float* g_layer_params, float* g_next_layer_params,
                                       void* stream) {
    return degnn::node_layer_bwd_launch(n_nodes, A, C, Na, flags, rowptr, h, node_vel, node_attr, agg_m, agg_v,
                                        layer_params, next_layer_params, g_x_out, g_vsum, batch32, g_h_out, g_P, g_Q, g_Hn,
                                        g_h, g_x, g_agg_x, g_trans_v, g_agg_m, g_agg_v, g_layer_params,
                                        g_next_layer_params, nullptr, nullptr, stream);
}

extern "C" int distegnn_node_layer_bwd_inputs(int64_t n_nodes, int A, int C, int Na, unsigned flags, const int32_t* rowptr,
                                              const float* h, const float* node_vel, const float* node_attr,
                                              const float* agg_m, const float* agg_v, const float* layer_params,
                                              const float* next_layer_params, const float* g_x_out, const float* g_vsum,
                                              const int32_t* batch32, const float* g_h_out, const float* g_P,
                                              const float* g_Q, const float* g_Hn, float* g_h, float* g_x, float* g_agg_x,
                                              float* g_trans_v, float* g_agg_m, float* g_agg_v, float* g_layer_params,
                                              float* g_next_layer_params, float* g_node_vel, float* g_node_attr,
                                              void* stream) {
    return degnn::node_layer_bwd_launch(n_nodes, A, C, Na, flags, rowptr, h, node_vel, node_attr, agg_m, agg_v,
                                        layer_params, next_layer_params, g_x_out, g_vsum, batch32, g_h_out, g_P, g_Q, g_Hn,
                                        g_h, g_x, g_agg_x, g_trans_v, g_agg_m, g_agg_v, g_layer_params,
                                        g_next_layer_params, g_node_vel, g_node_attr, stream);
}

extern "C" int distegnn_embed_bwd(int64_t n_nodes, int F, int A, int C, int Na, const float* node_feat, const float* h0,
                                  const float* layer0_params, const float* g_h, const float* g_P, const float* g_Q,
                                  const float* g_Hn, float* g_emb_wt, float* g_emb_b, float* g_layer0_params, void* stream) {
    return degnn::embed_bwd_launch(n_nodes, F, A, C, Na, node_feat, h0, layer0_params, g_h, g_P, g_Q, g_Hn, g_emb_wt,
                                   g_emb_b, g_layer0_params, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int distegnn_embed_bwd_inputs(int64_t n_nodes, int F, int A, int C, int Na, const float* node_feat,
                                         const float* h0, const float* layer0_params, const float* g_h, const float* g_P,
                                         const float* g_Q, const float* g_Hn, float* g_emb_wt, float* g_emb_b,
                                         float* g_layer0_params, const float* emb_wt, const int32_t* batch32,
                                         const float* g_x0, const float* g_vsum0, float* g_node_feat, float* g_node_loc,
                                         void* stream) {
    return degnn::embed_bwd_launch(n_nodes, F, A, C, Na, node_feat, h0, layer0_params, g_h, g_P, g_Q, g_Hn, g_emb_wt,
                                   g_emb_b, g_layer0_params, emb_wt, batch32, g_x0, g_vsum0, g_node_feat, g_node_loc,
                                   stream);
}
