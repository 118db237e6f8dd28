// Shared device code for the DistEGNN sm_90a kernels: the 128x64x64 fp32 tile GEMM every fused
// stage is built from, SiLU, parameter-block offsets, error plumbing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/distegnn_b200.h"

namespace degnn {

constexpr int H = 64;          // hidden width
constexpr int TILE_M = 128;    // rows (edges / node·channel pairs / nodes) per CTA tile
constexpr int LDA = 68;        // smem leading dimension of an activation tile (floats); 68 = 64+4 keeps
                               // float4 alignment and shifts consecutive rows by 4 banks
constexpr int NTHREADS = 256;  // 16 (ty) x 16 (tx); thread owns rows ty+16*i (i<8), cols 4*tx..4*tx+3
constexpr unsigned FULL = 0xffffffffu;

// ---- host side: error string + parameter layout ------------------------------------------------
void set_error(const char* fmt, ...);
struct Layout {
    int64_t off[DISTEGNN_P_NUM_FIELDS];
    int64_t total;
};
Layout make_layout(int A, int C, int Na);
int check_dims(int A, int C, int Na);

#define DEGNN_CHECK_ARG(cond, msg)                                  \
    do {                                                            \
        if (!(cond)) {                                              \
            ::degnn::set_error("%s: %s", __func__, msg);            \
            return DISTEGNN_EINVAL;                                 \
        }                                                           \
    } while (0)

#define DEGNN_CHECK_LAUNCH()                                                             \
    do {                                                                                 \
        cudaError_t e__ = cudaPeekAtLastError();                                         \
        if (e__ != cudaSuccess) {                                                        \
            ::degnn::set_error("%s: CUDA error: %s", __func__, cudaGetErrorString(e__)); \
            return DISTEGNN_ECUDA;                                                       \
        }                                                                                \
    } while (0)

int sm_count();   // cached multiprocessor count of the current device
// Opt `kernel` in to `bytes` of dynamic shared memory, once per (device, kernel).  Not a stream operation, so it is
// done on the first (eager) call and never again — nothing but launches happens under CUDA-graph capture.
void ensure_dynamic_smem(const void* kernel, int bytes);

// ---- device helpers -----------------------------------------------------------------------------
__device__ __forceinline__ float silu(float x) {
    // x·σ(x) = x · rcp(1 + 2^{-x·log2 e}): FMUL, MUFU.EX2, FADD, MUFU.RCP, FMUL — no range fix-ups needed:
    // x → −∞ gives 2^{+big} = inf, rcp(inf) = 0, x·0 = −0;  x → +∞ gives rcp(1) = 1.  |rel err| ≲ 5e-7.
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
}
__device__ __forceinline__ float4 silu4(float4 v) {
    return make_float4(silu(v.x), silu(v.y), silu(v.z), silu(v.w));
}

// ---- fp32 register pairs --------------------------------------------------------------------------------------------
// The elementwise chains around the MMAs work on register PAIRS (f32x2: two fp32 in one 64-bit value, even column in the
// low half) so that they line up with the packed fp16 words of the A operand.  sm_90 has no packed fp32 instructions:
// add2 / sub2 / mul2 / fma2 are two scalar round-to-nearest operations each.  The SiLU of the pair chains takes one
// reciprocal per FOUR activations:  1/d_i = d_j·d_k·d_l / (d_0 d_1 d_2 d_3)  (5 MUFU per 4 instead of 8; falls back to
// 4 RCPs when the product leaves the fp32 range, i.e. some x < about −21)
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk2(float lo, float hi) {
    f32x2 r;
    asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ f32x2 pk2u(uint32_t lo, uint32_t hi) {
    f32x2 r;
    asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "r"(lo), "r"(hi));
    return r;
}
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
    asm("mov.b64 {%0,%1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ f32x2 bc2(float x) { return pk2(x, x); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1)); }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1)); }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
    float a0, a1, b0, b1, c0, c1; upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
    return pk2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ float ex2_approx(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
// d = 1 + 2^{-x·log2 e} for a pair
__device__ __forceinline__ f32x2 silu_den2(f32x2 x) {
    float t0, t1;
    upk2(mul2(x, bc2(-1.4426950408889634f)), t0, t1);
    return add2(pk2(ex2_approx(t0), ex2_approx(t1)), bc2(1.0f));
}
__device__ __forceinline__ f32x2 rcp2(f32x2 d) {
    float d0, d1;
    upk2(d, d0, d1);
    return pk2(rcp_approx(d0), rcp_approx(d1));
}
__device__ __forceinline__ f32x2 silu2(f32x2 x) { return mul2(x, rcp2(silu_den2(x))); }
// Four activations (two pairs) at once.  The caller owns the range guard: `qmax` accumulates the largest
// product d0·d1·d2·d3 seen; if silu_q_overflow(qmax) the results of that batch are invalid (1/q is not a normal
// number: some x < about −21) and must be recomputed with SAFE = true, which is the per-element-reciprocal form.
// A guard per quad would either be if-converted by ptxas into predicated MUFUs on the hot path or, as a real
// branch, serialise the quads — so it is hoisted to once per stage, next to the fp16-range rescue.
constexpr float SILU_Q_LIMIT = 8.0e37f;
__device__ __forceinline__ bool silu_q_overflow(float qmax) { return !(qmax < SILU_Q_LIMIT); }
template <bool SAFE>
__device__ __forceinline__ void silu4p(f32x2& a, f32x2& b, float& qmax) {
    if (SAFE) {
        a = silu2(a);
        b = silu2(b);
        return;
    }
    const f32x2 da = silu_den2(a), db = silu_den2(b);        // (d0,d1), (d2,d3), every d in [1, inf]
    const f32x2 p = mul2(da, db);                             // (d0 d2, d1 d3)
    float p0, p1;
    upk2(p, p0, p1);
    const float q = p0 * p1;
    qmax = fmaxf(qmax, q);
    const float r = rcp_approx(q);
    const f32x2 u = pk2(r * p1, r * p0);                      // (1/(d0 d2), 1/(d1 d3)): two scalar FMULs land in a
                                                              // register pair directly (a packed form needs 3 MOVs)
    a = mul2(a, mul2(u, db));                                 // x · (1/d0, 1/d1)
    b = mul2(b, mul2(u, da));                                 // x · (1/d2, 1/d3)
}
// The same in the "t domain": the inputs are t = −log2(e)·x (the producer folds the factor into its weights / biases), the
// outputs s = t / (1 + 2^t) = −log2(e)·SiLU(x) — the consumer folds −ln 2 into whatever multiplies s next.  Saves the
// multiply per element that forms the exponent argument.
constexpr float SILU_T_IN = -1.4426950408889634f;    // t = SILU_T_IN · x
constexpr float SILU_T_OUT = -0.6931471805599453f;   // SiLU(x) = SILU_T_OUT · s
__device__ __forceinline__ f32x2 silu_den2_t(f32x2 t) {
    float t0, t1;
    upk2(t, t0, t1);
    return add2(pk2(ex2_approx(t0), ex2_approx(t1)), bc2(1.0f));
}
template <bool SAFE>
__device__ __forceinline__ void silu4t(f32x2& a, f32x2& b, float& qmax) {
    const f32x2 da = silu_den2_t(a), db = silu_den2_t(b);
    if (SAFE) {
        a = mul2(a, rcp2(da));
        b = mul2(b, rcp2(db));
        return;
    }
    const f32x2 p = mul2(da, db);
    float p0, p1;
    upk2(p, p0, p1);
    const float q = p0 * p1;
    qmax = fmaxf(qmax, q);
    const float r = rcp_approx(q);
    const f32x2 u = pk2(r * p1, r * p0);
    a = mul2(a, mul2(u, db));
    b = mul2(b, mul2(u, da));
}
__device__ __forceinline__ float4 ldg4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
// The fp32 squared edge length, the one expression behind every edge length on the device: the radius build's fill pass
// (d2 < r2, edge_attr = sqrtf(d2)), the rollout's edge lengths and their backward, and the cutoff's keys.  They must
// agree bit for bit: the differentiable rollout's backward rebuilds each step's graph and checks its edge count, and the
// cutoff ranks edges by keys that must equal the build's edge_attr.
__device__ __forceinline__ float edge_len2(float dx, float dy, float dz) { return dx * dx + dy * dy + dz * dz; }
// pos[i] − pos[j] of pos [N,3]
__device__ __forceinline__ void edge_delta(const float* pos, int i, int j, float& dx, float& dy, float& dz) {
    dx = __ldg(pos + (int64_t)i * 3) - __ldg(pos + (int64_t)j * 3);
    dy = __ldg(pos + (int64_t)i * 3 + 1) - __ldg(pos + (int64_t)j * 3 + 1);
    dz = __ldg(pos + (int64_t)i * 3 + 2) - __ldg(pos + (int64_t)j * 3 + 2);
}
__device__ __forceinline__ float4 fma4(float s, float4 w, float4 a) {
    return make_float4(fmaf(s, w.x, a.x), fmaf(s, w.y, a.y), fmaf(s, w.z, a.z), fmaf(s, w.w, a.w));
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

// Copy a k-major [64][64] weight chunk global -> smem (16 KB, 4 float4 per thread).
__device__ __forceinline__ void load_w64(float* Ws, const float* __restrict__ Wg, int tid) {
    const float4* g = reinterpret_cast<const float4*>(Wg);
    float4* s = reinterpret_cast<float4*>(Ws);
#pragma unroll
    for (int i = 0; i < 4; ++i) s[tid + NTHREADS * i] = __ldg(g + tid + NTHREADS * i);
}

// Copy a [rows<=128][64] fp32 row block (row stride 64) global -> As (row stride LDA), optionally
// scaling row r by scale[r] (smem array) — used for agg_m / max(deg,1).  Rows >= rows_valid zeroed.
__device__ __forceinline__ void load_a_tile(float* As, const float* __restrict__ src, int rows_valid,
                                            const float* row_scale, int tid) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int idx = tid + NTHREADS * i;   // 0..2047 float4 slots: row = idx/16, quad = idx%16
        int r = idx >> 4, q = idx & 15;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < rows_valid) {
            v = ldg4(src + (size_t)r * H + 4 * q);
            if (row_scale) {
                float s = row_scale[r];
                v.x *= s; v.y *= s; v.z *= s; v.w *= s;
            }
        }
        *reinterpret_cast<float4*>(As + r * LDA + 4 * q) = v;
    }
}

__device__ __forceinline__ void zero_acc(float (&acc)[8][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
}

// acc[i][j] += Σ_k As[ty+16i][k] · Ws[k][4tx+j]   (128x64 tile, K=64, fp32 FMA)
__device__ __forceinline__ void gemm_tile(float (&acc)[8][4], const float* As, const float* Ws, int ty,
                                          int tx) {
#pragma unroll 2
    for (int k4 = 0; k4 < 16; ++k4) {
        float4 w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            w[j] = *reinterpret_cast<const float4*>(Ws + (4 * k4 + j) * H + 4 * tx);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float4 a = *reinterpret_cast<const float4*>(As + (ty + 16 * i) * LDA + 4 * k4);
            acc[i][0] = fmaf(a.x, w[0].x, acc[i][0]);
            acc[i][1] = fmaf(a.x, w[0].y, acc[i][1]);
            acc[i][2] = fmaf(a.x, w[0].z, acc[i][2]);
            acc[i][3] = fmaf(a.x, w[0].w, acc[i][3]);
            acc[i][0] = fmaf(a.y, w[1].x, acc[i][0]);
            acc[i][1] = fmaf(a.y, w[1].y, acc[i][1]);
            acc[i][2] = fmaf(a.y, w[1].z, acc[i][2]);
            acc[i][3] = fmaf(a.y, w[1].w, acc[i][3]);
            acc[i][0] = fmaf(a.z, w[2].x, acc[i][0]);
            acc[i][1] = fmaf(a.z, w[2].y, acc[i][1]);
            acc[i][2] = fmaf(a.z, w[2].z, acc[i][2]);
            acc[i][3] = fmaf(a.z, w[2].w, acc[i][3]);
            acc[i][0] = fmaf(a.w, w[3].x, acc[i][0]);
            acc[i][1] = fmaf(a.w, w[3].y, acc[i][1]);
            acc[i][2] = fmaf(a.w, w[3].z, acc[i][2]);
            acc[i][3] = fmaf(a.w, w[3].w, acc[i][3]);
        }
    }
}

// same with the [64][64] weight matrix read straight from global memory (L1/L2 resident, 16 KB): used by the backward
// kernels, whose shared memory is taken by activation / gradient tiles
__device__ __forceinline__ void gemm_tile_g(float (&acc)[8][4], const float* As, const float* __restrict__ Wg, int ty,
                                            int tx) {
#pragma unroll 2
    for (int k4 = 0; k4 < 16; ++k4) {
        float4 w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = ldg4(Wg + (4 * k4 + j) * H + 4 * tx);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float4 a = *reinterpret_cast<const float4*>(As + (ty + 16 * i) * LDA + 4 * k4);
            acc[i][0] = fmaf(a.x, w[0].x, acc[i][0]); acc[i][1] = fmaf(a.x, w[0].y, acc[i][1]);
            acc[i][2] = fmaf(a.x, w[0].z, acc[i][2]); acc[i][3] = fmaf(a.x, w[0].w, acc[i][3]);
            acc[i][0] = fmaf(a.y, w[1].x, acc[i][0]); acc[i][1] = fmaf(a.y, w[1].y, acc[i][1]);
            acc[i][2] = fmaf(a.y, w[1].z, acc[i][2]); acc[i][3] = fmaf(a.y, w[1].w, acc[i][3]);
            acc[i][0] = fmaf(a.z, w[2].x, acc[i][0]); acc[i][1] = fmaf(a.z, w[2].y, acc[i][1]);
            acc[i][2] = fmaf(a.z, w[2].z, acc[i][2]); acc[i][3] = fmaf(a.z, w[2].w, acc[i][3]);
            acc[i][0] = fmaf(a.w, w[3].x, acc[i][0]); acc[i][1] = fmaf(a.w, w[3].y, acc[i][1]);
            acc[i][2] = fmaf(a.w, w[3].z, acc[i][2]); acc[i][3] = fmaf(a.w, w[3].w, acc[i][3]);
        }
    }
}

// act = SiLU(acc + bias) written back to the activation tile (the A operand of the next GEMM).
// Caller must __syncthreads() before (all reads of As done) and after.
__device__ __forceinline__ void bias_silu_to_tile(const float (&acc)[8][4], float4 b, float* As, int ty,
                                                  int tx) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float4 v = make_float4(silu(acc[i][0] + b.x), silu(acc[i][1] + b.y), silu(acc[i][2] + b.z),
                               silu(acc[i][3] + b.w));
        *reinterpret_cast<float4*>(As + (ty + 16 * i) * LDA + 4 * tx) = v;
    }
}

// 1-wide head: out[row] = Σ_col w3[col]·SiLU(acc[row][col] + b[col]); reduced over the 16 tx lanes,
// lane tx==0 stores to dst[row] (smem).
__device__ __forceinline__ void head_dot_to_smem(const float (&acc)[8][4], float4 b, float4 w3,
                                                 float* dst, int ty, int tx) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float v = silu(acc[i][0] + b.x) * w3.x;
        v = fmaf(silu(acc[i][1] + b.y), w3.y, v);
        v = fmaf(silu(acc[i][2] + b.z), w3.z, v);
        v = fmaf(silu(acc[i][3] + b.w), w3.w, v);
        v += __shfl_xor_sync(FULL, v, 1);
        v += __shfl_xor_sync(FULL, v, 2);
        v += __shfl_xor_sync(FULL, v, 4);
        v += __shfl_xor_sync(FULL, v, 8);
        if (tx == 0) dst[ty + 16 * i] = v;
    }
}

}  // namespace degnn
