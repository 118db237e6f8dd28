// The row rules of the tensor-core backward kernels (edge_layer_bwd_tc.cuh, virtual_layer_bwd_tc.cu), each in one place:
// a thread owns one row of a 128-row tile and holds the whole 64-wide row in registers.
#pragma once
#include <cuda_fp16.h>

#include "bwd_common.cuh"
#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

__device__ __forceinline__ float row_absmax(const float (&v)[64], float fm = 0.f) {
#pragma unroll
    for (int j = 0; j < 64; ++j) fm = fmaxf(fm, fabsf(v[j]));
    return fm;
}
// power-of-two scale that brings a row maximum `fm` into [2^13, 2^14) (rows of zeros / non-finite maxima keep 1) + inverse
__device__ __forceinline__ void row_scale(float fm, float& s, float& inv) {
    const uint32_t eb = (__float_as_uint(fm) >> 23) & 0xffu;
    const bool live = eb > 0u && eb < 255u;
    const uint32_t sb = live ? min(max(267u - eb, 1u), 254u) : 127u;        // biased exponent of the scale
    s = __uint_as_float(sb << 23);
    inv = __uint_as_float((254u - sb) << 23);
}
// Encode a whole 64-wide row held in registers, times the power-of-two `s`, into the A operand.
__device__ __forceinline__ void encode_row(const float (&v)[64], float s, uint32_t ta_hi, uint32_t ta_lo) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        uint32_t hi[8], lo[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            tc16::split_pair(mul2(pk2(v[16 * c + 2 * j], v[16 * c + 2 * j + 1]), bc2(s)), hi[j], lo[j]);
        tmma::tm_st8(ta_hi + 8 * c, hi);
        tmma::tm_st8(ta_lo + 8 * c, lo);
    }
}
// The same with the row's own power-of-two scale; returns 1/scale.
__device__ __forceinline__ float encode_row_own_scale(const float (&v)[64], uint32_t ta_hi, uint32_t ta_lo) {
    float s, inv;
    row_scale(row_absmax(v), s, inv);
    encode_row(v, s, ta_hi, ta_lo);
    return inv;
}
// D (+)= A_lo·B_hiᵀ + A_hi·B_loᵀ + A_hi·B_hiᵀ over the whole 128-row tile, K = N = 64 (12 wgmma of K = 16 per 64-row
// block): A_hi / A_lo = tile-memory columns a_hi / a_lo (32 each), B = a 64x64 weight in the layout of
// tc16::stage_weight, D = tile-memory columns d .. d + 63.  `accumulate` = add to the D already in tile memory.  Issued
// by every thread of the warpgroup and synchronous: on return D is in tile memory (other warps read it after a barrier).
__device__ __forceinline__ void mma_f16x3_tile(uint32_t d, uint32_t a_hi, uint32_t a_lo, const __half* b_hi,
                                               const __half* b_lo, bool accumulate) {
    constexpr uint32_t LBO = tc16::lbo_bytes(64);
    constexpr uint64_t B_KSTEP = (2 * LBO) >> 4, A_KSTEP = (2 * tmma::TM_COLGROUP_BYTES) >> 4;
    const uint64_t bh = tmma::make_desc(tmma::smem_u32(b_hi), LBO, 128);
    const uint64_t bl = tmma::make_desc(tmma::smem_u32(b_lo), LBO, 128);
#pragma unroll 1
    for (int mb = 0; mb < 2; ++mb) {
        const uint64_t ahi = tmma::make_desc(tmma::tm_addr_rc(64u * mb, a_hi), tmma::TM_COLGROUP_BYTES, 128);
        const uint64_t alo = tmma::make_desc(tmma::tm_addr_rc(64u * mb, a_lo), tmma::TM_COLGROUP_BYTES, 128);
        float acc[32];
        if (accumulate) {
            tmma::frag_load(acc, d, mb);
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        }
        tmma::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            tmma::wgmma_f16_m64n64k16(acc, alo + ks * A_KSTEP, bh + ks * B_KSTEP, (accumulate || ks > 0) ? 1u : 0u);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) tmma::wgmma_f16_m64n64k16(acc, ahi + ks * A_KSTEP, bl + ks * B_KSTEP, 1u);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) tmma::wgmma_f16_m64n64k16(acc, ahi + ks * A_KSTEP, bh + ks * B_KSTEP, 1u);
        tmma::wgmma_commit();
        tmma::wgmma_wait_all();
        tmma::frag_store(acc, d, mb);
    }
}
// one 64-wide fp32 row <-> 64 tile-memory columns of the own row
__device__ __forceinline__ void tm_store_row(uint32_t taddr, const float (&v)[64]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        uint32_t d[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) d[j] = __float_as_uint(v[16 * c + j]);
        tmma::tm_st16(taddr + 16 * c, d);
    }
}
__device__ __forceinline__ void tm_load_row(uint32_t taddr, float (&v)[64]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        uint32_t d[16];
        tmma::tm_ld16(taddr + 16 * c, d);
#pragma unroll
        for (int j = 0; j < 16; ++j) v[16 * c + j] = __uint_as_float(d[j]);
    }
}
__device__ __forceinline__ void smem_store_row(float* dst, const float (&v)[64]) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
        *reinterpret_cast<float4*>(dst + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}
// Column sums over the 32 rows of a warp of a 64-wide row held in registers (destroys u): after five exchange rounds lane
// l holds the sums of columns 2l and 2l+1 in u[0], u[1] (62 shuffles instead of 64 same-address shared-memory atomics).
__device__ __forceinline__ void warp_colsum64(float (&u)[64], int lane) {
#pragma unroll
    for (int b = 16, n = 64; b >= 1; b >>= 1, n >>= 1) {
        const bool up = lane & b;
        const int half = n >> 1;
#pragma unroll
        for (int i = 0; i < 32; ++i)
            if (i < half) {
                const float lo = u[i], hi = u[i + half];
                const float recv = __shfl_xor_sync(FULL, up ? lo : hi, b);
                u[i] = (up ? hi : lo) + recv;
            }
    }
}
// Backward through a φ head for the own row, D = A·Wᵀ with A encoded at scale 1/inv: zc = D·inv + b, returns
// φ = Σ_k SiLU(zc_k)·w3_k, adds the column sums over the warp's rows of gφ·SiLU(zc) to g_w3 (two shared atomics per
// lane) and turns the row into g_zc = gφ·w3 ⊙ SiLU'(zc); one σ serves SiLU and SiLU' = σ·(1 + zc·(1 − σ)).
__device__ __forceinline__ float phi_head_bwd(float (&v)[64], float inv, const float* b, const float* w3, float gphi,
                                              float* g_w3, int lane) {
    float phi = 0.f, u[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) {
        const float zc = fmaf(v[j], inv, b[j]);
        const float s = sigmoid_f(zc);
        const float ac = zc * s, w3j = w3[j];
        phi = fmaf(ac, w3j, phi);
        u[j] = gphi * ac;
        v[j] = gphi * w3j * (s * fmaf(zc, 1.0f - s, 1.0f));
    }
    warp_colsum64(u, lane);
    atomicAdd(g_w3 + 2 * lane, u[0]);
    atomicAdd(g_w3 + 2 * lane + 1, u[1]);
    return phi;
}
// acc[c] += Σ_e tile[e][c], the column sums of a 128-row tile: thread t <-> (column t & 63, half t >> 6 of the rows)
__device__ __forceinline__ void tile_colsum(float* acc, const float* tile, int t) {
    const int c = t & 63, h = t >> 6;
    float s0 = 0.f, s1 = 0.f;
    for (int e = 64 * h; e < 64 * h + 64; e += 2) {
        s0 += tile[e * LDA + c];
        s1 += tile[(e + 1) * LDA + c];
    }
    atomicAdd(acc + c, s0 + s1);
}
// acc[i][j] += Σ_e Gs[e][n0+i]·Act[e][k0+j], n0 = 8·(t >> 4), k0 = 4·(t & 15): 128 threads cover the 64x64 gradient
__device__ __forceinline__ void wgrad128(float (&acc)[8][4], const float* Gs, const float* Act, int t) {
    const int n0 = 8 * (t >> 4), k0 = 4 * (t & 15);
#pragma unroll 2
    for (int e = 0; e < TILE_M; ++e) {
        const float4 g0 = *reinterpret_cast<const float4*>(Gs + e * LDA + n0);
        const float4 g1 = *reinterpret_cast<const float4*>(Gs + e * LDA + n0 + 4);
        const float4 w = *reinterpret_cast<const float4*>(Act + e * LDA + k0);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            acc[i][0] = fmaf(gg[i], w.x, acc[i][0]);
            acc[i][1] = fmaf(gg[i], w.y, acc[i][1]);
            acc[i][2] = fmaf(gg[i], w.z, acc[i][2]);
            acc[i][3] = fmaf(gg[i], w.w, acc[i][3]);
        }
    }
}
__device__ __forceinline__ void wgrad128_flush(float* g_kmajor, const float (&acc)[8][4], int t) {
    const int n0 = 8 * (t >> 4), k0 = 4 * (t & 15);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) atomicAdd(g_kmajor + (k0 + j) * H + n0 + i, acc[i][j]);
}


}  // namespace degnn
