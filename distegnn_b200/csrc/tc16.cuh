// fp16 2-term split helpers shared by the tensor-core kernels (wgmma f16 path).
//   x = hi + lo,  hi = fp16(x),  lo = fp16(x − hi)          (22 significant bits)
//   A·Wᵀ ≈ A_lo·W_hiᵀ + A_hi·W_loᵀ + A_hi·W_hiᵀ             (fp32 accumulation)
// A rows live in tile memory (tile_mma.cuh: row = thread, two fp16 per 32-bit column, even k in the low half); W lives in
// shared memory
// in the canonical no-swizzle K-major layout for 16-bit types: core matrix = 8 rows x 8 halfs (128 B),
// element (n,k) at (k/8)*LBO + (n/8)*128 B + (n%8)*16 B + (k%8)*2 B with LBO = (N/8)*128 B.
// fp16 range: a row whose |max| exceeds 3e4 is re-encoded with a power-of-two scale s (cold path) and the
// caller multiplies the accumulator row by 1/s — results stay range-safe like fp32.
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "tile_mma.cuh"

namespace degnn {
namespace tc16 {

constexpr float RANGE = 3.0e4f;
// (hi, lo) fp16 pairs of the fp32 pair x: hi = rn(x), lo = rn(x − hi).  x − hi is exact in fp32 (hi is within half an fp16
// ulp of x).
__device__ __forceinline__ void split_pair(f32x2 x, uint32_t& hi, uint32_t& lo) {
    float x0, x1, l0, l1;
    upk2(x, x0, x1);
    const __half2 h = __floats2half2_rn(x0, x1);                // x0 -> low half (even k)
    hi = *reinterpret_cast<const uint32_t*>(&h);
    const float2 hf = __half22float2(h);
    upk2(sub2(x, pk2(hf.x, hf.y)), l0, l1);
    const __half2 l = __floats2half2_rn(l0, l1);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// stage W[n][k] (given k-major: wt[k*64+n]) as rows n_off..n_off+63 of an N_total-row B operand, fp16 hi/lo
// NTHREADS is a template parameter so that the H·H / NTHREADS loads of a thread are all issued before the first conversion
// (a rolled load -> convert -> store loop pays one global round trip per element and thread).
template <int NTHREADS>
__device__ __forceinline__ void stage_weight(__half* hi, __half* lo, const float* __restrict__ wt_kmajor, int n_off,
                                             int n_total, int tid, float scale = 1.0f) {
    static_assert((H * H) % NTHREADS == 0, "thread count must divide the matrix");
    constexpr int R = H * H / NTHREADS;
    const uint32_t lbo_h = (uint32_t)(n_total / 8) * 64u;     // halfs per K chunk of 8
    float w[R];
#pragma unroll
    for (int r = 0; r < R; ++r) w[r] = __ldg(wt_kmajor + tid + r * NTHREADS);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int i = tid + r * NTHREADS;
        const int k = i >> 6, n = (i & 63) + n_off;
        const float ws = w[r] * scale;
        const __half h = __float2half_rn(ws);
        const uint32_t o = (uint32_t)(k >> 3) * lbo_h + (uint32_t)(n >> 3) * 64u + (uint32_t)(n & 7) * 8u + (k & 7);
        hi[o] = h;
        lo[o] = __float2half_rn(ws - __half2float(h));
    }
}
__host__ __device__ constexpr uint32_t lbo_bytes(int n_total) { return (uint32_t)(n_total / 8) * 128u; }

// D (+)= A_lo·B_hiᵀ + A_hi·B_loᵀ + A_hi·B_hiᵀ with K = 64 (12 wgmma of K = 16 per 64x64 block) for the 64-row blocks
// mb0 .. mb0 + nmb − 1 of the tile and N = 64·nchunks columns: A_hi / A_lo = tile-memory columns a_hi / a_lo (32 each),
// B rows n = 64·chunk .. of the staged weights, D = tile-memory columns d .. d + 64·nchunks − 1.  `accumulate` = add to
// the D already in tile memory.  Issued by every thread of ONE warpgroup and synchronous: on return the D rows of the
// warpgroup's blocks are in tile memory (threads of other warps read them after a barrier).
template <uint32_t LBO>
__device__ __forceinline__ void mma_f16x3(uint32_t d, uint32_t a_hi, uint32_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                          int nchunks, bool accumulate, int mb0, int nmb) {
    constexpr uint64_t B_KSTEP = (2 * LBO) >> 4, A_KSTEP = (2 * tmma::TM_COLGROUP_BYTES) >> 4, B_NCHUNK = (8 * 128) >> 4;
#pragma unroll 1
    for (int mb = mb0; mb < mb0 + nmb; ++mb) {
        const uint64_t ahi = tmma::make_desc(tmma::tm_addr_rc(64u * mb, a_hi), tmma::TM_COLGROUP_BYTES, 128);
        const uint64_t alo = tmma::make_desc(tmma::tm_addr_rc(64u * mb, a_lo), tmma::TM_COLGROUP_BYTES, 128);
#pragma unroll 1
        for (int nc = 0; nc < nchunks; ++nc) {
            float acc[32];
            if (accumulate) {
                tmma::frag_load(acc, d + 64u * nc, mb);
            } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            }
            const uint64_t bh = b_hi + nc * B_NCHUNK, bl = b_lo + nc * B_NCHUNK;
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
            tmma::frag_store(acc, d + 64u * nc, mb);
        }
    }
}

// 16 fp32 values (·s) -> 8 packed hi words + 8 packed lo words; `mx` tracks max |hi|
template <bool SCALED>
__device__ __forceinline__ void split16(const float (&v)[16], float s, uint32_t (&hi)[8], uint32_t (&lo)[8],
                                        __half2& mx) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float x0 = SCALED ? v[2 * j] * s : v[2 * j], x1 = SCALED ? v[2 * j + 1] * s : v[2 * j + 1];
        const __half2 h = __floats2half2_rn(x0, x1);            // x0 -> low half (even k)
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
        mx = __hmax2(mx, __habs2(h));
        hi[j] = *reinterpret_cast<const uint32_t*>(&h);
        lo[j] = *reinterpret_cast<const uint32_t*>(&l);
    }
}
__device__ __forceinline__ bool row_overflow(__half2 mx) {
    return fmaxf(__low2float(mx), __high2float(mx)) > RANGE;
}
// power-of-two scale that brings |rowmax| below 2^15, and its inverse
__device__ __forceinline__ void range_scale(float rowmax, float& s, float& inv_s) {
    const uint32_t eb = (__float_as_uint(rowmax) >> 23) & 0xffu;
    const uint32_t sb = eb > 141u ? 268u - eb : 127u;
    s = __uint_as_float((sb < 1u ? 1u : sb) << 23);
    inv_s = 1.0f / s;
}

// Encode one 64-wide fp32 row, produced 16 values at a time by f(chunk, v, first_pass), into the A operand
// (tile-memory columns ta_hi.. / ta_lo.., both including the warp's lane offset) with row scale `s_in` (a power of two
// the row already carries, 1 normally).  Returns the scale actually used (<= s_in): smaller only if the row
// would leave the fp16 range.  The caller issues tm_st_fence() afterwards and multiplies the accumulator row
// by 1/scale in its epilogue.
template <class F>
__device__ __forceinline__ float encode_row_s(F&& f, uint32_t ta_hi, uint32_t ta_lo, float s_in) {
    __half2 mx = __floats2half2_rn(0.f, 0.f);
    const bool pre_scaled = __any_sync(FULL, s_in != 1.0f);
    if (!pre_scaled) {
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
            float v[16];
            uint32_t hi[8], lo[8];
            f(c, v, true);
            split16<false>(v, 1.0f, hi, lo, mx);
            tmma::tm_st8(ta_hi + 8 * c, hi);
            tmma::tm_st8(ta_lo + 8 * c, lo);
        }
        if (!__any_sync(FULL, row_overflow(mx))) return 1.0f;
    }
    // cold: some row of this warp carries a scale already or leaves the fp16 range
    float fm = 0.f, sc, inv_unused;
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        float v[16];
        f(c, v, pre_scaled && true);
#pragma unroll
        for (int j = 0; j < 16; ++j) fm = fmaxf(fm, fabsf(v[j]));
    }
    range_scale(fm, sc, inv_unused);
    sc = fminf(sc, s_in);
    tmma::tm_st_fence();
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        float v[16];
        uint32_t hi[8], lo[8];
        f(c, v, false);
        split16<true>(v, sc, hi, lo, mx);
        tmma::tm_st8(ta_hi + 8 * c, hi);
        tmma::tm_st8(ta_lo + 8 * c, lo);
    }
    return sc;
}
// ---- register-pair flavour (fp32 pairs, common.cuh) ------------------------------------------------------------
constexpr std::false_type kFast{};   // silu4p flavour tags
constexpr std::true_type kSafe{};
template <bool SCALED>
__device__ __forceinline__ void split16p(const f32x2 (&v)[8], float s, uint32_t (&hi)[8], uint32_t (&lo)[8],
                                         __half2& mx) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        split_pair(SCALED ? mul2(v[j], bc2(s)) : v[j], hi[j], lo[j]);
        mx = __hmax2(mx, __habs2(*reinterpret_cast<const __half2*>(&hi[j])));
    }
}
// Same contract as encode_row_s, for producers f(chunk, v[8 pairs], first_pass, flavour tag, qmax) that run their
// SiLUs through silu4p<flavour>(…, qmax).  The hot pass uses the batched-reciprocal flavour; if its range guard
// fires (or a row leaves the fp16 range) the warp redoes the row with the per-element flavour.  The first cold
// pass is told first_pass = true again so that side effects (rows copied to shared memory) are rewritten with
// valid values — producers must keep those side effects idempotent.
template <class F>
__device__ __forceinline__ float encode_row2_s(F&& f, uint32_t ta_hi, uint32_t ta_lo, float s_in) {
    __half2 mx = __floats2half2_rn(0.f, 0.f);
    float qmax = 0.f;
    const bool pre_scaled = __any_sync(FULL, s_in != 1.0f);
    if (!pre_scaled) {
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
            f32x2 v[8];
            uint32_t hi[8], lo[8];
            f(c, v, true, kFast, qmax);
            split16p<false>(v, 1.0f, hi, lo, mx);
            tmma::tm_st8(ta_hi + 8 * c, hi);
            tmma::tm_st8(ta_lo + 8 * c, lo);
        }
        if (!__any_sync(FULL, row_overflow(mx) || silu_q_overflow(qmax))) return 1.0f;
    }
    float fm = 0.f, sc, inv_unused;
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        f32x2 v[8];
        f(c, v, true, kSafe, qmax);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v0, v1;
            upk2(v[j], v0, v1);
            fm = fmaxf(fm, fmaxf(fabsf(v0), fabsf(v1)));
        }
    }
    range_scale(fm, sc, inv_unused);
    sc = fminf(sc, s_in);
    tmma::tm_st_fence();
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        f32x2 v[8];
        uint32_t hi[8], lo[8];
        f(c, v, false, kSafe, qmax);
        split16p<true>(v, sc, hi, lo, mx);
        tmma::tm_st8(ta_hi + 8 * c, hi);
        tmma::tm_st8(ta_lo + 8 * c, lo);
    }
    return sc;
}
// Same contract for stages whose input is a 64-column fp32 accumulator in tile memory at `t_src` (lane offset included):
// the producer is f(chunk, d[16 raw accumulator words], v[8 pairs], first_pass, flavour tag, qmax).
template <class F>
__device__ __forceinline__ float encode_row2_tm(F&& f, uint32_t t_src, uint32_t ta_hi, uint32_t ta_lo) {
    __half2 mx = __floats2half2_rn(0.f, 0.f);
    float qmax = 0.f;
    {
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
            f32x2 v[8];
            uint32_t hi[8], lo[8], d[16];
            tmma::tm_ld16(t_src + 16 * c, d);
            f(c, d, v, true, kFast, qmax);
            split16p<false>(v, 1.0f, hi, lo, mx);
            tmma::tm_st8(ta_hi + 8 * c, hi);
            tmma::tm_st8(ta_lo + 8 * c, lo);
        }
        if (!__any_sync(FULL, row_overflow(mx) || silu_q_overflow(qmax))) return 1.0f;
    }
    float fm = 0.f, sc, inv_unused;                 // cold: per-row range rescue / per-element SiLU flavour
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        f32x2 v[8];
        uint32_t d[16];
        tmma::tm_ld16(t_src + 16 * c, d);
        f(c, d, v, true, kSafe, qmax);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v0, v1;
            upk2(v[j], v0, v1);
            fm = fmaxf(fm, fmaxf(fabsf(v0), fabsf(v1)));
        }
    }
    range_scale(fm, sc, inv_unused);
    sc = fminf(sc, 1.0f);
    tmma::tm_st_fence();
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
        f32x2 v[8];
        uint32_t hi[8], lo[8], d[16];
        tmma::tm_ld16(t_src + 16 * c, d);
        f(c, d, v, false, kSafe, qmax);
        split16p<true>(v, sc, hi, lo, mx);
        tmma::tm_st8(ta_hi + 8 * c, hi);
        tmma::tm_st8(ta_lo + 8 * c, lo);
    }
    return sc == 1.0f ? 1.0f : 1.0f / sc;
}

template <class F>
__device__ __forceinline__ float encode_row2(F&& f, uint32_t ta_hi, uint32_t ta_lo) {
    const float sc = encode_row2_s(f, ta_hi, ta_lo, 1.0f);
    return sc == 1.0f ? 1.0f : 1.0f / sc;
}

// Convenience: unscaled input, returns 1/scale for the epilogue.
template <class F>
__device__ __forceinline__ float encode_row(F&& f, uint32_t ta_hi, uint32_t ta_lo) {
    const float sc = encode_row_s(f, ta_hi, ta_lo, 1.0f);
    return sc == 1.0f ? 1.0f : 1.0f / sc;
}

}  // namespace tc16
}  // namespace degnn
