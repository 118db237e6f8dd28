// fp16 2-term split helpers shared by the tensor-core kernels (wgmma f16 path).
//   x = hi + lo,  hi = fp16(x),  lo = fp16(x − hi)          (22 significant bits)
//   A·Wᵀ ≈ A_lo·W_hiᵀ + A_hi·W_loᵀ + A_hi·W_hiᵀ             (fp32 accumulation)
// A rows live in tile memory (tile_mma.cuh: row = thread, two fp16 per 32-bit column, even k in the low half); W lives in
// shared memory
// in the canonical no-swizzle K-major layout for 16-bit types: core matrix = 8 rows x 8 halfs (128 B),
// element (n,k) at (k/8)*LBO + (n/8)*128 B + (n%8)*16 B + (k%8)*2 B with LBO = (N/8)*128 B.
// fp16 range: a row whose |max| exceeds 3e4 is re-encoded with a power-of-two scale s (cold path) and the
// caller multiplies the accumulator row by 1/s — results stay range-safe like fp32.  encode_rows is that rescue for the
// forward kernels' register fragments, together with the batched SiLU's stage-level guard; phi_head_t is their
// t-domain φ head.
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

// stage W[n][k] (given k-major: wt[k*64+n]) as rows n_off..n_off+63 of an N_total-row B operand, fp16 hi/lo;
// TRANSPOSED: stage Wᵀ instead, B[n][k] = wt[n*64+k].  Every B operand and weight image is laid out here.
// NTHREADS is a template parameter so that the H·H / NTHREADS loads of a thread are all issued before the first conversion
// (a rolled load -> convert -> store loop pays one global round trip per element and thread).  The element offset stays
// written out in the loop: as a function of its own, the compiler simplifies it before inlining and the forward kernels'
// address arithmetic and register allocation change.
template <int NTHREADS, bool TRANSPOSED = false>
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
        const int k = TRANSPOSED ? i & 63 : i >> 6, n = (TRANSPOSED ? i >> 6 : i & 63) + n_off;
        const float ws = w[r] * scale;
        const __half h = __float2half_rn(ws);
        const uint32_t o = (uint32_t)(k >> 3) * lbo_h + (uint32_t)(n >> 3) * 64u + (uint32_t)(n & 7) * 8u + (k & 7);
        hi[o] = h;
        lo[o] = __float2half_rn(ws - __half2float(h));
    }
}
__host__ __device__ constexpr uint32_t lbo_bytes(int n_total) { return (uint32_t)(n_total / 8) * 128u; }

// Register-operand flavour for one 64-row block held by a warpgroup: D = A_lo·B_hiᵀ + A_hi·B_loᵀ + A_hi·B_hiᵀ, K = 64,
// N = 64.  a_hi / a_lo are the A fragments of the four k-steps (tile_mma.cuh wgmma_f16_m64n64k16_rA: registers 4ks ..
// 4ks+3 for k-step ks), i.e. element (row, k) sits where an m64n64 accumulator keeps (row, column k).  Asynchronous:
// issues the 12 wgmma and commits them; mma_f16x3_rA_wait completes the group before d is read or a_hi / a_lo reused.
// ACCUMULATE: D += instead of D =.
template <uint32_t LBO, bool ACCUMULATE = false>
__device__ __forceinline__ void mma_f16x3_rA(float (&d)[32], const uint32_t (&a_hi)[16], const uint32_t (&a_lo)[16],
                                             uint64_t b_hi, uint64_t b_lo) {
    constexpr uint64_t B_KSTEP = (2 * LBO) >> 4;
    auto mma = [&](auto acc, const uint32_t (&a)[16], int ks, uint64_t b) {
        tmma::wgmma_f16_m64n64k16_rA<decltype(acc)::value>(d, a[4 * ks], a[4 * ks + 1], a[4 * ks + 2], a[4 * ks + 3],
                                                            b + ks * B_KSTEP);
    };
    tmma::wgmma_fence();
    mma(std::integral_constant<bool, ACCUMULATE>{}, a_lo, 0, b_hi);
#pragma unroll
    for (int ks = 1; ks < 4; ++ks) mma(std::true_type{}, a_lo, ks, b_hi);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) mma(std::true_type{}, a_hi, ks, b_lo);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) mma(std::true_type{}, a_hi, ks, b_hi);
    tmma::wgmma_commit();
}
__device__ __forceinline__ void mma_f16x3_rA_wait(float (&d)[32], uint32_t (&a_hi)[16], uint32_t (&a_lo)[16]) {
    tmma::wgmma_wait_all();
#pragma unroll
    for (int i = 0; i < 32; ++i) tmma::wgmma_keep(d[i]);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        tmma::wgmma_keep(a_hi[i]);
        tmma::wgmma_keep(a_lo[i]);
    }
}

__device__ __forceinline__ bool row_overflow(__half2 mx) {
    return fmaxf(__low2float(mx), __high2float(mx)) > RANGE;
}
// power-of-two scale that brings |rowmax| below 2^15 (1 for a smaller rowmax)
__device__ __forceinline__ float range_scale(float rowmax) {
    const uint32_t eb = (__float_as_uint(rowmax) >> 23) & 0xffu;
    const uint32_t sb = eb > 141u ? 268u - eb : 127u;
    return __uint_as_float((sb < 1u ? 1u : sb) << 23);
}
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(FULL, v, 1));
    return fmaxf(v, __shfl_xor_sync(FULL, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(FULL, v, 1);
    return v + __shfl_xor_sync(FULL, v, 2);
}

// ---- A fragments of the register-operand GEMMs: the fp16 range rescue --------------------------------------------
// The power-of-two scales of the calling thread's rows a and b (1: not scaled) and their inverses.
struct RowScales {
    float a = 1.0f, b = 1.0f, inv_a = 1.0f, inv_b = 1.0f;
};
// The passes of encode_rows, given to its producer as std::integral_constant<int, pass>.
constexpr int FAST_PASS = 0, MAX_PASS = 1, ENCODE_PASS = 2;
template <int P>
using Pass = std::integral_constant<int, P>;
struct NoGuard {
    __device__ __forceinline__ bool operator()() const { return false; }
};

// Encode the thread's rows a and b, produced as column pairs by f(j, xa, xb, pass) (columns 8j + 2q, +1), into the fp16
// hi/lo A fragments (register 2j + r holds pair j of row a / b for r = 0 / 1).  The fast pass splits the values as they
// are and tests |hi| > RANGE.  When a row of the warp fails it, or guard() (evaluated once, after the fast pass) is true,
// the warp takes the cold path: a pass that takes max |v| per row, then an encode pass with the row scaled by the
// power-of-two s = range_scale(max); s.a, s.b become those scales (only smaller than 1 where a row would leave the fp16
// range) and s.inv_a, s.inv_b their inverses.  f returns the same values on every pass, except that the fast pass may
// return values the guard rejects (the batched SiLU, silu4p / silu4t); where it stores what it produces is its own
// business (each pass is told apart).  Masking of invalid rows is the producer's too: a row it zeroes is 0 in the
// fragments and leaves the row maximum at 0.
//   SCALES_IN: the rows may already carry scales s.a, s.b != 1 (accumulation over several encodes into one D); then the
//              warp goes straight to the cold path and a row keeps the smaller of its incoming and its own scale.  Without
//              it s must come in as 1 and the call votes once less.
//   ROLLED_MAX: the row-max pass is not unrolled (only for producers that read memory, not accumulator registers).
// One range test for every producer, with the same decisions and scales as a test on the side that can overflow:
//   - SiLU outputs are ≥ −0.279 and t-domain outputs (SILU_T_IN·SiLU) ≤ 0.41, so |hi| > RANGE and max |v| differ from
//     the one-sided max hi / −min hi only where both are below 2^15;
//   - __hmax2 ignores NaN with or without __habs2, as fmaxf does in the row maximum;
//   - range_scale changes the scale only for a row maximum ≥ 2^15.
template <bool SCALES_IN, bool ROLLED_MAX = false, class F, class Guard = NoGuard>
__device__ __forceinline__ void encode_rows(F&& f, uint32_t (&hi)[16], uint32_t (&lo)[16], RowScales& s,
                                            Guard&& guard = Guard{}) {
    bool cold = SCALES_IN && __any_sync(FULL, s.a != 1.0f || s.b != 1.0f);
    if (!cold) {
        __half2 mx = __floats2half2_rn(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            f32x2 xa, xb;
            f(j, xa, xb, Pass<FAST_PASS>{});
            split_pair(xa, hi[2 * j], lo[2 * j]);
            split_pair(xb, hi[2 * j + 1], lo[2 * j + 1]);
            mx = __hmax2(mx, __habs2(*reinterpret_cast<const __half2*>(&hi[2 * j])));
            mx = __hmax2(mx, __habs2(*reinterpret_cast<const __half2*>(&hi[2 * j + 1])));
        }
        cold = __any_sync(FULL, row_overflow(mx) || guard());
    }
    if (!cold) return;
    // cold, per warp: some row of the warp carries a scale already or leaves the fp16 range, or the guard fired
    float fa = 0.f, fb = 0.f;
    auto row_max = [&](int j) {
        f32x2 xa, xb;
        float v0, v1;
        f(j, xa, xb, Pass<MAX_PASS>{});
        upk2(xa, v0, v1);
        fa = fmaxf(fa, fmaxf(fabsf(v0), fabsf(v1)));
        upk2(xb, v0, v1);
        fb = fmaxf(fb, fmaxf(fabsf(v0), fabsf(v1)));
    };
    if constexpr (ROLLED_MAX) {
#pragma unroll 1
        for (int j = 0; j < 8; ++j) row_max(j);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) row_max(j);
    }
    // row a's scale and inverse before row b's: with both divisions after both scales, ptxas spills in the edge kernel's
    // FLAG_LAST instantiations
    float ca = range_scale(quad_max(fa)), ia = 1.0f / ca;
    float cb = range_scale(quad_max(fb)), ib = 1.0f / cb;
    if constexpr (SCALES_IN) {
        ca = fminf(ca, s.a);
        cb = fminf(cb, s.b);
        ia = 1.0f / ca;
        ib = 1.0f / cb;
    }
    s = {ca, cb, ia, ib};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        f32x2 xa, xb;
        f(j, xa, xb, Pass<ENCODE_PASS>{});
        split_pair(mul2(xa, bc2(s.a)), hi[2 * j], lo[2 * j]);
        split_pair(mul2(xb, bc2(s.b)), hi[2 * j + 1], lo[2 * j + 1]);
    }
}

// The φ head of the t-domain kernels (common.cuh silu4t): φ = Σ_k w[k]·SiLU_t(D[row, k]·inv + b[k]) for the thread's rows
// a and b, summed over the quad, with b = SILU_T_IN·bias and w = SILU_T_OUT·w3 in shared memory.  The batched SiLU's
// guard redoes the warp with the per-element form; no range rescue (no fp16 operand follows).  Each pass forms the
// pre-activations from D again.
__device__ __forceinline__ void phi_head_t(const float (&d)[32], float inv_a, float inv_b, const float* b, const float* w,
                                           int q, float& phia, float& phib) {
    float qmax = 0.f;
    f32x2 pha, phb;
    auto pass = [&](auto safe) {
        pha = phb = bc2(0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const f32x2 bb = *reinterpret_cast<const f32x2*>(b + 8 * j + 2 * q);
            const f32x2 ww = *reinterpret_cast<const f32x2*>(w + 8 * j + 2 * q);
            f32x2 sa = fma2(pk2(d[4 * j + 0], d[4 * j + 1]), bc2(inv_a), bb);
            f32x2 sb = fma2(pk2(d[4 * j + 2], d[4 * j + 3]), bc2(inv_b), bb);
            silu4t<decltype(safe)::value>(sa, sb, qmax);
            pha = fma2(sa, ww, pha);
            phb = fma2(sb, ww, phb);
        }
    };
    pass(std::false_type{});
    if (__any_sync(FULL, silu_q_overflow(qmax))) pass(std::true_type{});
    float p0, p1;
    upk2(pha, p0, p1);
    phia = quad_sum(p0 + p1);
    upk2(phb, p0, p1);
    phib = quad_sum(p0 + p1);
}

}  // namespace tc16
}  // namespace degnn
