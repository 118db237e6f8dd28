// The tensor-core edge-stage backward kernel (template; see edge_layer_bwd_tc.cu for the algorithm).  Each of its two
// instantiations lives in its own translation unit: edge_layer_bwd_tc.cu (<false>, the weights-only kernel) and
// edge_layer_bwd_tc_inputs.cu (<true>, also the gradient w.r.t. edge_attr).  Compiled together, the second one changes
// the compiler's inlining decisions for the first, and the weights-only kernel should not change with a feature it
// does not use.
#pragma once

#include <cuda_fp16.h>

#include "bwd_common.cuh"
#include "bwd_tc_common.cuh"
#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct EdgeBwdTcArgs {
    int64_t N, E;
    const int32_t* E_dev;   // optional device-side edge count (E = capacity)
    int A;
    unsigned flags;
    const int32_t* row;
    const int32_t* col;
    const float* ea;
    const float* x4;
    const float* P;
    const float* Q;
    const float* w1r;
    const float* w1e;
    const float* w2;
    const float* b2;
    const float* wc;
    const float* bc;
    const float* w3;
    const float* g_aggm;
    const float* g_aggx;
    float* g_P;
    float* g_Q;
    float* g_x;
    float* g_w1r; float* g_w1e; float* g_w2; float* g_b2; float* g_wc; float* g_bc; float* g_w3;
    float* g_ea;            // [E,A] CSR order, accumulated (kInputs only)
};

constexpr int BT_THREADS = 128, BT_GROUPS = 1, BT_GROUP = 128;
constexpr int BT_TM_COLS = 128;                                // per tile group: A_hi 32 | A_lo 32 (= D 64) | z2 64
constexpr int BT_W = 64 * 64;                                   // halfs per staged weight matrix
constexpr int BT_SMEM_BYTES = tmma::tm_bytes(BT_GROUPS * BT_TM_COLS)
                              + 8 * BT_W * 2                    // W2, Wc, W2ᵀ, Wcᵀ (hi + lo each)
                              + BT_GROUPS * 2 * TILE_M * LDA * 4    // gradient tile + activation tile per group
                              + (4 * H + DISTEGNN_MAX_EDGE_ATTR * H) * 4     // b2, bc, w3, w1r, w1e
                              + (4 * H + DISTEGNN_MAX_EDGE_ATTR * H) * 4     // gradient accumulators of the same
                              + BT_GROUPS * TILE_M * (DISTEGNN_MAX_EDGE_ATTR + 1) * 4   // per-row edge attrs + radial
                              + BT_GROUPS * TILE_M * 2 * 4      // row, col per edge
                              + BT_GROUPS * 4 * 4               // run-start masks
                              ;
constexpr uint32_t BT_LBO = 1024;

// B operand of D = A·Bᵀ holding Wᵀ: B[n'][k'] = src[n'*64 + k'] (src = the k-major array of W itself)
__device__ __forceinline__ void stage_weight_t(__half* hi, __half* lo, const float* __restrict__ src, int tid, int nthreads) {
    for (int i = tid; i < H * H; i += nthreads) {
        const int n = i >> 6, k = i & 63;
        const float w = __ldg(src + i);
        const __half h = __float2half_rn(w);
        const uint32_t o = (uint32_t)(k >> 3) * 512u + (uint32_t)(n >> 3) * 64u + (uint32_t)(n & 7) * 8u + (k & 7);
        hi[o] = h;
        lo[o] = __float2half_rn(w - __half2float(h));
    }
}

// kInputs: also accumulate g_ea[e,k] += Σ_n g_z1[e,n]·W_e[k,n] (edge_attr in CSR order); the edge's row thread owns the
// row, so plain read-modify-writes suffice.  The <false> instantiation is the weights-only kernel, unchanged.
template <bool kInputs>
__global__ void __launch_bounds__(BT_THREADS, 1) edge_layer_bwd_tc_kernel(const EdgeBwdTcArgs a) {
    using namespace tmma;
    uint8_t* const smem_raw = degnn_dyn_smem + tm_bytes(BT_GROUPS * BT_TM_COLS);
    __half* W2hi = reinterpret_cast<__half*>(smem_raw);
    __half* W2lo = W2hi + BT_W;
    __half* Wchi = W2lo + BT_W;
    __half* Wclo = Wchi + BT_W;
    __half* W2Thi = Wclo + BT_W;
    __half* W2Tlo = W2Thi + BT_W;
    __half* WcThi = W2Tlo + BT_W;
    __half* WcTlo = WcThi + BT_W;
    float* tiles = reinterpret_cast<float*>(WcTlo + BT_W);                 // [groups][G tile | Act tile]
    float* b2s = tiles + BT_GROUPS * 2 * TILE_M * LDA;
    float* bcs = b2s + H;
    float* w3s = bcs + H;
    float* w1rs = w3s + H;
    float* w1es = w1rs + H;
    float* gb2 = w1es + DISTEGNN_MAX_EDGE_ATTR * H;
    float* gbc = gb2 + H;
    float* gw3 = gbc + H;
    float* gw1r = gw3 + H;
    float* gw1e = gw1r + H;
    float* rowsc_all = gw1e + DISTEGNN_MAX_EDGE_ATTR * H;                  // [groups][128][9]: edge attrs, radial
    int* srow_all = reinterpret_cast<int*>(rowsc_all + BT_GROUPS * TILE_M * (DISTEGNN_MAX_EDGE_ATTR + 1));
    int* scol_all = srow_all + BT_GROUPS * TILE_M;
    uint32_t* rmask_all = reinterpret_cast<uint32_t*>(scol_all + BT_GROUPS * TILE_M);

    const int tid = threadIdx.x;
    const int grp = tid / BT_GROUP, t = tid % BT_GROUP, lane = tid & 31, wq = (tid >> 5) & 3;
    const int A = a.A;
    const bool normalize = a.flags & DISTEGNN_FLAG_NORMALIZE;
    const bool need_m = !(a.flags & DISTEGNN_FLAG_LAST) && a.g_aggm != nullptr;

    // ---- one-time setup -------------------------------------------------------------------------------------
    tc16::stage_weight<BT_THREADS>(W2hi, W2lo, a.w2, 0, 64, tid);
    tc16::stage_weight<BT_THREADS>(Wchi, Wclo, a.wc, 0, 64, tid);
    stage_weight_t(W2Thi, W2Tlo, a.w2, tid, BT_THREADS);
    stage_weight_t(WcThi, WcTlo, a.wc, tid, BT_THREADS);
    if (tid < H) {
        b2s[tid] = a.b2[tid];
        bcs[tid] = a.bc[tid];
        w3s[tid] = a.w3[tid];
        w1rs[tid] = a.w1r[tid];
    }
    for (int i = tid; i < DISTEGNN_MAX_EDGE_ATTR * H; i += BT_THREADS) w1es[i] = i < A * H ? a.w1e[i] : 0.f;
    for (int i = tid; i < 4 * H + DISTEGNN_MAX_EDGE_ATTR * H; i += BT_THREADS) gb2[i] = 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    const uint32_t col0 = (uint32_t)(grp * BT_TM_COLS);
    const uint32_t lane_off = ((uint32_t)(32 * wq)) << 16;
    const uint32_t tA_hi = lane_off + col0, tA_lo = lane_off + col0 + 32, tD = lane_off + col0;
    const uint32_t tZ2 = lane_off + col0 + 64;
    float* Gt = tiles + grp * 2 * TILE_M * LDA;
    float* At = Gt + TILE_M * LDA;
    float* rowsc = rowsc_all + grp * TILE_M * (DISTEGNN_MAX_EDGE_ATTR + 1);
    int* srow = srow_all + grp * TILE_M;
    int* scol = scol_all + grp * TILE_M;
    uint32_t* rmask = rmask_all + grp * 4;
    const uint32_t bar_id = 1 + grp;
    // after the group barrier that publishes the A operand: D = A·Wᵀ over the whole tile by the group's warpgroup, written
    // over A; mma_done() publishes D to every row thread
    auto issue = [&](const __half* whi, const __half* wlo) {
        tc16::mma_f16x3<BT_LBO>(col0, col0, col0 + 32u, make_b_desc(smem_u32(whi), BT_LBO, 128),
                                make_b_desc(smem_u32(wlo), BT_LBO, 128), 1, false, 0, 2);
    };
    auto mma_done = [&]() { named_bar(bar_id, BT_GROUP); };
    auto a_ready = [&]() {
        tm_st_fence();
        named_bar(bar_id, BT_GROUP);
    };
    // column sums of the gradient tile into a shared accumulator: thread <-> (column, half of the rows)
    auto colsum_G = [&](float* acc) {
        const int c = t & 63, h = t >> 6;
        float s0 = 0.f, s1 = 0.f;
        for (int e = 64 * h; e < 64 * h + 64; e += 2) {
            s0 += Gt[e * LDA + c];
            s1 += Gt[(e + 1) * LDA + c];
        }
        atomicAdd(acc + c, s0 + s1);
    };

    float gW2[8][4], gWc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) gW2[i][j] = gWc[i][j] = 0.f;

    const int64_t nE = a.E_dev ? min((int64_t)__ldg(a.E_dev), a.E) : a.E;
    const int64_t num_tiles = (nE + TILE_M - 1) / TILE_M;
    for (int64_t tile = (int64_t)blockIdx.x * BT_GROUPS + grp; tile < num_tiles; tile += (int64_t)gridDim.x * BT_GROUPS) {
        // ---- the thread's edge: ids, attributes, geometry, upstream scalars ---------------------------------------
        const int64_t e = tile * TILE_M + t;
        const bool valid = e < nE;
        const int r = valid ? __ldg(a.row + e) : -1;
        const int c = valid ? __ldg(a.col + e) : 0;
        const int rr = max(r, 0);
        float dx, dy, dz, radial, invn = 0.f, gphi = 0.f;
        float4 gx = make_float4(0.f, 0.f, 0.f, 0.f);
        {
            const float4 xi = ldg4(a.x4 + (size_t)rr * 4), xj = ldg4(a.x4 + (size_t)c * 4);
            dx = xi.x - xj.x; dy = xi.y - xj.y; dz = xi.z - xj.z;
            radial = dx * dx + dy * dy + dz * dz;
            if (valid) {
                invn = normalize ? 1.0f / (sqrtf(radial) + 1e-8f) : 1.0f;
                gx = ldg4(a.g_aggx + (size_t)rr * 4);
                gphi = (gx.x * dx + gx.y * dy + gx.z * dz) * invn;
            }
        }
        float* myrs = rowsc + t * (DISTEGNN_MAX_EDGE_ATTR + 1);
        for (int k = 0; k < A; ++k) myrs[k] = valid ? __ldg(a.ea + e * A + k) : 0.f;
        myrs[DISTEGNN_MAX_EDGE_ATTR] = valid ? radial : 0.f;
        srow[t] = r;
        scol[t] = c;

        // z1 = P[row] + Q[col] + w_r·r + W_e·a of the own edge (stage 1, and again where SiLU(z1) / SiLU'(z1) are needed)
        auto z1_row = [&](float (&z1)[64]) {
            const float* prow = a.P + (size_t)rr * H;
            const float* qrow = a.Q + (size_t)c * H;
#pragma unroll
            for (int j4 = 0; j4 < 16; ++j4) {
                float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                if (valid) {
                    z = fma4(radial, *reinterpret_cast<const float4*>(w1rs + 4 * j4), add4(ldg4(prow + 4 * j4), ldg4(qrow + 4 * j4)));
                    for (int k = 0; k < A; ++k) z = fma4(myrs[k], *reinterpret_cast<const float4*>(w1es + k * H + 4 * j4), z);
                }
                z1[4 * j4] = z.x; z1[4 * j4 + 1] = z.y; z1[4 * j4 + 2] = z.z; z1[4 * j4 + 3] = z.w;
            }
        };
        float v[64];
        // ---- stage 1: a1 = SiLU(z1) -> A --------------------------------------------------------------------------
        {
            z1_row(v);
#pragma unroll
            for (int j = 0; j < 64; ++j) v[j] = silu(v[j]);
        }
        const float inv1 = encode_row_regs(v, tA_hi, tA_lo);
        a_ready();                                  // also publishes srow/scol/rowsc of this tile to the group
        issue(W2hi, W2lo);
        if (t < 128 && lane < 32) {                 // run starts (whole warps): bit i of rmask[q] = edge 32q+i starts a run
            const int prev = t > 0 ? srow[t - 1] : -2;
            const uint32_t starts = __ballot_sync(FULL, prev != r);
            if (lane == 0) rmask[wq] = starts;
        }
        mma_done();

        // ---- stage 2: z2 = D/s + b2 -> tile memory; m = SiLU(z2) -> activation tile + A -------------------------------
        tm_load_row(tD, v);
#pragma unroll
        for (int j = 0; j < 64; ++j) v[j] = fmaf(v[j], inv1, b2s[j]);
        tm_store_row(tZ2, v);
#pragma unroll
        for (int j = 0; j < 64; ++j) v[j] = silu(v[j]);
        smem_store_row(At + t * LDA, v);
        const float inv2 = encode_row_regs(v, tA_hi, tA_lo);
        a_ready();
        issue(Wchi, Wclo);
        mma_done();

        // ---- stage 3: zc = D/s + bc; φ; g_w3; g_zc = gφ·w3 ⊙ SiLU'(zc) -> gradient tile + A ------------------------------
        float phi = 0.f;
        tm_load_row(tD, v);
        {
            float u[64];                            // gφ·SiLU(zc): its column sums over the tile are g_w3
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                const float zc = fmaf(v[j], inv2, bcs[j]);
                const float s = sigmoid_f(zc);
                const float ac = zc * s, w3j = w3s[j];
                phi = fmaf(ac, w3j, phi);
                u[j] = gphi * ac;                   // gφ = 0 on rows beyond E
                v[j] = gphi * w3j * (s * fmaf(zc, 1.0f - s, 1.0f));
            }
            warp_colsum64(u, lane);
            atomicAdd(gw3 + 2 * lane, u[0]);
            atomicAdd(gw3 + 2 * lane + 1, u[1]);
        }
        smem_store_row(Gt + t * LDA, v);
        const float inv3 = encode_row_regs(v, tA_hi, tA_lo);
        a_ready();                                  // gradient tile + activation tile visible, A complete, D fully read
        issue(WcThi, WcTlo);
        wgrad128(gWc, Gt, At, t);                   // g_Wc += g_zcᵀ·m
        colsum_G(gbc);
        named_bar(bar_id, BT_GROUP);                // both tiles fully read
        mma_done();

        // ---- stage 4: g_m = D/s + g_aggm[row]; g_z2 = g_m ⊙ SiLU'(z2) -> gradient tile + A; a1 -> activation tile ----------
        {
            float z2[64];
            tm_load_row(tD, v);
            tm_load_row(tZ2, z2);
            const float* gm = a.g_aggm + (size_t)rr * H;
#pragma unroll
            for (int j4 = 0; j4 < 16; ++j4) {
                float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
                if (need_m && valid) u = ldg4(gm + 4 * j4);
                v[4 * j4 + 0] = fmaf(v[4 * j4 + 0], inv3, u.x) * dsilu(z2[4 * j4 + 0]);
                v[4 * j4 + 1] = fmaf(v[4 * j4 + 1], inv3, u.y) * dsilu(z2[4 * j4 + 1]);
                v[4 * j4 + 2] = fmaf(v[4 * j4 + 2], inv3, u.z) * dsilu(z2[4 * j4 + 2]);
                v[4 * j4 + 3] = fmaf(v[4 * j4 + 3], inv3, u.w) * dsilu(z2[4 * j4 + 3]);
            }
            smem_store_row(Gt + t * LDA, v);
            const float inv4_ = encode_row_regs(v, tA_hi, tA_lo);
            z1_row(z2);                             // reuse the buffer: z1 -> a1 row for the weight gradient
#pragma unroll
            for (int j = 0; j < 64; ++j) z2[j] = silu(z2[j]);
            smem_store_row(At + t * LDA, z2);
            a_ready();
            issue(W2Thi, W2Tlo);
            wgrad128(gW2, Gt, At, t);               // g_W2 += g_z2ᵀ·a1
            colsum_G(gb2);
            named_bar(bar_id, BT_GROUP);
            mma_done();

            // ---- stage 5: g_z1 = D/s ⊙ SiLU'(z1) -> gradient tile; g_r ---------------------------------------------------
            tm_load_row(tD, v);
            z1_row(z2);
            float gr = 0.f;
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                v[j] = v[j] * inv4_ * dsilu(z2[j]);
                gr = fmaf(v[j], w1rs[j], gr);
            }
            smem_store_row(Gt + t * LDA, v);
            if constexpr (kInputs) {
                if (valid && a.g_ea) {
                    for (int k = 0; k < A; ++k) {
                        float s = 0.f;
#pragma unroll
                        for (int j = 0; j < 64; ++j) s = fmaf(v[j], w1es[k * H + j], s);
                        a.g_ea[e * A + k] += s;
                    }
                }
            }
            // geometry: gΔ_raw = g_aggx[i]·φ/norm + 2·g_r·Δ_raw.  A self loop's +gΔ and −gΔ land on the same node and its
            // exact gradient is zero, but under FLAG_NORMALIZE gΔ carries 1/(0 + 1e-8): the pair would round the node's sum
            if (valid && r != c) {
                const float s = phi * invn, t2 = 2.0f * gr;
                const float gdx = fmaf(gx.x, s, t2 * dx), gdy = fmaf(gx.y, s, t2 * dy), gdz = fmaf(gx.z, s, t2 * dz);
                atomicAdd(a.g_x + (size_t)r * 4 + 0, gdx);
                atomicAdd(a.g_x + (size_t)r * 4 + 1, gdy);
                atomicAdd(a.g_x + (size_t)r * 4 + 2, gdz);
                atomicAdd(a.g_x + (size_t)c * 4 + 0, -gdx);
                atomicAdd(a.g_x + (size_t)c * 4 + 1, -gdy);
                atomicAdd(a.g_x + (size_t)c * 4 + 2, -gdz);
            }
        }
        named_bar(bar_id, BT_GROUP);                // g_z1 tile visible

        // ---- scatter of the g_z1 tile: g_P by runs of equal row, g_Q per edge, g_w_r / g_W_e column sums -----------------
        {   // g_P: warp <-> 32 edges, lane <-> column pair, one RED.v2 per run
            const float* colp = Gt + (32 * wq) * LDA + 2 * lane;
            uint32_t M = rmask[wq] | 1u;
            while (M) {
                const int s0 = __ffs((int)M) - 1;
                M &= M - 1;
                const int s1 = M ? __ffs((int)M) - 1 : 32;
                float2 s = make_float2(0.f, 0.f);
                for (int q = s0; q < s1; ++q) {
                    const float2 u = *reinterpret_cast<const float2*>(colp + q * LDA);
                    s.x += u.x; s.y += u.y;
                }
                const int pr = srow[32 * wq + s0];
                if (pr >= 0) red_add_v2(a.g_P + (size_t)pr * H + 2 * lane, s.x, s.y);
            }
        }
        {   // g_Q: half-warp per edge, RED.v4
            const int l = lane & 15;
#pragma unroll 2
            for (int it = 0; it < 16; ++it) {
                const int el = 32 * wq + 2 * it + (lane >> 4);
                if (srow[el] >= 0) red_add_v4(a.g_Q + (size_t)scol[el] * H + 4 * l, *reinterpret_cast<const float4*>(Gt + el * LDA + 4 * l));
            }
        }
        {   // g_w_r[n] += Σ_e g_z1[e][n]·radial_e,  g_W_e[k][n] += Σ_e g_z1[e][n]·a_ek: thread <-> (column, half of the rows)
            const int cc = t & 63, h = t >> 6;
            float sr = 0.f, se[DISTEGNN_MAX_EDGE_ATTR];
#pragma unroll
            for (int k = 0; k < DISTEGNN_MAX_EDGE_ATTR; ++k) se[k] = 0.f;
            for (int q = 64 * h; q < 64 * h + 64; ++q) {
                const float u = Gt[q * LDA + cc];
                const float* rs = rowsc + q * (DISTEGNN_MAX_EDGE_ATTR + 1);
                sr = fmaf(u, rs[DISTEGNN_MAX_EDGE_ATTR], sr);
#pragma unroll
                for (int k = 0; k < DISTEGNN_MAX_EDGE_ATTR; ++k)
                    if (k < A) se[k] = fmaf(u, rs[k], se[k]);
            }
            atomicAdd(gw1r + cc, sr);
#pragma unroll
            for (int k = 0; k < DISTEGNN_MAX_EDGE_ATTR; ++k)
                if (k < A) atomicAdd(gw1e + k * H + cc, se[k]);
        }
        named_bar(bar_id, BT_GROUP);                // tiles and per-row arrays are rewritten by the next iteration
    }

    // ---- flush the CTA's parameter gradients ------------------------------------------------------------------------
    wgrad128_flush(a.g_w2, gW2, t);
    wgrad128_flush(a.g_wc, gWc, t);
    __syncthreads();
    if (tid < H) {
        atomicAdd(a.g_b2 + tid, gb2[tid]);
        atomicAdd(a.g_bc + tid, gbc[tid]);
        atomicAdd(a.g_w3 + tid, gw3[tid]);
        atomicAdd(a.g_w1r + tid, gw1r[tid]);
    }
    for (int i = tid; i < A * H; i += BT_THREADS) atomicAdd(a.g_w1e + i, gw1e[i]);
}

}  // namespace degnn
