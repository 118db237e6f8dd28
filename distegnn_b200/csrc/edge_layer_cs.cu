// Real<->real edge stage, column-split flavour — production kernel behind distegnn_edge_layer_fwd.
// Same outputs as testing/edge_layer.cu (fp32-FMA twin, distegnn_edge_layer_fwd_simt); replaces reference models/FastEGNN.py:237-246 (coord2radial), 144-150 (edge_model), 169-177 (edge part of
// coord_model_vel), 206 (edge part of node_model) and the scatter_add_ of :322-337 (twins models/basic.py:22-66).
//
// Column split: TWO threads share a row, each owning 32 of its 64 columns end to end, so that a whole 64-wide row of
// state never has to sit in one thread's registers.
//
// One CTA per SM, one tile group of 8 warps = 2 warpgroups.  Warp k of the group: row quarter k & 3, column half k >> 2;
// thread (quarter, lane, half) owns row 32·quarter + lane, columns 32·half .. +31 of the group's current 128-edge tile.
// The A operand and the accumulator live in tile memory (tile_mma.cuh: A_hi 32 | A_lo 32 | D 64 columns, 64 KB of shared
// memory); warpgroup h computes the 64-row block h of every tile GEMM with wgmma.  Per tile (numerics as in the other
// tensor-core kernels: fp16 2-term split, per-row power-of-two range rescue, one reciprocal per four SiLUs with a
// stage-level guard):
//   stage 1  a1 = SiLU(P[row] + Q[col] + w_r·r + W_e·a) -> fp16 hi/lo -> A                   MMA 1: D = a1·W2ᵀ
//   stage 2  m = SiLU(D + b2) -> own half row to shared + hi/lo -> A                          MMA 2: D = m·Wcᵀ
//            segment sum of m over destination rows after MMA 2 (warp <-> 16 edges, lane <-> column pair)
//   stage 3  φ_half = w3·SiLU(D + bc) over the own 32 columns; Δx·φ_half reduced over runs of equal row by warp
//            shuffles, RED.ADD (the two halves add their partial sums independently: no cross-warp exchange).
// The range rescue needs ONE scale per row, i.e. agreement between the two warps that share it: every warp posts
// an "anything out of range" flag before the group barrier that precedes the MMA; if any flag is set the whole
// group takes the cold path (row maxima exchanged through shared memory, two more barriers).
// Everything a tile needs from memory is requested at least one stage ahead:
//   (row, col, edge_attr) of tile i+1   LDGSTS at the start of stage 1 of tile i (double buffered)
//   Q[col] rows of tile i+1             one TMA bulk copy per row, after the segment sum of tile i
//   x[row], x[col] of tile i+1          one cp.async pair per edge after the stage-1 barrier, read by both halves at the tile end
//   P[row] of tile i+1, chunk 0         LDG at the end of stage 3 of tile i; chunk j+1 before the math of chunk j
// Stages 2 and 3 run in the "t domain" (common.cuh silu4t): −log2(e) is folded into W2 and the biases, −ln 2 into w3 and
// the segment-sum flush, so the SiLU never forms its exponent argument explicitly.
#include <cuda_fp16.h>
#include <string.h>

#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct EdgeCsArgs {
    int64_t N, E;
    const int32_t* E_dev;   // optional: the edge count on the device (graphs built without a host round trip); E = capacity
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
    const float* w2;   // k-major [k][n]
    const float* b2;
    const float* wc;   // k-major [k][n]
    const float* bc;
    const float* w3;
    float* agg_m;
    float* agg_x;
};

// One tile group per CTA: its 64 KB of tile memory and 35 KB staging buffer next to the weights leave no room for a second
// one in 227 KB of shared memory.  The per-group indexing below follows CS_GROUPS.
constexpr int CS_THREADS = 256, CS_GROUPS = 1, CS_GROUP = 256, CS_WARPS = 8;
// padded row pitch of the staging buffer (floats): 68 = conflict-free row-per-thread LDS.128 / STS.128
constexpr int CS_QROW = 68;
constexpr int CS_QBUF = TILE_M * CS_QROW;
__host__ __device__ constexpr int cs_qoff(int r) { return r * CS_QROW; }
constexpr int CS_TM_COLS = 128;                           // per tile group: A_hi 32 | A_lo 32 | D 64
constexpr int CS_W = 64 * 64;                             // fp16 elements per weight matrix (8 KB)
constexpr int CS_IDX = TILE_M * 4;                        // ints per index buffer: row 128 | col 128 | ea 128x2
constexpr int CS_SMEM_BYTES = tmma::tm_bytes(CS_GROUPS * CS_TM_COLS)
                              + 4 * CS_W * 2                // W2 hi/lo, Wc hi/lo
                              + CS_GROUPS * CS_QBUF * 4
                              + (4 * H + DISTEGNN_MAX_EDGE_ATTR * H) * 4   // b2, bc, w3, w1r, w1e
                              + CS_GROUPS * 2 * TILE_M * 4    // srow, double buffered by tile parity
                              + CS_GROUPS * 4 * 4             // run-start bit masks (one word per lane quarter)
                              + CS_GROUPS * 2 * CS_IDX * 4    // staged indices of the next tile, double buffered
                              + CS_GROUPS * 2 * CS_WARPS * 4  // out-of-range flags per warp, one set per stage
                              + CS_GROUPS * 2 * TILE_M * 4    // row maxima of the two column halves (cold path)
                              + CS_GROUPS * TILE_M * 8 * 4    // x[row], x[col] of the next tile's edges
                              + 128;                          // mbarriers
constexpr uint32_t CS_LBO = 1024;                         // fp16 K-major no-swizzle, N = 64
using tc16::kFast;
using tc16::kSafe;

// 8 fp32 values held as 4 register pairs (·s) -> 4 packed hi words + 4 packed lo words.  `mx` tracks the side of the values
// that can leave the fp16 range: SiLU outputs are bounded below (−0.28), so the positive side — or, for t-domain values
// (NEG: s = −log2(e)·SiLU), the negative one, tracked as a running minimum.
template <bool SCALED, bool NEG>
__device__ __forceinline__ void split8(const f32x2 (&v)[4], float s, uint32_t (&hi)[4], uint32_t (&lo)[4], __half2& mx) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        tc16::split_pair(SCALED ? mul2(v[j], bc2(s)) : v[j], hi[j], lo[j]);
        const __half2 h = *reinterpret_cast<const __half2*>(&hi[j]);
        mx = NEG ? __hmin2(mx, h) : __hmax2(mx, h);
    }
}
template <bool NEG>
__device__ __forceinline__ bool row_overflow8(__half2 mx) {
    return NEG ? fminf(__low2float(mx), __high2float(mx)) < -tc16::RANGE : tc16::row_overflow(mx);
}
template <bool NEG>
__device__ __forceinline__ float max8(const f32x2 (&v)[4], float fm) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float v0, v1;
        upk2(v[j], v0, v1);
        fm = NEG ? fmaxf(fm, -fminf(v0, v1)) : fmaxf(fm, fmaxf(v0, v1));
    }
    return fm;
}

template <int AT, bool LASTL>
__global__ void __launch_bounds__(CS_THREADS, 1) edge_layer_cs_kernel(const EdgeCsArgs a) {
    using namespace tmma;
    constexpr int AMAX = AT >= 0 ? (AT > 0 ? AT : 1) : DISTEGNN_MAX_EDGE_ATTR;
    constexpr bool kEaStaged = (AT == 1 || AT == 2);
    uint8_t* const smem_raw = degnn_dyn_smem + tm_bytes(CS_GROUPS * CS_TM_COLS);
    __half* W2hi = reinterpret_cast<__half*>(smem_raw);
    __half* W2lo = W2hi + CS_W;
    __half* Wchi = W2lo + CS_W;
    __half* Wclo = Wchi + CS_W;
    float* qbufs = reinterpret_cast<float*>(Wclo + CS_W);            // [groups][QBUF]
    float* b2s = qbufs + CS_GROUPS * CS_QBUF;
    float* bcs = b2s + H;
    float* w3s = bcs + H;
    float* w1rs = w3s + H;
    float* w1es = w1rs + H;
    int* srow_all = reinterpret_cast<int*>(w1es + DISTEGNN_MAX_EDGE_ATTR * H);      // [groups][2][128]
    uint32_t* rmask_all = reinterpret_cast<uint32_t*>(srow_all + CS_GROUPS * 2 * TILE_M);   // [groups][4]
    int* nidx_all = reinterpret_cast<int*>(rmask_all + CS_GROUPS * 4);              // [groups][2][CS_IDX]
    uint32_t* oflag_all = reinterpret_cast<uint32_t*>(nidx_all + CS_GROUPS * 2 * CS_IDX);   // [groups][2][8]
    float* rowmax_all = reinterpret_cast<float*>(oflag_all + CS_GROUPS * 2 * CS_WARPS);      // [groups][2][128]
    float* xs_all = rowmax_all + CS_GROUPS * 2 * TILE_M;                                       // [groups][128][8]
    uint64_t* bars = reinterpret_cast<uint64_t*>(xs_all + CS_GROUPS * TILE_M * 8);             // [groups]

    const int tid = threadIdx.x;
    const int grp = tid >> 8;              // tile group 0 .. CS_GROUPS-1
    const int tg = tid & 255;              // thread inside the group
    const int wk = tg >> 5;                // warp inside the group 0..7
    const int lane = tid & 31;
    const int wq = wk & 3;                 // row quarter
    const int hf = wk >> 2;                // column half owned by this thread
    const int r = 32 * wq + lane;          // edge (row) of the tile shared with the thread of the other half
    const int cb = 32 * hf;                // first owned column
    const int A = AT >= 0 ? AT : a.A;
    const bool normalize = a.flags & DISTEGNN_FLAG_NORMALIZE;
    constexpr bool need_m = !LASTL;        // the last layer only moves coordinates (DISTEGNN_FLAG_LAST): no segment sum of m

    // ---- one-time setup -------------------------------------------------------------------------
    tc16::stage_weight<CS_THREADS>(W2hi, W2lo, a.w2, 0, 64, tid, SILU_T_IN);   // t2 = SILU_T_IN·(a1·W2ᵀ + b2)
    tc16::stage_weight<CS_THREADS>(Wchi, Wclo, a.wc, 0, 64, tid);   // t3 = s2·Wcᵀ + SILU_T_IN·bc  (SILU_T_IN·SILU_T_OUT = 1)
    if (tid < H) {
        b2s[tid] = a.b2[tid] * SILU_T_IN;
        bcs[tid] = a.bc[tid] * SILU_T_IN;
        w3s[tid] = a.w3[tid] * SILU_T_OUT;
        w1rs[tid] = a.w1r[tid];
    }
    for (int i = tid; i < DISTEGNN_MAX_EDGE_ATTR * H; i += CS_THREADS) w1es[i] = i < A * H ? a.w1e[i] : 0.f;
    if (tid == 0) {
        for (int i = 0; i < CS_GROUPS; ++i) mbar_init(&bars[i], 1);
        fence_mbar_init();
    }
    fence_proxy_async_smem();
    __syncthreads();

    const uint32_t col0 = (uint32_t)(grp * CS_TM_COLS);
    const uint32_t lane_off = ((uint32_t)(32 * wq)) << 16;
    const uint32_t tA_hi = lane_off + col0 + 16u * hf, tA_lo = lane_off + col0 + 32u + 16u * hf;   // own 16 words each
    const uint32_t tD = lane_off + col0 + 64u + 32u * hf;                                          // own 32 columns
    float* qb = qbufs + grp * CS_QBUF;
    float* myq = qb + cs_qoff(r) + cb;                           // own half row of the staging buffer
    int* srow2 = srow_all + grp * 2 * TILE_M;
    uint32_t* rmask = rmask_all + grp * 4;
    int* nidx = nidx_all + grp * 2 * CS_IDX;
    uint32_t* oflag = oflag_all + grp * 2 * CS_WARPS;
    float* rowmax = rowmax_all + grp * 2 * TILE_M;
    float* xs = xs_all + grp * TILE_M * 8 + 8 * r;               // (x_row, x_col) of edge r of the next tile
    uint64_t* qbar = bars + grp;
    const uint32_t bar_id = 1 + grp;

    const int64_t nE = a.E_dev ? min((int64_t)__ldg(a.E_dev), a.E) : a.E;     // valid edges (<= the host-side bound)
    const int64_t num_tiles = (nE + TILE_M - 1) / TILE_M;
    const int64_t stride = (int64_t)gridDim.x * CS_GROUPS;
    int64_t tile = (int64_t)blockIdx.x * CS_GROUPS + grp;

    // D[128x64] = A·Wᵀ with the three split products: warpgroup hf computes rows 64·hf .. +63; the group barrier of
    // mma_done() publishes all of D
    auto issue_mma = [&](const __half* whi, const __half* wlo) {
        tc16::mma_f16x3<CS_LBO>(col0 + 64u, col0, col0 + 32u, make_b_desc(smem_u32(whi), CS_LBO, 128),
                                make_b_desc(smem_u32(wlo), CS_LBO, 128), 1, false, hf, 1);
    };
    auto mma_done = [&]() { named_bar(bar_id, CS_GROUP); };
    // any flag of the group set?  (read after the group barrier that follows the flag writes)
    auto group_flag = [&](int stage) {
        const uint4 f0 = *reinterpret_cast<const uint4*>(oflag + stage * CS_WARPS);
        const uint4 f1 = *reinterpret_cast<const uint4*>(oflag + stage * CS_WARPS + 4);
        return ((f0.x | f0.y | f0.z | f0.w) | (f1.x | f1.y | f1.z | f1.w)) != 0u;
    };
    // start the copy of tile tl's (row, col, edge_attr) of edge r into index buffer `b` (threads of half 0)
    auto stage_idx = [&](int64_t tl, int b) {
        const int64_t e = tl * TILE_M + r;
        if (tl < num_tiles && e < nE) {
            int* dst = nidx + b * CS_IDX;
            cp_async4(dst + r, a.row + e);
            cp_async4(dst + TILE_M + r, a.col + e);
            if (AT == 1) cp_async4(dst + 2 * TILE_M + 2 * r, a.ea + e);
            if (AT == 2) cp_async8(dst + 2 * TILE_M + 2 * r, a.ea + e * 2);
        }
        cp_async_commit();
    };

    ulonglong2 p_first[2];        // the first 8 own columns of P[row] of the tile about to be processed
    p_first[0] = p_first[1] = make_ulonglong2(0ull, 0ull);
    int row_c = -1;
    float dx = 0.f, dy = 0.f, dz = 0.f, radial = 0.f;
    float ea_c[AMAX];
#pragma unroll
    for (int k = 0; k < AMAX; ++k) ea_c[k] = 0.f;
    auto set_geometry = [&](float4 xi, float4 xj) {
        dx = xi.x - xj.x; dy = xi.y - xj.y; dz = xi.z - xj.z;
        radial = dx * dx + dy * dy + dz * dz;
        if (normalize) {
            const float inv = 1.0f / (sqrtf(radial) + 1e-8f);
            dx *= inv; dy *= inv; dz *= inv;
        }
    };

    // Δx·φ_half summed over runs of equal destination row inside the warp (rows are sorted), one RED.ADD triple per run
    auto reduce_aggx = [&](float sx, float sy, float sz, int rw) {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int rk = __shfl_up_sync(FULL, rw, o);
            const float ox = __shfl_up_sync(FULL, sx, o), oy = __shfl_up_sync(FULL, sy, o), oz = __shfl_up_sync(FULL, sz, o);
            if (lane >= o && rk == rw) { sx += ox; sy += oy; sz += oz; }
        }
        const int rnext = __shfl_down_sync(FULL, rw, 1);
        if (rw >= 0 && (lane == 31 || rnext != rw)) {
            float* dst = a.agg_x + (size_t)rw * 4;
            atomicAdd(dst + 0, sx);
            atomicAdd(dst + 1, sy);
            atomicAdd(dst + 2, sz);
        }
    };

    // ---- prologue: first tile read directly, its Q rows fetched, the second tile's indices staged ---------------
    if (tile < num_tiles) {
        const int64_t e = tile * TILE_M + r;
        int col_c = 0;
        if (e < nE) {
            row_c = __ldg(a.row + e);
            col_c = __ldg(a.col + e);
#pragma unroll
            for (int k = 0; k < AMAX; ++k)
                if (AT < 0 ? k < A : true) ea_c[k] = (k < A) ? __ldg(a.ea + e * A + k) : 0.f;
        }
        if (tg == 0) {
            const int64_t nvalid = min((int64_t)TILE_M, nE - tile * TILE_M);
            mbar_expect_tx(qbar, (uint32_t)nvalid * (H * 4));
        }
        if (hf == 0 && row_c >= 0) bulk_g2s(qb + cs_qoff(r), a.Q + (size_t)col_c * H, H * 4, qbar);
        set_geometry(ldg4(a.x4 + (size_t)max(row_c, 0) * 4), ldg4(a.x4 + (size_t)col_c * 4));
        p_first[0] = __ldg(reinterpret_cast<const ulonglong2*>(a.P + (size_t)max(row_c, 0) * H + cb));
        p_first[1] = __ldg(reinterpret_cast<const ulonglong2*>(a.P + (size_t)max(row_c, 0) * H + cb + 4));
    }

    for (int it = 0; tile < num_tiles; ++it, tile += stride) {
        const int64_t ntile = tile + stride;
        const int nb = (it + 1) & 1;                         // index buffer that holds / will hold the next tile
        const int* nrow_s = nidx + nb * CS_IDX;
        const int* ncol_s = nrow_s + TILE_M;
        const float* nea_s = reinterpret_cast<const float*>(ncol_s + TILE_M);
        const bool nvalid_r = ntile < num_tiles && ntile * TILE_M + r < nE;     // edge r of the next tile exists
        // destination rows of this tile's edges, per tile parity: a fast warp writes the NEXT tile's rows (stage 1) while a slow
        // one may still read this tile's in the segment sum — no group barrier separates the two any more
        int* srow = srow2 + (it & 1) * TILE_M;

        // ---- stage 1: a1 = SiLU(P_i + Q_j + w_r·r + W_e·a), own 32 columns -> fp16 hi/lo -> A ------------------
        mbar_wait(qbar, (uint32_t)(it & 1));
        __syncwarp();
        if (hf == 0) stage_idx(ntile, nb);
        const float* prow = a.P + (size_t)max(row_c, 0) * H + cb;
        float qmax = 0.f;
        const f32x2 rad2 = bc2(radial);
        // P values of chunk j (8 columns) arrive as `pp`: on the hot path they were requested one chunk earlier
        auto pre_math = [&](int j, const ulonglong2 (&pp)[2], f32x2 (&v)[4], auto safe) {
#pragma unroll
            for (int j4 = 0; j4 < 2; ++j4) {
                const int cc = 8 * j + 4 * j4;               // relative to the own half
                const ulonglong2 qq = *reinterpret_cast<const ulonglong2*>(myq + cc);
                const ulonglong2 wr = *reinterpret_cast<const ulonglong2*>(w1rs + cb + cc);
                f32x2 p0 = fma2(rad2, wr.x, add2(pp[j4].x, qq.x)), p1 = fma2(rad2, wr.y, add2(pp[j4].y, qq.y));
#pragma unroll
                for (int k = 0; k < AMAX; ++k)
                    if (AT < 0 || k < A) {     // AT < 0: ea_c[k] = 0 and zero weight rows beyond A (a predicated FMA
                                               // chain crashes ptxas 12.9 at -O2 and above)
                        const ulonglong2 we = *reinterpret_cast<const ulonglong2*>(w1es + k * H + cb + cc);
                        const f32x2 e2 = bc2(ea_c[k]);
                        p0 = fma2(e2, we.x, p0);
                        p1 = fma2(e2, we.y, p1);
                    }
                silu4p<decltype(safe)::value>(p0, p1, qmax);
                v[2 * j4] = p0;
                v[2 * j4 + 1] = p1;
            }
        };
        auto load_p = [&](const float* base, int j, ulonglong2 (&pp)[2]) {
            pp[0] = __ldg(reinterpret_cast<const ulonglong2*>(base + 8 * j));
            pp[1] = __ldg(reinterpret_cast<const ulonglong2*>(base + 8 * j + 4));
        };
        auto pre_chunk = [&](int j, f32x2 (&v)[4], auto safe) {      // cold paths: load, then compute
            ulonglong2 pp[2];
            load_p(prow, j, pp);
            pre_math(j, pp, v, safe);
        };
        float inv_s1 = 1.0f;
        {
            __half2 mx = __floats2half2_rn(0.f, 0.f);
            // P[row] comes from L2 (the rows of a tile are few, but L1 keeps little between tiles): chunk 0 was requested at
            // the end of the previous tile (p_first), chunk j+1 is requested before the math of chunk j
            ulonglong2 pq[2][2];
            pq[0][0] = p_first[0];
            pq[0][1] = p_first[1];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                uint32_t hi[4], lo[4];
                if (j < 3) load_p(prow, j + 1, pq[(j + 1) & 1]);
                pre_math(j, pq[j & 1], v, kFast);
                split8<false, false>(v, 1.0f, hi, lo, mx);
                tm_st4(tA_hi + 4 * j, hi);
                tm_st4(tA_lo + 4 * j, lo);
            }
            const bool bad = __any_sync(FULL, row_overflow8<false>(mx) || silu_q_overflow(qmax));
            if (lane == 0) oflag[wk] = bad ? 1u : 0u;
        }
        tm_st_fence();
        if (hf == 0) {
            srow[r] = row_c;
            cp_async_wait_all();               // the staged indices of the next tile: visible to the group after the barrier
        }
        named_bar(bar_id, CS_GROUP);           // A complete; D of the previous tile fully read by the whole group
        if (group_flag(0)) {                   // cold: some row leaves the fp16 range, or the SiLU batch guard fired
            float fm = 0.f, sc;
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                pre_chunk(j, v, kSafe);
                fm = max8<false>(v, fm);
            }
            rowmax[hf * TILE_M + r] = fm;
            named_bar(bar_id, CS_GROUP);
            tc16::range_scale(fmaxf(rowmax[r], rowmax[TILE_M + r]), sc, inv_s1);
            __half2 mx = __floats2half2_rn(0.f, 0.f);
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                uint32_t hi[4], lo[4];
                pre_chunk(j, v, kSafe);
                split8<true, false>(v, sc, hi, lo, mx);
                tm_st4(tA_hi + 4 * j, hi);
                tm_st4(tA_lo + 4 * j, lo);
            }
            tm_st_fence();
            named_bar(bar_id, CS_GROUP);
        }

        // ---- MMA 1; then run masks and the next tile's P rows towards L1 --------------------------------------
        issue_mma(W2hi, W2lo);
        if (hf == 0) {   // bit i of rmask[q] = edge 32q+i starts a new run of equal destination rows
            const int prev = r > 0 ? srow[r - 1] : -2;
            const uint32_t starts = __ballot_sync(FULL, prev != row_c);
            if (lane == 0) rmask[wq] = starts;
            if (nvalid_r) {        // coordinates of the next tile's edge: one gather per edge, consumed after stage 3
                cp_async16(xs, a.x4 + (size_t)nrow_s[r] * 4);
                cp_async16(xs + 4, a.x4 + (size_t)ncol_s[r] * 4);
            }
            cp_async_commit();
        }
        if (nvalid_r) prefetch_l1(a.P + (size_t)nrow_s[r] * H + cb);      // one 128-byte line per thread

        mma_done();

        // ---- stage 2: m = SiLU(D/s + b2), own 32 columns -> shared (segment sum) and fp16 hi/lo -> A -------------
        qmax = 0.f;
        auto m_math = [&](int j, const uint32_t (&d)[8], f32x2 (&v)[4], bool store, auto safe) {
            const f32x2 is2 = bc2(inv_s1);
#pragma unroll
            for (int j4 = 0; j4 < 2; ++j4) {
                const int cc = 8 * j + 4 * j4;
                const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(b2s + cb + cc);
                f32x2 m0 = fma2(pk2u(d[4 * j4 + 0], d[4 * j4 + 1]), is2, bb.x);
                f32x2 m1 = fma2(pk2u(d[4 * j4 + 2], d[4 * j4 + 3]), is2, bb.y);
                silu4t<decltype(safe)::value>(m0, m1, qmax);     // (m0, m1) = SILU_T_IN·m: the flush and Wc's consumer undo it
                if (store) *reinterpret_cast<ulonglong2*>(myq + cc) = make_ulonglong2(m0, m1);
                v[2 * j4] = m0;
                v[2 * j4 + 1] = m1;
            }
        };
        auto m_chunk = [&](int j, f32x2 (&v)[4], bool store, auto safe) {      // cold paths: load, wait, compute
            uint32_t d[8];
            tm_ld8(tD + 8 * j, d);
            m_math(j, d, v, store, safe);
        };
        float inv_s2 = 1.0f;
        {
            __half2 mx = __floats2half2_rn(0.f, 0.f);
#pragma unroll 2
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                uint32_t hi[4], lo[4];
                m_chunk(j, v, need_m, kFast);
                split8<false, true>(v, 1.0f, hi, lo, mx);      // t-domain values: ≤ 0.41, unbounded below
                tm_st4(tA_hi + 4 * j, hi);
                tm_st4(tA_lo + 4 * j, lo);
            }
            const bool bad = __any_sync(FULL, row_overflow8<true>(mx) || silu_q_overflow(qmax));
            if (lane == 0) oflag[CS_WARPS + wk] = bad ? 1u : 0u;
        }
        tm_st_fence();
        if (hf == 0) cp_async_wait_all();      // the staged coordinates: visible to both halves after the barrier
        named_bar(bar_id, CS_GROUP);           // m tile visible in shared, A complete, D fully read
        if (group_flag(1)) {                   // cold
            float fm = 0.f, sc;
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                m_chunk(j, v, need_m, kSafe);  // also rewrites the m row in shared memory
                fm = max8<true>(v, fm);
            }
            rowmax[hf * TILE_M + r] = fm;
            named_bar(bar_id, CS_GROUP);
            tc16::range_scale(fmaxf(rowmax[r], rowmax[TILE_M + r]), sc, inv_s2);
            __half2 mx = __floats2half2_rn(0.f, 0.f);
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                f32x2 v[4];
                uint32_t hi[4], lo[4];
                m_chunk(j, v, false, kSafe);
                split8<true, true>(v, sc, hi, lo, mx);
                tm_st4(tA_hi + 4 * j, hi);
                tm_st4(tA_lo + 4 * j, lo);
            }
            tm_st_fence();
            named_bar(bar_id, CS_GROUP);
        }

        // ---- MMA 2 (φ head) overlapped with the segment sum of m ----------------------------------------------
        issue_mma(Wchi, Wclo);
        if (need_m) {
            // warp wk <-> edges 16wk .. 16wk+15 of the tile, lane <-> columns 2·lane, 2·lane+1: per edge one LDS.64
            // and one pair add; the run structure is warp-uniform, one RED.v2 per run and lane
            const float* colp = qb + cs_qoff(16 * wk) + 2 * lane;     // 16·wk is a multiple of 8: row e of the warp sits at cs_qoff(e)
            // one straight pass over the warp's 16 edges; bit e of M = edge e starts a new run of equal destination rows
            // (warp-uniform), where the running sum is flushed with one RED.v2 per lane
            const uint32_t M = (rmask[wk >> 1] >> (16 * (wk & 1))) & 0xffffu;
            const int* srw = srow + 16 * wk;
            auto flush = [&](f32x2 acc, int e_last) {
                const int rr = srw[e_last];
                if (rr >= 0) {
                    float v0, v1;
                    upk2(mul2(acc, bc2(SILU_T_OUT)), v0, v1);
                    red_add_v2(a.agg_m + (size_t)rr * H + 2 * lane, v0, v1);
                }
            };
            f32x2 s0 = *reinterpret_cast<const f32x2*>(colp);
            if ((M >> 1) == 0u) {       // no run starts inside the warp's 16 edges (about half of the warps at degree 20):
                f32x2 s1 = *reinterpret_cast<const f32x2*>(colp + cs_qoff(1));     // two plain chains, no per-edge test
#pragma unroll
                for (int e = 2; e < 16; e += 2) {
                    s0 = add2(s0, *reinterpret_cast<const f32x2*>(colp + cs_qoff(e)));
                    s1 = add2(s1, *reinterpret_cast<const f32x2*>(colp + cs_qoff(e + 1)));
                }
                flush(add2(s0, s1), 15);
            } else {
#pragma unroll
                for (int e = 1; e < 16; ++e) {
                    const f32x2 v = *reinterpret_cast<const f32x2*>(colp + cs_qoff(e));
                    if ((M >> e) & 1u) {
                        flush(s0, e - 1);
                        s0 = v;
                    } else {
                        s0 = add2(s0, v);
                    }
                }
                flush(s0, 15);
            }
        }
        // The rows a warp refills (16·wk .. +15) were last read by that same warp (segment sum) — their stage-1 / stage-2
        // accesses by the owner threads lie before the previous group barrier — so no group barrier is needed here: warp-level
        // ordering of the generic accesses before the async-proxy refill is enough.
        fence_proxy_async_smem();
        __syncwarp();

        // ---- Q rows of the next tile, addresses from the staged indices ----------------------------------------------------
        if (ntile < num_tiles) {
            if (tg == 0) {
                const int64_t nvalid = min((int64_t)TILE_M, nE - ntile * TILE_M);
                mbar_expect_tx(qbar, (uint32_t)nvalid * (H * 4));
            }
            const int rr = 16 * wk + (lane & 15);
            if (lane < 16 && ntile * TILE_M + rr < nE)
                bulk_g2s(qb + rr * CS_QROW, a.Q + (size_t)ncol_s[rr] * H, H * 4, qbar);
        }
        const int row_n = nvalid_r ? nrow_s[r] : -1;      // destination row of the next tile's edge

        mma_done();

        // ---- stage 3: φ_half = w3·SiLU(D/s + bc) over the own columns; Δx·φ_half summed per destination row -------
        f32x2 ph01, ph23;
        qmax = 0.f;
        auto phi_pass = [&](auto safe) {
            ph01 = bc2(0.f);
            ph23 = bc2(0.f);
            const f32x2 is2 = bc2(inv_s2);
            auto phi_math = [&](int j, const uint32_t (&d)[8]) {
#pragma unroll
                for (int j4 = 0; j4 < 2; ++j4) {
                    const int cc = cb + 8 * j + 4 * j4;
                    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(bcs + cc);
                    const ulonglong2 ww = *reinterpret_cast<const ulonglong2*>(w3s + cc);
                    f32x2 s0 = fma2(pk2u(d[4 * j4 + 0], d[4 * j4 + 1]), is2, bb.x);
                    f32x2 s1 = fma2(pk2u(d[4 * j4 + 2], d[4 * j4 + 3]), is2, bb.y);
                    silu4t<decltype(safe)::value>(s0, s1, qmax);
                    ph01 = fma2(s0, ww.x, ph01);
                    ph23 = fma2(s1, ww.y, ph23);
                }
            };
#pragma unroll 2
            for (int j = 0; j < 4; ++j) {
                uint32_t d[8];
                tm_ld8(tD + 8 * j, d);
                phi_math(j, d);
            }
        };
        phi_pass(kFast);
        if (__any_sync(FULL, silu_q_overflow(qmax))) phi_pass(kSafe);      // cold (warp-local: no scale)
        float ph0, ph1, ph2, ph3;
        upk2(ph01, ph0, ph1);
        upk2(ph23, ph2, ph3);
        const float phi = (ph0 + ph1) + (ph2 + ph3);
        {   // the next tile's first P chunk: in flight across the shuffle reduction, the roll and the wait for the Q rows
            const float* pn = a.P + (size_t)max(row_n, 0) * H + cb;
            p_first[0] = __ldg(reinterpret_cast<const ulonglong2*>(pn));
            p_first[1] = __ldg(reinterpret_cast<const ulonglong2*>(pn + 4));
        }
        reduce_aggx(dx * phi, dy * phi, dz * phi, row_c);

        // ---- roll the next tile's edge into place -------------------------------------------------------------
        row_c = row_n;
#pragma unroll
        for (int k = 0; k < AMAX; ++k) ea_c[k] = 0.f;
        if (nvalid_r) {
            if (AT == 1) ea_c[0] = nea_s[2 * r];
            if (AT == 2) {
                const float2 v = *reinterpret_cast<const float2*>(nea_s + 2 * r);
                ea_c[0] = v.x;
                ea_c[AMAX - 1] = v.y;
            }
            if (!kEaStaged) {
                const int64_t e = ntile * TILE_M + r;
#pragma unroll
                for (int k = 0; k < AMAX; ++k)
                    if (k < A) ea_c[k] = __ldg(a.ea + e * A + k);
            }
        }
        float4 xi_n = make_float4(0.f, 0.f, 0.f, 0.f), xj_n = xi_n;
        if (nvalid_r) {
            xi_n = *reinterpret_cast<const float4*>(xs);
            xj_n = *reinterpret_cast<const float4*>(xs + 4);
        }
        set_geometry(xi_n, xj_n);
    }
}

}  // namespace degnn

extern "C" int distegnn_edge_layer_fwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                       const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                       const float* x4, const float* P, const float* Q,
                                       const float* layer_params, float* agg_m, float* agg_x,
                                       const int32_t* n_edges_dev, void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_edges == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_edges > 0, "negative size");
    DEGNN_CHECK_ARG(row && col && x4 && P && Q && layer_params && agg_x, "null pointer");
    DEGNN_CHECK_ARG(A == 0 || edge_attr_sorted, "null edge_attr with edge_attr_nf > 0");
    DEGNN_CHECK_ARG((flags & DISTEGNN_FLAG_LAST) || agg_m, "null agg_m");
    Layout L = make_layout(A, C, Na);
    EdgeCsArgs a;
    a.N = n_nodes; a.E = n_edges; a.E_dev = n_edges_dev; a.A = A; a.flags = flags & 0xffffu;
    a.row = row; a.col = col; a.ea = edge_attr_sorted; a.x4 = x4; a.P = P; a.Q = Q;
    a.w1r = layer_params + L.off[DISTEGNN_P_E_W1R];
    a.w1e = layer_params + L.off[DISTEGNN_P_E_W1E];
    a.w2 = layer_params + L.off[DISTEGNN_P_E_W2];
    a.b2 = layer_params + L.off[DISTEGNN_P_E_B2];
    a.wc = layer_params + L.off[DISTEGNN_P_E_WC];
    a.bc = layer_params + L.off[DISTEGNN_P_E_BC];
    a.w3 = layer_params + L.off[DISTEGNN_P_E_W3];
    a.agg_m = agg_m; a.agg_x = agg_x;
    const int64_t tiles = (n_edges + TILE_M - 1) / TILE_M;
    int64_t grid = (tiles + CS_GROUPS - 1) / CS_GROUPS;
    if (grid > sm_count()) grid = sm_count();
    auto launch = [&](auto kern) {
        ensure_dynamic_smem((const void*)kern, (int)CS_SMEM_BYTES);
        kern<<<(unsigned)grid, CS_THREADS, CS_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    };
    const bool last = flags & DISTEGNN_FLAG_LAST;
    switch (A) {
        case 0: last ? launch(edge_layer_cs_kernel<0, true>) : launch(edge_layer_cs_kernel<0, false>); break;
        case 1: last ? launch(edge_layer_cs_kernel<1, true>) : launch(edge_layer_cs_kernel<1, false>); break;
        case 2: last ? launch(edge_layer_cs_kernel<2, true>) : launch(edge_layer_cs_kernel<2, false>); break;
        default: last ? launch(edge_layer_cs_kernel<-1, true>) : launch(edge_layer_cs_kernel<-1, false>); break;
    }
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
