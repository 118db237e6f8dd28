// Real<->real edge stage — production kernel behind distegnn_edge_layer_fwd.
// Same outputs as testing/edge_layer.cu (fp32-FMA twin, distegnn_edge_layer_fwd_simt); replaces reference models/FastEGNN.py:237-246 (coord2radial), 144-150 (edge_model), 169-177 (edge part of
// coord_model_vel), 206 (edge part of node_model) and the scatter_add_ of :322-337 (twins models/basic.py:22-66).
//
// One CTA per SM, CS_WG warpgroups, each an independent pipeline: a warpgroup grid-strides over its own tiles of 64 edges
// and shares no barrier with the other warpgroups, so that while one waits on its GEMMs or its loads the others issue
// their SiLU epilogues.  Everything but the wgmma itself is warp-local: warp w of the warpgroup owns edges 16w .. 16w+15
// of the tile, which are exactly the rows of the m64n64 accumulator fragment it holds (tile_mma.cuh); thread (g = lane/4,
// q = lane%4) owns rows g and g+8 of the warp, columns 8j + 2q + {0,1} (j = 0..7).  The A operands and the accumulators
// stay in registers; only the weights (W2, Wc hi/lo) and the neighbour rows Q[col] are in shared memory.  Per tile
// (numerics as in the other tensor-core kernels: fp16 2-term split, per-row power-of-two range rescue, one reciprocal
// per four SiLUs with a stage-level guard; the rescue and the guard are tc16.cuh encode_rows, the φ head phi_head_t):
//   stage 1  a1 = SiLU(P[row] + Q[col] + w_r·r + W_e·a) -> fp16 hi/lo A fragments                MMA 1: D = a1·W2ᵀ
//   stage 2  m = SiLU(D + b2) -> fp32 into the warp's staging rows (segment sum) + hi/lo A fragments   MMA 2: D = m·Wcᵀ
//            segment sum of m over destination rows while MMA 2 runs (lane <-> column pair, one RED.v2 per run)
//   stage 3  φ = w3·SiLU(D + bc) per row (quad shuffles); Δx·φ summed over runs of equal row, RED.ADD
// The range rescue needs one scale per row: the four lanes of a quad share a row, so its maximum is two shuffles away and
// the cold path is taken per warp (__any_sync); every path reconverges before the warpgroup-collective wgmma.
// Everything a tile needs from memory is requested one tile ahead, per warp, as one cp.async commit group issued at the
// start of tile i and waited for at its end (a __syncwarp then publishes every lane's copies to the warp):
//   Q[col] rows of tile i+1           16-byte cp.async by all 32 lanes, two rows per pass (staging double buffered)
//   x[row], x[col] of tile i+1        read at the end of tile i
//   (row, col, edge_attr) of tile i+2 moved to registers at the end of tile i
//   P[row] of tile i+1                prefetched towards L1 at the start of tile i (rows are contiguous: a tile has few)
// Tile numbers and edge ids are int32: the host entry bounds the edge count (edge_layer_fwd).
// Stages 2 and 3 run in the "t domain" (common.cuh silu4t): −log2(e) is folded into W2 and the biases, −ln 2 into w3 and
// the segment-sum flush, so the SiLU never forms its exponent argument explicitly.
// Edge order: the one thing the kernel needs is that the edges of a destination row are contiguous (the run masks compare
// neighbouring rows; the deterministic slots compare row[e0 - 1] with the slice's first row).  The rows themselves may come
// in any order: the cached graph stores them in a spatial order (DESIGN §3), graphs from shards in id order.
#include <cuda_fp16.h>
#include <string.h>

#include "common.cuh"
#include "det.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct EdgeCsArgs {
    int64_t N;
    int E;                  // < 2^31 - 64 (edge_layer_fwd)
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
    float* slots;   // deterministic mode: one DET_EDGE_SLOT-float slot per 16-edge slice (det.cuh)
};

// 4 warpgroups = 16 warps per SM: 128 registers per thread (ptxas: no spills), 196 KB of shared memory
constexpr int CS_WG = 4;
constexpr int CS_THREADS = 128 * CS_WG, CS_WARPS = CS_THREADS / 32;
constexpr int CS_TILE = 64;                               // edges per warpgroup tile
// row pitch of the staging rows (floats): 72 = conflict-free LDS.64 / STS.64 in the accumulator fragment pattern
// (rows g, columns 2q: banks 8g + 2q) and in the segment sum's row pattern
constexpr int CS_QROW = 72;
constexpr int CS_WBUF = 16 * CS_QROW;                     // one staging buffer of a warp: its 16 edges
constexpr int CS_IDX = 64;                                // staged ints per warp: row 16 | col 16 | edge_attr 16x2
constexpr int CS_W = 64 * 64;                             // fp16 elements per weight matrix (8 KB)
constexpr int CS_SMEM_BYTES = 4 * CS_W * 2                // W2 hi/lo, Wc hi/lo
                              + (4 * H + DISTEGNN_MAX_EDGE_ATTR * H) * 4   // b2, bc, w3, w1r, w1e
                              + CS_WARPS * 2 * CS_WBUF * 4                // Q rows / m, double buffered
                              + CS_WARPS * CS_IDX * 4                     // indices of the tile after next
                              + CS_WARPS * 16 * 8 * 4;                    // x[row], x[col] of the next tile
constexpr uint32_t CS_LBO = 1024;                         // fp16 K-major no-swizzle, N = 64

// DET (deterministic mode, det.cuh): the partial of every run is stored, not added.  The run of a row whose first edge lies
// in the warp's 16-edge slice goes to the row itself; the slice's head run, when it continues a row of the slice before,
// goes to the slice's slot.  distegnn_edge_combine_det then adds the slots of each row in slice order.
template <int AT, bool LASTL, bool DET>
__global__ void __launch_bounds__(CS_THREADS, 1) edge_layer_cs_kernel(const EdgeCsArgs a) {
    using namespace tmma;
    constexpr int AMAX = AT >= 0 ? (AT > 0 ? AT : 1) : DISTEGNN_MAX_EDGE_ATTR;
    constexpr int AR = (AT == 1 || AT == 2) ? AT : 0;     // edge attributes staged a tile ahead and carried in registers
    constexpr bool need_m = !LASTL;        // the last layer only moves coordinates (DISTEGNN_FLAG_LAST): no segment sum of m
    __half* W2hi = reinterpret_cast<__half*>(degnn_dyn_smem);
    __half* W2lo = W2hi + CS_W;
    __half* Wchi = W2lo + CS_W;
    __half* Wclo = Wchi + CS_W;
    float* b2s = reinterpret_cast<float*>(Wclo + CS_W);
    float* bcs = b2s + H;
    float* w3s = bcs + H;
    float* w1rs = w3s + H;
    float* w1es = w1rs + H;
    float* qbufs = w1es + DISTEGNN_MAX_EDGE_ATTR * H;                          // [warps][2][16][CS_QROW]
    int* idx_all = reinterpret_cast<int*>(qbufs + CS_WARPS * 2 * CS_WBUF);     // [warps][CS_IDX]
    float* xs_all = reinterpret_cast<float*>(idx_all + CS_WARPS * CS_IDX);     // [warps][16][8]

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;
    const int wg = warp >> 2;              // warpgroup
    const int w = warp & 3;                // warp inside the warpgroup: edges 16w .. 16w+15 of its tile
    const int g = lane >> 2, q = lane & 3; // fragment rows g, g+8 of the warp; columns 8j + 2q
    const int A = AT >= 0 ? AT : a.A;
    const bool normalize = a.flags & DISTEGNN_FLAG_NORMALIZE;

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
    // staging rows of edges past the end are never loaded: keep them finite
    for (int i = tid; i < CS_WARPS * 2 * CS_WBUF / 4; i += CS_THREADS)
        reinterpret_cast<float4*>(qbufs)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    fence_proxy_async_smem();
    __syncthreads();

    float* qb = qbufs + warp * 2 * CS_WBUF;
    int* nidx = idx_all + warp * CS_IDX;
    float* xs = xs_all + warp * 16 * 8 + 8 * (lane & 15);     // (x_row, x_col) of edge `lane` of the next tile
    // per-thread bases of the row gathers, opaque to ptxas: a row address is then one IMAD.WIDE.U32 (row id x row bytes +
    // base) instead of a 64-bit re-derivation of array + column offset each time
    const float* Pq = a.P + 2 * q;                             // the thread's columns of P rows
    asm("" : "+l"(Pq));
    const uint64_t bW2hi = make_desc(smem_u32(W2hi), CS_LBO, 128), bW2lo = make_desc(smem_u32(W2lo), CS_LBO, 128);
    const uint64_t bWchi = make_desc(smem_u32(Wchi), CS_LBO, 128), bWclo = make_desc(smem_u32(Wclo), CS_LBO, 128);

    const int nE = a.E_dev ? min(__ldg(a.E_dev), a.E) : a.E;     // valid edges (<= the host-side bound)
    const int num_tiles = (nE + CS_TILE - 1) / CS_TILE;
    const int stride = gridDim.x * CS_WG;
    int tile = blockIdx.x * CS_WG + wg;

    // lanes 0..15 carry the per-edge state of the warp's 16 edges; lanes 16..31 carry row -1
    auto edge_of = [&](int tl) { return tl * CS_TILE + 16 * w + lane; };
    auto has_edge = [&](int tl) { return lane < 16 && tl < num_tiles && edge_of(tl) < nE; };
    // Q rows of the warp's 16 edges into staging buffer b (cp.async, the caller commits): pass k copies edges 2k and 2k + 1,
    // lane L its 16-byte chunk L & 15 of edge 2k + (L >> 4).  col_e = the edge's col on lanes 0..15, -1 for no edge.
    // Rows of edges past the end are not copied: they keep what the buffer held (zeros, or m of an earlier tile), finite;
    // the deterministic mode masks them in stage 1 (oka / okb).  Zero-filling them instead would change which rows take
    // the default mode's warp-wide cold paths, and with it the bits of its valid rows.
    auto fetch_q = [&](int b, int col_e) {
        // lanes 16 + j hold the col of edge j + 1, so that one 16-lane shuffle per pass serves both halves of the warp
        const int cols = __shfl_sync(FULL, col_e, (lane & 15) + (lane >> 4));
        const uint32_t dst = smem_u32(qb + b * CS_WBUF + (lane >> 4) * CS_QROW + 4 * (lane & 15));
        const char* src = reinterpret_cast<const char*>(a.Q + 4 * (lane & 15));
        asm("" : "+l"(src));                   // opaque, as Pq
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = __shfl_sync(FULL, cols, 2 * k, 16);
            if (c >= 0) cp_async16(dst + 2 * k * CS_QROW * 4, src + (size_t)(uint32_t)c * (H * 4));
        }
    };

    int row_c = -1;
    float dx = 0.f, dy = 0.f, dz = 0.f, radial = 0.f;
    auto set_geometry = [&](float4 xi, float4 xj) {
        dx = xi.x - xj.x; dy = xi.y - xj.y; dz = xi.z - xj.z;
        radial = dx * dx + dy * dy + dz * dz;
        if (normalize) {
            const float inv = 1.0f / (sqrtf(radial) + 1e-8f);
            dx *= inv; dy *= inv; dz *= inv;
        }
    };
    float ea_c[AR > 0 ? AR : 1], n_ea[AR > 0 ? AR : 1];
#pragma unroll
    for (int k = 0; k < (AR > 0 ? AR : 1); ++k) ea_c[k] = n_ea[k] = 0.f;
    int n_row = -1, n_col = 0;             // the next tile's edge (n_row = -1: none)

    // ---- prologue: first tile read directly and its Q rows fetched, the second tile's indices read ------------------
    if (tile < num_tiles) {
        int col_c = 0;
        if (has_edge(tile)) {
            const int e = edge_of(tile);
            row_c = __ldg(a.row + e);
            col_c = __ldg(a.col + e);
#pragma unroll
            for (int k = 0; k < AR; ++k) ea_c[k] = __ldg(a.ea + (size_t)e * AR + k);
        }
        fetch_q(0, row_c >= 0 ? col_c : -1);
        cp_async_commit();
        set_geometry(ldg4(a.x4 + (size_t)max(row_c, 0) * 4), ldg4(a.x4 + (size_t)col_c * 4));
        if (has_edge(tile + stride)) {
            const int e = edge_of(tile + stride);
            n_row = __ldg(a.row + e);
            n_col = __ldg(a.col + e);
#pragma unroll
            for (int k = 0; k < AR; ++k) n_ea[k] = __ldg(a.ea + (size_t)e * AR + k);
        }
        cp_async_wait_all();
        __syncwarp();                          // every lane's Q rows of the first tile have landed
    }

    for (int it = 0; tile < num_tiles; ++it, tile += stride) {
        const int nntile = tile + 2 * stride;
        const int b = it & 1;
        float* qcur = qb + b * CS_WBUF;

        int cont_row = -1;                     // DET: the row this slice continues from the slice before, if any
        if constexpr (DET) {
            const int e0 = tile * CS_TILE + 16 * w;
            const int r0 = __shfl_sync(FULL, row_c, 0);
            if (r0 >= 0 && e0 > 0 && __ldg(a.row + e0 - 1) == r0) cont_row = r0;
        }
        float* const slot = DET ? a.slots + (size_t)(tile * 4 + w) * DET_EDGE_SLOT : nullptr;

        // ---- requests for the next tile (its staging buffer was released at the end of the previous tile) -------------
        fetch_q(b ^ 1, n_row >= 0 ? n_col : -1);
        if (n_row >= 0) {
            cp_async16(xs, a.x4 + (size_t)n_row * 4);
            cp_async16(xs + 4, a.x4 + (size_t)n_col * 4);
            prefetch_l1(a.P + (size_t)n_row * H);
            prefetch_l1(a.P + (size_t)n_row * H + 32);
        }
        if (has_edge(nntile)) {
            const int e = edge_of(nntile);
            cp_async4(nidx + lane, a.row + e);
            cp_async4(nidx + 16 + lane, a.col + e);
            if (AT == 1) cp_async4(nidx + 32 + 2 * lane, a.ea + e);
            if (AT == 2) cp_async8(nidx + 32 + 2 * lane, a.ea + (size_t)e * 2);
        }
        cp_async_commit();

        // ---- stage 1: a1 = SiLU(P_i + Q_j + w_r·r + W_e·a) for rows g, g+8 -> fp16 hi/lo A fragments -----------------
        const int ra = __shfl_sync(FULL, row_c, g), rb = __shfl_sync(FULL, row_c, g + 8);
        const float rada = __shfl_sync(FULL, radial, g), radb = __shfl_sync(FULL, radial, g + 8);
        float eaa[AMAX], eab[AMAX];
#pragma unroll
        for (int k = 0; k < AMAX; ++k) {
            if (AR > 0) {
                eaa[k] = __shfl_sync(FULL, ea_c[k < AR ? k : 0], g);
                eab[k] = __shfl_sync(FULL, ea_c[k < AR ? k : 0], g + 8);
            } else if (AT < 0) {   // generic count: read in place; zero beyond A (zero weight rows there too)
                const int e = tile * CS_TILE + 16 * w + g;
                eaa[k] = (k < A && ra >= 0) ? __ldg(a.ea + (size_t)e * A + k) : 0.f;
                eab[k] = (k < A && rb >= 0) ? __ldg(a.ea + (size_t)(e + 8) * A + k) : 0.f;
            } else {
                eaa[k] = eab[k] = 0.f;
            }
        }
        const float* pa = Pq + (size_t)(uint32_t)max(ra, 0) * H;
        const float* pb = Pq + (size_t)(uint32_t)max(rb, 0) * H;
        const float* qa = qcur + g * CS_QROW + 2 * q;
        const float* qbr = qa + 8 * CS_QROW;
        // DET: rows past the edge count are zero — their staging rows and attributes are left over from earlier tiles, and
        // through the warp-wide cold-path tests they would make the bits of the valid rows depend on the tile order
        const bool oka = !DET || ra >= 0, okb = !DET || rb >= 0;
        auto pre = [&](int j, const float* prow, const float* qrow, float rad, const float (&ea)[AMAX], bool ok) {
            if (DET && !ok) return bc2(0.f);
            const int c = 8 * j + 2 * q;
            const f32x2 pp = __ldg(reinterpret_cast<const f32x2*>(prow + 8 * j));
            const f32x2 qq = *reinterpret_cast<const f32x2*>(qrow + 8 * j);
            f32x2 p = fma2(bc2(rad), *reinterpret_cast<const f32x2*>(w1rs + c), add2(pp, qq));
#pragma unroll
            for (int k = 0; k < AMAX; ++k)
                if (AT < 0 || k < A)     // AT < 0: zero attributes and weight rows beyond A (a predicated FMA chain
                                         // crashes ptxas 12.9 at -O2 and above)
                    p = fma2(bc2(ea[k]), *reinterpret_cast<const f32x2*>(w1es + k * H + c), p);
            return p;
        };
        // register i = 2j + r of a fragment array <-> row g + 8r, columns 8j + 2q + {0,1} (= accumulator pair d[2i], d[2i+1])
        uint32_t ahi[16], alo[16];
        float qmax = 0.f;
        auto silu_guard = [&] { return silu_q_overflow(qmax); };
        tc16::RowScales s1;
        tc16::encode_rows<false, true>(
            [&](int j, f32x2& va, f32x2& vb, auto pass) {
                va = pre(j, pa, qa, rada, eaa, oka);
                vb = pre(j, pb, qbr, radb, eab, okb);
                silu4p<decltype(pass)::value != tc16::FAST_PASS>(va, vb, qmax);
            },
            ahi, alo, s1, silu_guard);

        // ---- MMA 1; the run-start mask of the warp's edges while it runs --------------------------------------------
        float d[32];
        tc16::mma_f16x3_rA<CS_LBO>(d, ahi, alo, bW2hi, bW2lo);
        // bit e = edge e of the warp starts a new run of equal destination rows (rows are contiguous; warp-uniform)
        const int row_prev = __shfl_up_sync(FULL, row_c, 1);
        const uint32_t M = __ballot_sync(FULL, lane == 0 || row_prev != row_c) & 0xffffu;
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- stage 2: m = SiLU(D/s + b2) -> fp32 staging rows (segment sum) and fp16 hi/lo A fragments ----------------
        // (ma, mb) = SILU_T_IN·m: the flush and Wc's consumer undo it.  The rows are stored by the pass whose values are
        // final: the fast pass, and again by the row-max pass when the warp takes the cold path (batch guard included).
        qmax = 0.f;
        tc16::RowScales s2;
        tc16::encode_rows<false>(
            [&](int j, f32x2& ma, f32x2& mb, auto pass) {
                const f32x2 bb = *reinterpret_cast<const f32x2*>(b2s + 8 * j + 2 * q);
                ma = fma2(pk2(d[4 * j + 0], d[4 * j + 1]), bc2(s1.inv_a), bb);
                mb = fma2(pk2(d[4 * j + 2], d[4 * j + 3]), bc2(s1.inv_b), bb);
                silu4t<decltype(pass)::value != tc16::FAST_PASS>(ma, mb, qmax);
                if (need_m && decltype(pass)::value != tc16::ENCODE_PASS) {
                    *reinterpret_cast<f32x2*>(qcur + g * CS_QROW + 8 * j + 2 * q) = ma;
                    *reinterpret_cast<f32x2*>(qcur + (g + 8) * CS_QROW + 8 * j + 2 * q) = mb;
                }
            },
            ahi, alo, s2, silu_guard);

        // ---- MMA 2 (φ head) overlapped with the segment sum of m ----------------------------------------------
        tc16::mma_f16x3_rA<CS_LBO>(d, ahi, alo, bWchi, bWclo);
        if (need_m) {
            __syncwarp();                      // the warp's m rows, written in the fragment pattern, are complete
            // lane <-> columns 2·lane, 2·lane+1: per edge one LDS.64 and one pair add; one RED.v2 per run and lane
            const float* colp = qcur + 2 * lane;
            float* mrow = a.agg_m + 2 * lane;  // opaque, as Pq
            asm("" : "+l"(mrow));
            auto flush = [&](f32x2 acc, int e_last) {
                const int rr = __shfl_sync(FULL, row_c, e_last);
                if (rr >= 0) {
                    float v0, v1;
                    upk2(mul2(acc, bc2(SILU_T_OUT)), v0, v1);
                    if constexpr (DET)
                        *reinterpret_cast<float2*>(rr == cont_row ? slot + 2 * lane : mrow + (size_t)(uint32_t)rr * H) =
                            make_float2(v0, v1);
                    else
                        red_add_v2(mrow + (size_t)(uint32_t)rr * H, v0, v1);
                }
            };
            f32x2 s0 = *reinterpret_cast<const f32x2*>(colp);
            if ((M >> 1) == 0u) {       // no run starts inside the warp's 16 edges (about half of the warps at degree 20):
                f32x2 s1 = *reinterpret_cast<const f32x2*>(colp + CS_QROW);     // two plain chains, no per-edge test
#pragma unroll
                for (int e = 2; e < 16; e += 2) {
                    s0 = add2(s0, *reinterpret_cast<const f32x2*>(colp + e * CS_QROW));
                    s1 = add2(s1, *reinterpret_cast<const f32x2*>(colp + (e + 1) * CS_QROW));
                }
                flush(add2(s0, s1), 15);
            } else {
#pragma unroll
                for (int e = 1; e < 16; ++e) {
                    const f32x2 v = *reinterpret_cast<const f32x2*>(colp + e * CS_QROW);
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
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- stage 3: φ = w3·SiLU(D/s + bc) per row; Δx·φ summed per destination row ------------------------------
        float phia, phib;
        tc16::phi_head_t(d, s2.inv_a, s2.inv_b, bcs, w3s, q, phia, phib);
        {   // lane e < 16 <-> edge e = fragment row (e & 7) + 8·(e >> 3), held by quad e & 7
            const float fa = __shfl_sync(FULL, phia, 4 * (lane & 7)), fb = __shfl_sync(FULL, phib, 4 * (lane & 7));
            const float phi = (lane & 8) ? fb : fa;
            // Δx·φ summed over runs of equal destination row inside the warp, one RED.ADD triple per run
            float sx = dx * phi, sy = dy * phi, sz = dz * phi;
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) {
                const int rk = __shfl_up_sync(FULL, row_c, o);
                const float ox = __shfl_up_sync(FULL, sx, o), oy = __shfl_up_sync(FULL, sy, o), oz = __shfl_up_sync(FULL, sz, o);
                if (lane >= o && rk == row_c) { sx += ox; sy += oy; sz += oz; }
            }
            const int rnext = __shfl_down_sync(FULL, row_c, 1);
            if (row_c >= 0 && (lane == 15 || rnext != row_c)) {
                if constexpr (DET) {
                    float* dst = row_c == cont_row ? slot + H : a.agg_x + (size_t)row_c * 4;
                    dst[0] = sx;
                    dst[1] = sy;
                    dst[2] = sz;
                } else {
                    float* dst = a.agg_x + (size_t)row_c * 4;
                    atomicAdd(dst + 0, sx);
                    atomicAdd(dst + 1, sy);
                    atomicAdd(dst + 2, sz);
                }
            }
        }

        // ---- roll the next tile's edge into place -------------------------------------------------------------
        // the wait covers this lane's copies; the warp barrier publishes every lane's Q rows of the next tile and
        // orders every lane's reads of this tile's buffer before the copies that refill it at the start of the next
        cp_async_wait_all();
        __syncwarp();
        row_c = n_row;
        float4 xi_n = make_float4(0.f, 0.f, 0.f, 0.f), xj_n = xi_n;
        if (n_row >= 0) {
            xi_n = *reinterpret_cast<const float4*>(xs);
            xj_n = *reinterpret_cast<const float4*>(xs + 4);
        }
        set_geometry(xi_n, xj_n);
#pragma unroll
        for (int k = 0; k < AR; ++k) ea_c[k] = n_ea[k];
        n_row = -1;
        if (has_edge(nntile)) {
            n_row = nidx[lane];
            n_col = nidx[16 + lane];
            if (AT == 1) n_ea[0] = __int_as_float(nidx[32 + 2 * lane]);
            if (AT == 2) {
                n_ea[0] = __int_as_float(nidx[32 + 2 * lane]);
                n_ea[AR - 1] = __int_as_float(nidx[33 + 2 * lane]);
            }
        }
    }
}

}  // namespace degnn

namespace degnn {

template <bool DET>
static int edge_layer_fwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags, const int32_t* row,
                          const int32_t* col, const float* edge_attr_sorted, const float* x4, const float* P,
                          const float* Q, const float* layer_params, float* agg_m, float* agg_x,
                          const int32_t* n_edges_dev, void* workspace, int64_t workspace_bytes, void* stream,
                          int max_ctas) {
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_edges == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_edges > 0, "negative size");
    // The kernel's tile numbers and edge ids are int32.  An edge id tile·64 + 16w + lane of a tile (tile < ⌈E/64⌉) is
    // below E + 63, and tile + 2·stride (stride = 4·grid, grid <= the SM count) below 2^25 + 8·SMs: both fit when
    // E + 63 <= INT32_MAX.  With n_edges_dev, E is the capacity and bounds the device count.
    DEGNN_CHECK_ARG(n_edges <= INT32_MAX - (CS_TILE - 1), "n_edges (the capacity with n_edges_dev) above 2^31 - 64");
    DEGNN_CHECK_ARG(row && col && x4 && P && Q && layer_params && agg_x, "null pointer");
    DEGNN_CHECK_ARG(A == 0 || edge_attr_sorted, "null edge_attr with edge_attr_nf > 0");
    DEGNN_CHECK_ARG((flags & DISTEGNN_FLAG_LAST) || agg_m, "null agg_m");
    float* slots = nullptr;
    if (DET) {
        if (int rc = det_check_workspace(n_nodes, n_edges, C, workspace, workspace_bytes, "distegnn_edge_layer_fwd_det"))
            return rc;
        slots = det_edge_slots(workspace, n_nodes, C);
    }
    Layout L = make_layout(A, C, Na);
    EdgeCsArgs a;
    a.N = n_nodes; a.E = (int)n_edges; a.E_dev = n_edges_dev; a.A = A; a.flags = flags & 0xffffu;
    a.row = row; a.col = col; a.ea = edge_attr_sorted; a.x4 = x4; a.P = P; a.Q = Q;
    a.w1r = layer_params + L.off[DISTEGNN_P_E_W1R];
    a.w1e = layer_params + L.off[DISTEGNN_P_E_W1E];
    a.w2 = layer_params + L.off[DISTEGNN_P_E_W2];
    a.b2 = layer_params + L.off[DISTEGNN_P_E_B2];
    a.wc = layer_params + L.off[DISTEGNN_P_E_WC];
    a.bc = layer_params + L.off[DISTEGNN_P_E_BC];
    a.w3 = layer_params + L.off[DISTEGNN_P_E_W3];
    a.agg_m = agg_m; a.agg_x = agg_x; a.slots = slots;
    const int64_t tiles = (n_edges + CS_TILE - 1) / CS_TILE;
    int64_t grid = (tiles + CS_WG - 1) / CS_WG;
    if (grid > sm_count()) grid = sm_count();
    if (DET) grid = det_grid(grid, max_ctas);
    auto launch = [&](auto kern) {
        ensure_dynamic_smem((const void*)kern, (int)CS_SMEM_BYTES);
        kern<<<(unsigned)grid, CS_THREADS, CS_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    };
    const bool last = flags & DISTEGNN_FLAG_LAST;
    switch (A) {
        case 0: last ? launch(edge_layer_cs_kernel<0, true, DET>) : launch(edge_layer_cs_kernel<0, false, DET>); break;
        case 1: last ? launch(edge_layer_cs_kernel<1, true, DET>) : launch(edge_layer_cs_kernel<1, false, DET>); break;
        case 2: last ? launch(edge_layer_cs_kernel<2, true, DET>) : launch(edge_layer_cs_kernel<2, false, DET>); break;
        default: last ? launch(edge_layer_cs_kernel<-1, true, DET>) : launch(edge_layer_cs_kernel<-1, false, DET>); break;
    }
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int edge_layer_fwd_det(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags, const int32_t* row,
                       const int32_t* col, const float* edge_attr_sorted, const float* x4, const float* P, const float* Q,
                       const float* layer_params, float* agg_m, float* agg_x, const int32_t* n_edges_dev,
                       void* workspace, int64_t workspace_bytes, void* stream, int max_ctas) {
    return edge_layer_fwd<true>(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q, layer_params,
                                agg_m, agg_x, n_edges_dev, workspace, workspace_bytes, stream, max_ctas);
}

}  // namespace degnn

extern "C" int distegnn_edge_layer_fwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                       const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                       const float* x4, const float* P, const float* Q,
                                       const float* layer_params, float* agg_m, float* agg_x,
                                       const int32_t* n_edges_dev, void* stream) {
    return degnn::edge_layer_fwd<false>(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q,
                                        layer_params, agg_m, agg_x, n_edges_dev, nullptr, 0, stream, 0);
}

extern "C" int distegnn_edge_layer_fwd_det(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                           const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                           const float* x4, const float* P, const float* Q,
                                           const float* layer_params, float* agg_m, float* agg_x,
                                           const int32_t* n_edges_dev, void* workspace, int64_t workspace_bytes,
                                           void* stream) {
    return degnn::edge_layer_fwd_det(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q,
                                     layer_params, agg_m, agg_x, n_edges_dev, workspace, workspace_bytes, stream, 0);
}
