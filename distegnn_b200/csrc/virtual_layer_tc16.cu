// Real<->virtual stage on the tensor cores — production kernel behind distegnn_virtual_layer_fwd.
// Replaces reference models/FastEGNN.py:252-253 (virtual geometry), 154-163 (edge_mode_virtual), 180, 191-193,
// 207, 220-223 (virtual halves of coord_model_vel / coord_model_virtual / node_model / node_model_virtual) and
// the global_mean_pool scatters at :193,:222.  Same math/outputs as testing/virtual_layer.cu (fp32-FMA twin).
//
// Rows of a tile are (node, channel) pairs: TN = 64 / C whole nodes per 64-row tile, row = n_local·C + c; rows past TN·C
// (and past the last node) are padding and contribute nothing.  One CTA per SM, VW_WG warpgroups, each an independent
// pipeline: a warpgroup grid-strides over its own tiles and, once set up, shares no barrier with the other warpgroups.
// Warp w of a warpgroup owns rows 16w .. 16w+15 of its tile, which are exactly the rows of the m64n64 accumulator fragment
// it holds (tile_mma.cuh); thread (g = lane/4, q = lane%4) owns rows g and g+8 of the warp, columns 8j + 2q + {0,1}.
// The A operands and the accumulators stay in registers; the weights, the G rows of the warpgroup's current graph and the
// fp32 mv rows (for the pools) are in shared memory.  Per tile (numerics as in the edge kernel: fp16 2-term split,
// per-row power-of-two range rescue, one reciprocal per four SiLUs with a stage-level guard, cold paths per warp; the
// rescue and the guard are tc16.cuh encode_rows, both φ heads phi_head_t):
//   stage 1  a1 = SiLU(Hn[node] + G[graph,c] + w_r·‖ΔX‖) -> fp16 hi/lo A fragments                 MMA 1: D = a1·W2vᵀ
//   stage 2  mv = SiLU(D + b2v) -> fp32 staging rows + hi/lo A fragments (kept for both heads)        MMA 2: D = mv·Wxvᵀ
//            while MMA 2 runs: agg_v[node] = mean_c mv, Σ_i mv per graph (lane <-> column pair)
//   stage 3a φ_xv = w3xv·SiLU(D + bxv) per row (quad shuffles)                                        MMA 3: D = mv·WXᵀ
//            while MMA 3 runs: trans_v[node] = mean_c(−ΔX·φ_xv)
//   stage 3b φ_X = w3x·SiLU(D + bx) per row; Σ_i ΔX·φ_X per graph.
// For C in {1, 2, 4, 8, 16} a node never straddles two warps and the pools are warp-local; for other C they read rows of
// the other warps of the group behind a warpgroup barrier.  Per-graph sums are kept per warp in shared memory and flushed
// to vsum (per warpgroup, one atomic per element) when the group's graph changes and at the end; tiles that straddle
// graphs add their rows to vsum directly.  The next tile's Hn rows, coordinates and graph ids are prefetched towards L1.
// Stages 2 and 3 run in the "t domain" (common.cuh silu4t): −log2(e) is folded into W2v and the biases, −ln 2 into the
// head projections and the mv pools.
#include "common.cuh"
#include "det.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct VirtT16Args {
    int64_t N;
    int B;
    unsigned flags;
    const int32_t* batch;
    const float* x4;
    const float* Hn;
    const float* Xv;
    const float* G;
    const float* w1r;
    const float* w2; const float* b2;
    const float* wxv; const float* bxv; const float* w3xv;
    const float* wx; const float* bx; const float* w3x;
    float* agg_v;
    float* trans_v;
    float* vsum;
    float* slots;   // deterministic mode: one K-float slot per chunk of 2^chunk_shift tiles (det.cuh)
    int chunk_shift;
};

// 4 warpgroups = 16 warps per SM
constexpr int VW_WG = 4;
constexpr int VW_THREADS = 128 * VW_WG, VW_WARPS = VW_THREADS / 32;
constexpr int VW_TILE = 64;                    // rows per warpgroup tile
// row pitch (floats) of the mv staging rows and the cached G rows: 72 = conflict-free LDS.64 / STS.64 in the accumulator
// fragment pattern (rows g, columns 2q: banks 8g + 2q) and in the pools' row pattern
constexpr int VW_ROW = 72;
constexpr int VW_W = 64 * 64;                  // fp16 elements per weight matrix (8 KB)
constexpr uint32_t VW_LBO = 1024;              // fp16 K-major no-swizzle, N = 64
// shared memory (floats) for C channels: weights | w1r, b2v, bxv, w3xv, bx, w3x | mv rows per warp | ΔX, φ_xv, φ_X per
// row and group | G rows of the current graph per group | Σ mv [C][64] per warp | Σ ΔX·φ_X [3][C] per warp (pitch 4C)
__host__ __device__ constexpr int vw_smem_floats(int C) {
    return 6 * VW_W / 2 + 6 * H + VW_WARPS * 16 * VW_ROW + VW_WG * VW_TILE * 6 + VW_WG * C * VW_ROW + VW_WARPS * C * H
           + VW_WARPS * 4 * C;
}
__host__ __device__ constexpr int vw_smem_bytes(int C) { return vw_smem_floats(C) * 4; }

// DET (deterministic mode, det.cuh): a warpgroup takes whole chunks of 2^chunk_shift consecutive tiles, in tile order, and
// the per-graph sums are walked node by node in row order by the thread that owns the element (accumulators in the
// group's accH / accX, which DET does not use per warp); a graph's partial of the chunk is stored to vsum when the graph
// starts in the chunk, else to the chunk's slot.
static_assert(VW_TILE == DET_VTILE, "det.cuh sizes the slots from the tile");
// C (the virtual channels) is a template parameter: every row <-> (node, channel) index, the pools' and sums' trip counts
// and the tile -> node mapping are compile-time constants, so no runtime division is left on the hot path.
template <int C, bool DET>
__global__ void __launch_bounds__(VW_THREADS, 1) virtual_layer_t16_kernel(const VirtT16Args a) {
    using namespace tmma;
    __half* W2hi = reinterpret_cast<__half*>(degnn_dyn_smem);
    __half* W2lo = W2hi + VW_W;
    __half* Wxvhi = W2lo + VW_W;
    __half* Wxvlo = Wxvhi + VW_W;
    __half* Wxhi = Wxvlo + VW_W;
    __half* Wxlo = Wxhi + VW_W;
    float* w1rs = reinterpret_cast<float*>(Wxlo + VW_W);
    float* b2s = w1rs + H;
    float* bxvs = b2s + H;
    float* w3xvs = bxvs + H;
    float* bxs = w3xvs + H;
    float* w3xs = bxs + H;
    float* stage_all = w3xs + H;                                   // [warps][16][VW_ROW]
    float* dX_all = stage_all + VW_WARPS * 16 * VW_ROW;            // [groups][64][4]
    float* phi_all = dX_all + VW_WG * VW_TILE * 4;                 // [groups][2][64]: φ_xv, φ_X
    float* gs_all = phi_all + VW_WG * VW_TILE * 2;                 // [groups][C][VW_ROW]
    float* accH_all = gs_all + VW_WG * C * VW_ROW;                 // [warps][C][64]
    float* accX_all = accH_all + VW_WARPS * C * H;                 // [warps][4C]: [3][C] used

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;
    const int wg = warp >> 2;              // warpgroup
    const int w = warp & 3;                // warp inside the warpgroup: rows 16w .. 16w+15 of its tile
    const int t = tid & 127;               // thread inside the warpgroup
    const int g = lane >> 2, q = lane & 3; // fragment rows g, g+8 of the warp; columns 8j + 2q
    constexpr int K = 4 + 3 * C + H * C;
    const bool need_feat = !(a.flags & DISTEGNN_FLAG_LAST);
    constexpr int TN = VW_TILE / C;
    constexpr bool warp_local = (16 % C) == 0;   // nodes never straddle warps: the pools need no warpgroup barrier

    // ---- one-time setup -------------------------------------------------------------------------
    tc16::stage_weight<VW_THREADS>(W2hi, W2lo, a.w2, 0, 64, tid, SILU_T_IN);   // t2 = SILU_T_IN·(a1·W2vᵀ + b2v); mv' = SILU_T_IN·mv
    tc16::stage_weight<VW_THREADS>(Wxvhi, Wxvlo, a.wxv, 0, 64, tid);
    tc16::stage_weight<VW_THREADS>(Wxhi, Wxlo, a.wx, 0, 64, tid);
    if (tid < H) {
        w1rs[tid] = a.w1r[tid];
        b2s[tid] = a.b2[tid] * SILU_T_IN;
        bxvs[tid] = a.bxv[tid] * SILU_T_IN;   // t3 = mv'·Wᵀ + SILU_T_IN·b  (SILU_T_IN·SILU_T_OUT = 1: the 64x64 head weights stay)
        w3xvs[tid] = a.w3xv[tid] * SILU_T_OUT;
        bxs[tid] = a.bx[tid] * SILU_T_IN;
        w3xs[tid] = a.w3x[tid] * SILU_T_OUT;
    }
    for (int i = tid; i < VW_WARPS * (C * H + 4 * C); i += VW_THREADS) accH_all[i] = 0.f;   // accH and accX
    fence_proxy_async_smem();
    __syncthreads();

    // descriptor of weight matrix k (W2v hi, lo, Wxv hi, lo, WX hi, lo): the matrices are 8 KB apart, and the start-address
    // field (bits 0..13, address >> 4) of the first one has room for all six
    const uint64_t bW0 = make_desc(smem_u32(W2hi), VW_LBO, 128);
    auto bW = [&](int k) { return bW0 + (uint64_t)(k * (VW_W * 2 / 16)); };
    float* tile_s = stage_all + wg * VW_TILE * VW_ROW;            // the group's 64 mv rows (warp w: rows 16w ..)
    float* dXs = dX_all + wg * VW_TILE * 4;
    float* phis = phi_all + wg * VW_TILE * 2;
    float* gs = gs_all + wg * C * VW_ROW;
    float* accH = accH_all + warp * C * H;
    float* accX = accX_all + warp * 4 * C;
    float* accH_g = accH_all + 4 * wg * C * H;                    // the four warps' sums of the group
    float* accX_g = accX_all + 4 * wg * 4 * C;
    const uint32_t bar_id = 1 + wg;
    int cur_graph = -1;                                           // graph of the G cache and the per-warp sums (group-uniform)

    // the group's per-warp sums of graph gr -> vsum, one atomic per element; all threads of the group, behind a group barrier
    auto flush = [&](int gr) {
        if (gr < 0) return;
        float* dst = a.vsum + (size_t)gr * K;
        if (need_feat)
            for (int i = t; i < C * H; i += 128) {
                float s = 0.f;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    s += accH_g[k * C * H + i];
                    accH_g[k * C * H + i] = 0.f;
                }
                atomicAdd(dst + 4 + 3 * C + i, s * SILU_T_OUT);
            }
        if (t < 3 * C) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s += accX_g[k * 4 * C + t];
                accX_g[k * 4 * C + t] = 0.f;
            }
            atomicAdd(dst + 4 + t, s);
        }
    };

    const int num_tiles = (int)((a.N + TN - 1) / TN);            // < 2^31 (the launch checks)
    const int stride = (int)gridDim.x * VW_WG;
    // DET: pipeline p takes the chunks p, p + stride, ...; inside a chunk the tiles follow each other
    const int CH = 1 << a.chunk_shift;                 // DET: tiles per chunk (a power of two: tile % CH = tile & (CH − 1))
    auto next_tile = [&](int tl) {
        if constexpr (DET) return ((tl + 1) & (CH - 1)) != 0 ? tl + 1 : tl + 1 + (stride - 1) * CH;
        else return tl + stride;
    };
    float* accG = accH_all + 4 * wg * C * H;          // DET: the group's sums [C][64] and [3][C], thread-owned elements
    float* accXG = accX_all + 4 * wg * 4 * C;
    int curM = -1, curX = -1, cont = -1;               // DET: graphs of those sums; the graph continued into the chunk
    auto det_dst = [&](int gr, int tl) {
        return gr == cont ? a.slots + (size_t)(tl >> a.chunk_shift) * K : a.vsum + (size_t)gr * K;
    };
    auto det_flush_m = [&](int tl) {                   // thread t: columns 2(t & 31), +1 of channels t/32, t/32 + 4, ...
        for (int c = t >> 5; c < C; c += 4) {
            f32x2* acc = reinterpret_cast<f32x2*>(accG + c * H + 2 * (t & 31));
            if (curM >= 0) {        // two scalar stores: rows of K = 4 + 67C floats are only 4-byte aligned for odd C
                float* dst = det_dst(curM, tl) + 4 + 3 * C + c * H + 2 * (t & 31);
                upk2(mul2(*acc, bc2(SILU_T_OUT)), dst[0], dst[1]);
            }
            *acc = 0ull;
        }
    };
    auto det_flush_x = [&](int tl) {                   // thread t < 3C: entry t of [3][C]
        if (t < 3 * C) {
            if (curX >= 0) det_dst(curX, tl)[4 + t] = accXG[t];
            accXG[t] = 0.f;
        }
    };
    const int ra = 16 * w + g, rb = ra + 8;            // the thread's tile rows
    const float* colp = tile_s + 2 * lane;             // pools: lane <-> columns 2·lane, 2·lane + 1

    for (int tile = DET ? ((int)blockIdx.x * VW_WG + wg) * CH : (int)blockIdx.x * VW_WG + wg; tile < num_tiles;
         tile = next_tile(tile)) {
        const int64_t n0 = (int64_t)tile * TN;
        if (DET && (tile & (CH - 1)) == 0)
            cont = (n0 > 0 && __ldg(a.batch + n0 - 1) == __ldg(a.batch + n0)) ? __ldg(a.batch + n0) : -1;
        const int nvalid = (int)min((int64_t)TN, a.N - n0);
        const int rows = nvalid * C;
        {   // pull the next tile's inputs (Hn rows, x4, graph ids) into L1 while this one computes
            const int64_t nn0 = (int64_t)next_tile(tile) * TN;
            const int nnv = (int)min((int64_t)TN, a.N - nn0);
            for (int i = t; i < 2 * nnv; i += 128) prefetch_l1(a.Hn + (size_t)nn0 * H + 32 * i);
            if (nnv > 0) {
                if (t < (nnv * 16 + 127) / 128) prefetch_l1(a.x4 + (size_t)nn0 * 4 + 32 * t);
                if (t == 127) prefetch_l1(a.batch + nn0);
                if (t == 126) prefetch_l1(a.batch + nn0 + nnv - 1);
            }
        }
        const int g_first = __ldg(a.batch + n0), g_last = __ldg(a.batch + n0 + nvalid - 1);
        const bool single = (g_first == g_last);
        if (single && g_first != cur_graph) {          // group-uniform; rare: once per graph and group
            named_bar(bar_id, 128);                    // every warp is done with the cache and its sums
            if constexpr (!DET) flush(cur_graph);
            cur_graph = g_first;
            for (int i = t; i < C * (H / 4); i += 128) {
                const int c = i / (H / 4), q4 = i - c * (H / 4);
                *reinterpret_cast<float4*>(gs + c * VW_ROW + 4 * q4) = ldg4(a.G + ((size_t)g_first * C + c) * H + 4 * q4);
            }
            named_bar(bar_id, 128);
        }

        // ---- stage 1: a1 = SiLU(Hn + G + w_r·‖ΔX‖) for rows ra, rb -> fp16 hi/lo A fragments -----------------------
        const bool va = ra < rows, vb = rb < rows;
        const float* pa;
        const float* pb;
        const float* ga;
        const float* gb;
        float vra, vrb;
        {   // a row's geometry comes from its node (x4, graph id) and its channel (Xv[graph, :, c]).  The thread's second row
            // reuses the first one's loads where the two share them: the node when C = 16 (rows g, g + 8 of one node), the
            // channel when C divides 8 (and so the Xv values, when the graph is the same).  Invalid rows read node 0 of
            // the tile: their values are never used.
            const int nla = va ? ra / C : 0, nlb = vb ? rb / C : 0;
            const int cha = va ? ra - nla * C : 0;
            const int chb = 8 % C == 0 ? cha : (vb ? rb - nlb * C : 0);
            const size_t nda = (size_t)(n0 + nla), ndb = C == 16 ? nda : (size_t)(n0 + nlb);
            const int gra = single ? g_first : __ldg(a.batch + nda);
            const int grb = (C == 16 || single) ? gra : __ldg(a.batch + ndb);
            const float4 xia = ldg4(a.x4 + nda * 4);
            const float4 xib = C == 16 ? xia : ldg4(a.x4 + ndb * 4);
            auto xv = [&](int gr, int ch) {
                const float* Xg = a.Xv + (size_t)gr * 3 * C + ch;
                return make_float3(__ldg(Xg), __ldg(Xg + C), __ldg(Xg + 2 * C));
            };
            const float3 xva = xv(gra, cha);
            const float3 xvb = (8 % C == 0 && grb == gra) ? xva : xv(grb, chb);
            auto row_geo = [&](int r, size_t node, int gr, int ch, float4 xi, float3 xg, const float*& hrow,
                               const float*& grow) {
                const float dx = xg.x - xi.x, dy = xg.y - xi.y, dz = xg.z - xi.z;
                if (q == 0) *reinterpret_cast<float4*>(dXs + 4 * r) = make_float4(dx, dy, dz, 0.f);
                hrow = a.Hn + node * H + 2 * q;
                // rows of the cached graph read shared memory, the others (tiles that straddle graphs) global memory
                grow = (gr == cur_graph ? (const float*)(gs + ch * VW_ROW) : a.G + ((size_t)gr * C + ch) * H) + 2 * q;
                return sqrtf(dx * dx + dy * dy + dz * dz);
            };
            vra = row_geo(ra, nda, gra, cha, xia, xva, pa, ga);
            vrb = row_geo(rb, ndb, grb, chb, xib, xvb, pb, gb);
        }
        auto pre = [&](int j, const float* hrow, const float* grow, float vr) {
            const f32x2 hh = __ldg(reinterpret_cast<const f32x2*>(hrow + 8 * j));
            const f32x2 gg = *reinterpret_cast<const f32x2*>(grow + 8 * j);
            return fma2(bc2(vr), *reinterpret_cast<const f32x2*>(w1rs + 8 * j + 2 * q), add2(hh, gg));
        };
        // register i = 2j + r of a fragment array <-> row g + 8r, columns 8j + 2q + {0,1} (= accumulator pair d[2i], d[2i+1])
        uint32_t ahi[16], alo[16];
        float qmax = 0.f;
        auto silu_guard = [&] { return silu_q_overflow(qmax); };
        tc16::RowScales s1;
        tc16::encode_rows<false, true>(
            [&](int j, f32x2& xa, f32x2& xb, auto pass) {
                xa = pre(j, pa, ga, vra);
                xb = pre(j, pb, gb, vrb);
                silu4p<decltype(pass)::value != tc16::FAST_PASS>(xa, xb, qmax);
                if (!va) xa = 0ull;
                if (!vb) xb = 0ull;
            },
            ahi, alo, s1, silu_guard);

        // ---- MMA 1 ----------------------------------------------------------------------------------------------
        float d[32];
        tc16::mma_f16x3_rA<VW_LBO>(d, ahi, alo, bW(0), bW(1));
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- stage 2: mv = SiLU(D/s + b2v) -> fp32 staging rows (pools) and fp16 hi/lo A fragments ----------------------
        // (ma, mb) = SILU_T_IN·mv -> the staging rows: the pools undo the factor, and MMA 3 re-splits its A operand from
        // them.  The rows are stored by the pass whose values are final: the fast pass, and again by the row-max pass when
        // the warp takes the cold path (batch guard included).
        qmax = 0.f;
        tc16::RowScales s2;
        tc16::encode_rows<false>(
            [&](int j, f32x2& ma, f32x2& mb, auto pass) {
                const f32x2 bb = *reinterpret_cast<const f32x2*>(b2s + 8 * j + 2 * q);
                ma = fma2(pk2(d[4 * j + 0], d[4 * j + 1]), bc2(s1.inv_a), bb);
                mb = fma2(pk2(d[4 * j + 2], d[4 * j + 3]), bc2(s1.inv_b), bb);
                silu4t<decltype(pass)::value != tc16::FAST_PASS>(ma, mb, qmax);
                if (decltype(pass)::value != tc16::ENCODE_PASS) {
                    *reinterpret_cast<f32x2*>(tile_s + ra * VW_ROW + 8 * j + 2 * q) = ma;
                    *reinterpret_cast<f32x2*>(tile_s + rb * VW_ROW + 8 * j + 2 * q) = mb;
                }
            },
            ahi, alo, s2, silu_guard);

        // the nodes whose per-node outputs (agg_v, trans_v) this warp writes: its own when nodes never straddle warps,
        // else every fourth node of the tile (the rows of the other warps are read behind a group barrier)
        const int nb = warp_local ? (16 * w) / C : w;
        const int ne = warp_local ? min(nb + 16 / C, nvalid) : nvalid;
        const int ns = warp_local ? 1 : 4;
        const int r_end = min(16 * w + 16, rows);     // the warp's valid rows are 16w .. r_end − 1

        // ---- MMA 2 (φ_xv head) overlapped with the pools of mv ------------------------------------------------------
        tc16::mma_f16x3_rA<VW_LBO>(d, ahi, alo, bW(2), bW(3));
        if (need_feat) {
            if (warp_local && !DET) __syncwarp();
            else named_bar(bar_id, 128);
            auto ld2 = [](const float* p) { return *reinterpret_cast<const f32x2*>(p); };
            const f32x2 invC2 = bc2(SILU_T_OUT / (float)C);     // the rows hold mv' = SILU_T_IN·mv
#pragma unroll 1
            for (int n = nb; n < ne; n += ns) {                  // mean over channels per node
                const float* base = colp + (n * C) * VW_ROW;
                f32x2 s0 = 0ull, s1 = 0ull;                      // even channels in s0, odd in s1
#pragma unroll
                for (int c = 0; c + 1 < C; c += 2) {
                    s0 = add2(s0, ld2(base + c * VW_ROW));
                    s1 = add2(s1, ld2(base + (c + 1) * VW_ROW));
                }
                if constexpr (C % 2 == 1) s0 = add2(s0, ld2(base + (C - 1) * VW_ROW));
                *reinterpret_cast<f32x2*>(a.agg_v + (size_t)(n0 + n) * H + 2 * lane) = mul2(add2(s0, s1), invC2);
            }
            if constexpr (DET) {                                 // every row of the tile, in row order
                for (int n = 0; n < nvalid; ++n) {
                    const int gr = single ? g_first : __ldg(a.batch + n0 + n);
                    if (gr != curM) {
                        det_flush_m(tile);
                        curM = gr;
                    }
#pragma unroll
                    for (int c = t >> 5; c < C; c += 4) {
                        f32x2* acc = reinterpret_cast<f32x2*>(accG + c * H + 2 * (t & 31));
                        *acc = add2(*acc, ld2(tile_s + (n * C + c) * VW_ROW + 2 * (t & 31)));
                    }
                }
            } else if (single) {                                 // sum of the warp's own rows per channel
#pragma unroll 1
                for (int i = 0; i < C; ++i) {                    // C <= 16: one first row per channel
                    const int r = 16 * w + i;
                    if (r >= r_end) break;
                    f32x2 s = ld2(colp + r * VW_ROW);
#pragma unroll
                    for (int k = 1; k < (16 - i + C - 1) / C; ++k)   // rows r + C, r + 2C, ... inside the warp's 16
                        if (r + k * C < r_end) s = add2(s, ld2(colp + (r + k * C) * VW_ROW));
                    f32x2* acc = reinterpret_cast<f32x2*>(accH + (r % C) * H + 2 * lane);
                    *acc = add2(*acc, s);
                }
            } else {                                             // straddling tile: the warp's rows straight to vsum
#pragma unroll 1
                for (int r = 16 * w; r < r_end; ++r) {
                    const int n = r / C, c = r - n * C;
                    float* dst = a.vsum + (size_t)__ldg(a.batch + n0 + n) * K + 4 + 3 * C + c * H + 2 * lane;
                    float v0, v1;
                    upk2(ld2(colp + r * VW_ROW), v0, v1);
                    atomicAdd(dst, v0 * SILU_T_OUT);
                    atomicAdd(dst + 1, v1 * SILU_T_OUT);
                }
            }
        }
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- stage 3: φ = w3·SiLU(D/s + b) per row (quad shuffles) ----------------------------------------------------
        {
            float phia, phib;
            tc16::phi_head_t(d, s2.inv_a, s2.inv_b, bxvs, w3xvs, q, phia, phib);
            if (q == 0) {
                phis[ra] = phia;
                phis[rb] = phib;
            }
        }

        // ---- MMA 3 (φ_X head) overlapped with trans_v[node] = mean_c(−ΔX_c·φ_xv,c) -----------------------------------------
        // A = mv again, re-split from the thread's own staging rows (bit for bit the fragments of MMA 2, scale 1 exact): the
        // fragments do not stay live across the φ_xv epilogue, which would not fit the register budget
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const f32x2 ma = *reinterpret_cast<const f32x2*>(tile_s + ra * VW_ROW + 8 * j + 2 * q);
            const f32x2 mb = *reinterpret_cast<const f32x2*>(tile_s + rb * VW_ROW + 8 * j + 2 * q);
            tc16::split_pair(mul2(ma, bc2(s2.a)), ahi[2 * j], alo[2 * j]);
            tc16::split_pair(mul2(mb, bc2(s2.b)), ahi[2 * j + 1], alo[2 * j + 1]);
        }
        tc16::mma_f16x3_rA<VW_LBO>(d, ahi, alo, bW(4), bW(5));
        if (warp_local) __syncwarp();
        else named_bar(bar_id, 128);
        for (int i = lane; i < (ne - nb + ns - 1) / ns * 3; i += 32) {
            const int n = nb + (i / 3) * ns, dd = i - 3 * (i / 3);
            float s = 0.f;
#pragma unroll 8   // not all 16 of C = 16: the loads in flight would spill under MMA 3
            for (int c = 0; c < C; ++c) s = fmaf(-dXs[4 * (n * C + c) + dd], phis[n * C + c], s);
            a.trans_v[(size_t)(n0 + n) * 4 + dd] = s / (float)C;
        }
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- stage 3b: φ_X; Σ_i ΔX_ic·φ_X,ic over the warp's own rows, per graph [3][C] -------------------------------
        {
            float phia, phib;
            tc16::phi_head_t(d, s2.inv_a, s2.inv_b, bxs, w3xs, q, phia, phib);
            if (q == 0) {
                phis[VW_TILE + ra] = phia;
                phis[VW_TILE + rb] = phib;
            }
        }
        __syncwarp();
        const float* phx = phis + VW_TILE;
        if constexpr (DET) {
            named_bar(bar_id, 128);                              // φ_X of every row
            if (t < 3 * C) {
                const int dd = t / C, c = t - dd * C;
                for (int n = 0; n < nvalid; ++n) {
                    const int gr = single ? g_first : __ldg(a.batch + n0 + n);
                    if (gr != curX) {
                        det_flush_x(tile);
                        curX = gr;
                    }
                    accXG[t] = fmaf(dXs[4 * (n * C + c) + dd], phx[n * C + c], accXG[t]);
                }
            }
        } else if (single) {
            for (int it = lane; it < 3 * C; it += 32) {       // lane <-> (component, first row of a channel); C <= 16
                const int dd = it / C, i = it - dd * C, r = 16 * w + i;
                if (r < r_end) {
                    float s = 0.f;
#pragma unroll
                    for (int k = 0; k < (16 + C - 1) / C; ++k)       // rows r, r + C, ... inside the warp's 16
                        if (r + k * C < r_end) s = fmaf(dXs[4 * (r + k * C) + dd], phx[r + k * C], s);
                    accX[dd * C + r % C] += s;
                }
            }
        } else {
            for (int it = lane; it < 48; it += 32) {          // lane <-> (row, component)
                const int r = 16 * w + it / 3, dd = it - 3 * (it / 3);
                if (r < r_end) {
                    const int n = r / C, c = r - n * C;
                    atomicAdd(a.vsum + (size_t)__ldg(a.batch + n0 + n) * K + 4 + dd * C + c, dXs[4 * r + dd] * phx[r]);
                }
            }
        }
        // the staging rows, ΔX and φ are rewritten by the next tile: after the reads of this one (group-wide when the pools
        // read other warps' rows)
        if (warp_local && !DET) __syncwarp();
        else named_bar(bar_id, 128);
        if (DET && (((tile + 1) & (CH - 1)) == 0 || tile + 1 >= num_tiles)) {     // end of the chunk
            if (need_feat) det_flush_m(tile);
            det_flush_x(tile);
            curM = curX = -1;
        }
    }
    if constexpr (!DET) {
        named_bar(bar_id, 128);      // every warp's sums are complete
        flush(cur_graph);
    }
}

}  // namespace degnn

namespace degnn {

// launches the instantiation for channel count c (check_dims has kept it in [1, DISTEGNN_MAX_CHANNELS])
template <bool DET, int C = 1>
static void launch_virtual(int c, unsigned grid, const VirtT16Args& a, cudaStream_t stream) {
    if constexpr (C <= DISTEGNN_MAX_CHANNELS) {
        if (c != C) return launch_virtual<DET, C + 1>(c, grid, a, stream);
        static_assert(vw_smem_bytes(C) <= 232448, "the shared memory of every C must fit");
        ensure_dynamic_smem((const void*)virtual_layer_t16_kernel<C, DET>, vw_smem_bytes(C));
        virtual_layer_t16_kernel<C, DET><<<grid, VW_THREADS, vw_smem_bytes(C), stream>>>(a);
    }
}

template <bool DET>
static int virtual_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags, const int32_t* batch32,
                             const float* x4, const float* Hn, const float* Xv, const float* G, const float* layer_params,
                             float* agg_v, float* trans_v, float* vsum, void* workspace, int64_t workspace_bytes,
                             void* stream, int max_ctas) {
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(batch32 && x4 && Hn && Xv && G && layer_params && trans_v && vsum, "null pointer");
    DEGNN_CHECK_ARG((flags & DISTEGNN_FLAG_LAST) || agg_v, "null agg_v");
    if (DET)
        if (int rc = det_check_workspace(n_nodes, -1, C, workspace, workspace_bytes, "distegnn_virtual_layer_fwd_det"))
            return rc;
    Layout L = make_layout(A, C, Na);
    VirtT16Args a;
    a.N = n_nodes; a.B = n_graphs; a.flags = flags;
    a.batch = batch32; a.x4 = x4; a.Hn = Hn; a.Xv = Xv; a.G = G;
    a.w1r = layer_params + L.off[DISTEGNN_P_V_W1R];
    a.w2 = layer_params + L.off[DISTEGNN_P_V_W2];
    a.b2 = layer_params + L.off[DISTEGNN_P_V_B2];
    a.wxv = layer_params + L.off[DISTEGNN_P_V_WXV];
    a.bxv = layer_params + L.off[DISTEGNN_P_V_BXV];
    a.w3xv = layer_params + L.off[DISTEGNN_P_V_W3XV];
    a.wx = layer_params + L.off[DISTEGNN_P_V_WX];
    a.bx = layer_params + L.off[DISTEGNN_P_V_BX];
    a.w3x = layer_params + L.off[DISTEGNN_P_V_W3X];
    a.agg_v = agg_v; a.trans_v = trans_v; a.vsum = vsum;
    a.slots = DET ? det_vsum_slots(workspace) : nullptr;
    a.chunk_shift = DET ? det_chunk_shift(n_nodes, C) : 0;
    const int TN = VW_TILE / C;
    const int64_t tiles = (n_nodes + TN - 1) / TN;
    const int64_t units = DET ? det_chunks(n_nodes, C) : tiles;       // what the pipelines grid-stride over
    DEGNN_CHECK_ARG(tiles + ((int64_t)sm_count() * VW_WG << (DET ? det_chunk_shift(n_nodes, C) : 0)) < ((int64_t)1 << 31),
                    "too many nodes");
    int64_t grid = (units + VW_WG - 1) / VW_WG;
    if (grid > sm_count()) grid = sm_count();
    if (DET) grid = det_grid(grid, max_ctas);
    launch_virtual<DET>(C, (unsigned)grid, a, (cudaStream_t)stream);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

int virtual_layer_fwd_det(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags, const int32_t* batch32,
                          const float* x4, const float* Hn, const float* Xv, const float* G, const float* layer_params,
                          float* agg_v, float* trans_v, float* vsum, void* workspace, int64_t workspace_bytes,
                          void* stream, int max_ctas) {
    return virtual_layer_fwd<true>(n_nodes, n_graphs, A, C, Na, flags, batch32, x4, Hn, Xv, G, layer_params, agg_v,
                                   trans_v, vsum, workspace, workspace_bytes, stream, max_ctas);
}

}  // namespace degnn

extern "C" int distegnn_virtual_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                          const int32_t* batch32, const float* x4, const float* Hn,
                                          const float* Xv, const float* G, const float* layer_params,
                                          float* agg_v, float* trans_v, float* vsum, void* stream) {
    return degnn::virtual_layer_fwd<false>(n_nodes, n_graphs, A, C, Na, flags, batch32, x4, Hn, Xv, G, layer_params,
                                           agg_v, trans_v, vsum, nullptr, 0, stream, 0);
}

extern "C" int distegnn_virtual_layer_fwd_det(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                              const int32_t* batch32, const float* x4, const float* Hn,
                                              const float* Xv, const float* G, const float* layer_params,
                                              float* agg_v, float* trans_v, float* vsum, void* workspace,
                                              int64_t workspace_bytes, void* stream) {
    return degnn::virtual_layer_fwd_det(n_nodes, n_graphs, A, C, Na, flags, batch32, x4, Hn, Xv, G, layer_params,
                                        agg_v, trans_v, vsum, workspace, workspace_bytes, stream, 0);
}
