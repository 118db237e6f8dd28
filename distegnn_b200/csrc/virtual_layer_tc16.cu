// Real<->virtual stage on the tensor cores — production kernel behind distegnn_virtual_layer_fwd (thread per row).
// Replaces reference models/FastEGNN.py:252-253 (virtual geometry), 154-163 (edge_mode_virtual), 180, 191-193,
// 207, 220-223 (virtual halves of coord_model_vel / coord_model_virtual / node_model / node_model_virtual) and
// the global_mean_pool scatters at :193,:222.  Same math/outputs as testing/virtual_layer.cu (fp32-FMA twin).
//
// Rows of a tile are (node, channel) pairs: TN = 128 / C nodes per tile, row = n_local*C + c, one tile-memory row per
// tile row.  One CTA per SM, 128 threads = 1 tile group = 1 warpgroup; thread r owns row r.
// All three 64x64 layers run as wgmma tile GEMMs with the fp16 2-term split (tc16.cuh); tile memory per group
// (tile_mma.cuh): A_hi 32 + A_lo 32 + D 64 columns (the two coordinate heads reuse D one after the other).
//   stage 1  a1 = SiLU(Hn[node] + G[graph,c] + w_r·‖ΔX‖)  -> A              MMA 1: D = a1·W2vᵀ
//            (the C x 64 G rows of the group's current graph are cached in shared memory: every (node, channel) row re-reads
//             its G row, and shared memory leaves little L1)
//   stage 2  mv = SiLU(D + b2v) -> shared tile + A                            MMA 2: D = mv·Wxvᵀ
//            (then: agg_v[node] = mean_c mv, per-graph Σ_i mv accumulated in shared memory)
//   stage 3a φ_xv = w3xv·SiLU(D + bxv)                                        MMA 3: D = mv·WXᵀ
//   stage 3b φ_X  = w3x·SiLU(D + bx);  trans_v[node] = mean_c(−ΔX·φ_xv);  per-graph Σ_i ΔX·φ_X accumulated.
#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct VirtT16Args {
    int64_t N;
    int B, C;
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
    int g_smem;     // the launch reserved V16_GROUPS * C * 68 floats behind V16_SMEM_BYTES for the G rows of the current graph
};

constexpr int V16_THREADS = 128, V16_GROUPS = 1, V16_GROUP = 128;
constexpr int V16_TM_COLS = 128;                  // per tile group: A_hi 32 | A_lo 32 | D 64
constexpr int V16_ROW = 68;
constexpr int V16_MAXC = DISTEGNN_MAX_CHANNELS;
constexpr int V16_W = 4096;
constexpr int V16_SMEM_BYTES = tmma::tm_bytes(V16_GROUPS * V16_TM_COLS)
                               + 6 * V16_W * 2                         // W2v, Wxv, WX (hi+lo)
                               + V16_GROUPS * TILE_M * V16_ROW * 4     // mv tile per group
                               + V16_GROUPS * V16_MAXC * H * 4         // Σ mv accumulators per group
                               + V16_GROUPS * 4 * V16_MAXC * 4         // Σ ΔX·φ_X accumulators per group
                               + 6 * H * 4                             // w1r, b2v, bxv, w3xv, bx, w3x
                               + V16_GROUPS * TILE_M * 4 * 4           // ΔX per row
                               + V16_GROUPS * 2 * TILE_M * 4           // φ_xv, φ_X per row
                               + V16_GROUPS * TILE_M * 4               // graph id per local node
                               // + (launch time, if it fits) V16_GROUPS * C * V16_ROW * 4: G rows of the current graph
                               + 128;
constexpr uint32_t V16_LBO = 1024;

__global__ void __launch_bounds__(V16_THREADS, 1) virtual_layer_t16_kernel(const VirtT16Args a) {
    using namespace tmma;
    uint8_t* const smem_raw = degnn_dyn_smem + tm_bytes(V16_GROUPS * V16_TM_COLS);
    __half* W2hi = reinterpret_cast<__half*>(smem_raw);
    __half* W2lo = W2hi + V16_W;
    __half* Wxvhi = W2lo + V16_W;
    __half* Wxvlo = Wxvhi + V16_W;
    __half* Wxhi = Wxvlo + V16_W;
    __half* Wxlo = Wxhi + V16_W;
    float* tiles = reinterpret_cast<float*>(Wxlo + V16_W);
    float* accH_all = tiles + V16_GROUPS * TILE_M * V16_ROW;
    float* accX_all = accH_all + V16_GROUPS * V16_MAXC * H;
    float* w1rs = accX_all + V16_GROUPS * 4 * V16_MAXC;
    float* b2s = w1rs + H;
    float* bxvs = b2s + H;
    float* w3xvs = bxvs + H;
    float* bxs = w3xvs + H;
    float* w3xs = bxs + H;
    float* dX_all = w3xs + H;
    float* phi_all = dX_all + V16_GROUPS * TILE_M * 4;
    int* sgraph_all = reinterpret_cast<int*>(phi_all + V16_GROUPS * 2 * TILE_M);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sgraph_all + V16_GROUPS * TILE_M);
    float* gs_all = reinterpret_cast<float*>(degnn_dyn_smem + V16_SMEM_BYTES);      // present iff a.g_smem

    const int tid = threadIdx.x;
    const int grp = tid / V16_GROUP, t = tid % V16_GROUP, wq = (tid >> 5) & 3;
    const int C = a.C;
    const int K = 4 + 3 * C + H * C;
    const bool need_feat = !(a.flags & DISTEGNN_FLAG_LAST);
    const int TN = TILE_M / C;
    const bool pow2C = (C & (C - 1)) == 0 && C <= 32;
    const int lane = tid & 31;

    // ---- one-time setup ---------------------------------------------------------------------------
    tc16::stage_weight<V16_THREADS>(W2hi, W2lo, a.w2, 0, 64, tid, SILU_T_IN);   // t2 = SILU_T_IN·(a1·W2vᵀ + b2v); mv' = SILU_T_IN·mv
    tc16::stage_weight<V16_THREADS>(Wxvhi, Wxvlo, a.wxv, 0, 64, tid);
    tc16::stage_weight<V16_THREADS>(Wxhi, Wxlo, a.wx, 0, 64, tid);
    if (tid < H) {
        w1rs[tid] = a.w1r[tid];
        b2s[tid] = a.b2[tid] * SILU_T_IN;
        bxvs[tid] = a.bxv[tid] * SILU_T_IN;   // t3 = mv'·Wᵀ + SILU_T_IN·b  (SILU_T_IN·SILU_T_OUT = 1: the 64x64 head weights stay)
        w3xvs[tid] = a.w3xv[tid] * SILU_T_OUT;
        bxs[tid] = a.bx[tid] * SILU_T_IN;
        w3xs[tid] = a.w3x[tid] * SILU_T_OUT;
    }
    for (int i = tid; i < V16_GROUPS * (V16_MAXC * H + 4 * V16_MAXC); i += V16_THREADS) accH_all[i] = 0.f;
    if (tid == 0) {
        for (int i = 0; i < V16_GROUPS; ++i) mbar_init(&bars[i], 1);
        fence_mbar_init();
    }
    fence_proxy_async_smem();
    __syncthreads();

    const uint32_t lane_off = ((uint32_t)(32 * wq)) << 16;
    const uint32_t col0 = (uint32_t)(grp * V16_TM_COLS);
    const uint32_t tA_hi = col0, tA_lo = col0 + 32, tD = col0 + 64;
    auto desc = [&](const __half* p) { return make_b_desc(smem_u32(p), V16_LBO, 128); };
    const uint64_t dW2hi = desc(W2hi), dW2lo = desc(W2lo), dWxvhi = desc(Wxvhi), dWxvlo = desc(Wxvlo),
                   dWxhi = desc(Wxhi), dWxlo = desc(Wxlo);
    float* tile_s = tiles + grp * TILE_M * V16_ROW;
    float* myrow = tile_s + t * V16_ROW;
    float* accH = accH_all + grp * V16_MAXC * H;
    float* accX = accX_all + grp * 4 * V16_MAXC;
    float* dXs = dX_all + grp * TILE_M * 4;
    float* phis = phi_all + grp * 2 * TILE_M;
    int* sgraph = sgraph_all + grp * TILE_M;
    float* gs = gs_all + grp * a.C * V16_ROW;          // [C][68]: pitch 68 keeps the channel rows of a node on distinct banks
    const bool g_smem = a.g_smem;
    uint64_t* hbar = bars + grp;                  // Hn block landed (fetch_hn)
    const uint32_t bar_id = 1 + grp;
    int cur_graph = -1;

    auto flush = [&](int g) {                      // all threads of the group
        if (g >= 0) {
            float* dst = a.vsum + (size_t)g * K;
            if (need_feat)
                for (int i = t; i < C * H; i += V16_GROUP) {
                    atomicAdd(dst + 4 + 3 * C + i, accH[i] * SILU_T_OUT);
                    accH[i] = 0.f;
                }
            if (t < 3 * C) {
                atomicAdd(dst + 4 + t, accX[t]);
                accX[t] = 0.f;
            }
        }
    };
    auto a_ready = [&]() {
        tm_st_fence();
        named_bar(bar_id, V16_GROUP);
    };
    // D = A·Wᵀ over the whole tile by the group's warpgroup; mma_done() publishes D to every row thread
    auto issue = [&](uint64_t bhi, uint64_t blo) { tc16::mma_f16x3<V16_LBO>(tD, tA_hi, tA_lo, bhi, blo, 1, false, 0, 2); };
    auto mma_done = [&]() { named_bar(bar_id, V16_GROUP); };

    const int64_t num_tiles = (a.N + TN - 1) / TN;
    const int64_t tstride = (int64_t)gridDim.x * V16_GROUPS;
    // Hn rows n0 .. n0+nvalid-1 of tile `tl` -> the start of the group's mv tile at the padded pitch V16_ROW (the channel rows
    // of 4 different nodes that a warp reads together then sit on different banks): one 256-byte bulk copy per node, issued by
    // the first `nvalid` threads of the group; thread 0 posts the byte count.
    // Not called: stage 1 reads Hn with LDG behind an L1 prefetch.  Deleting even this unused lambda changes the kernel's
    // SASS, so it goes together with the Hn mbarrier init above in a change that is benchmarked on its own.
    [[maybe_unused]] auto fetch_hn = [&](int64_t tl) {
        if (tl < num_tiles) {
            const int64_t m0 = tl * TN;
            const int nv = (int)min((int64_t)TN, a.N - m0);
            if (t == 0) mbar_expect_tx(hbar, (uint32_t)nv * (H * 4));     // may land after the first bytes: the count just dips below 0
            if (t < nv) bulk_g2s(tile_s + t * V16_ROW, a.Hn + (size_t)(m0 + t) * H, H * 4, hbar);
        }
    };
    for (int64_t tile = (int64_t)blockIdx.x * V16_GROUPS + grp; tile < num_tiles; tile += tstride) {
        const int64_t n0 = tile * TN;
        const int nvalid = (int)min((int64_t)TN, a.N - n0);
        const int rows = nvalid * C;
        {   // pull the next tile's small inputs (x4, graph ids) into L1 while this one computes
            const int64_t nn0 = (tile + tstride) * TN;
            const int nnv = (int)min((int64_t)TN, a.N - nn0);
            for (int i = t; i < 2 * nnv; i += V16_GROUP) prefetch_l1(a.Hn + (size_t)nn0 * H + 32 * i);
            if (nnv > 0) {
                if (t < (nnv * 16 + 127) / 128) prefetch_l1(a.x4 + (size_t)nn0 * 4 + 32 * t);
                if (t == 127) prefetch_l1(a.batch + nn0);
                if (t == 126) prefetch_l1(a.batch + nn0 + nnv - 1);
            }
        }
        if (t < TN) sgraph[t] = (t < nvalid) ? __ldg(a.batch + n0 + t) : -1;
        named_bar(bar_id, V16_GROUP);
        const int g_first = sgraph[0], g_last = sgraph[nvalid - 1];
        const bool single = (g_first == g_last);
        if (single && g_first != cur_graph) {
            flush(cur_graph);
            cur_graph = g_first;
            if (g_smem)
                for (int i = t; i < C * (H / 4); i += V16_GROUP) {       // G[g_first] -> shared (rare: once per graph and group)
                    const int c = i / (H / 4), q = i - c * (H / 4);
                    *reinterpret_cast<float4*>(gs + c * V16_ROW + 4 * q) = ldg4(a.G + ((size_t)g_first * C + c) * H + 4 * q);
                }
            named_bar(bar_id, V16_GROUP);
        }

        // ---- stage 1 ------------------------------------------------------------------------------
        const bool rvalid = t < rows;
        const int nl = rvalid ? t / C : 0;
        const int ch = rvalid ? t - nl * C : 0;
        const int g = rvalid ? sgraph[nl] : g_first;
        const size_t node = (size_t)(n0 + nl);
        float vr;
        {
            const float4 xi = ldg4(a.x4 + node * 4);
            const float* Xg = a.Xv + (size_t)g * 3 * C;
            const float dx = __ldg(Xg + ch) - xi.x, dy = __ldg(Xg + C + ch) - xi.y, dz = __ldg(Xg + 2 * C + ch) - xi.z;
            vr = sqrtf(dx * dx + dy * dy + dz * dz);
            *reinterpret_cast<float4*>(dXs + 4 * t) = make_float4(dx, dy, dz, 0.f);
        }
        const float* hrow = a.Hn + node * H;
        // rows of the cached graph read shared memory, the others (tiles that straddle graphs) global memory: generic loads
        const float* grow = (g_smem && g == cur_graph) ? (const float*)(gs + ch * V16_ROW) : a.G + ((size_t)g * C + ch) * H;
        const f32x2 vr2 = bc2(vr);
        const float inv1 = tc16::encode_row2(
            [&](int c, f32x2 (&v)[8], bool, auto safe, float& qmax) {
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    const int cc = 16 * c + 4 * j4;
                    const ulonglong2 hh = __ldg(reinterpret_cast<const ulonglong2*>(hrow + cc));
                    const ulonglong2 gg = *reinterpret_cast<const ulonglong2*>(grow + cc);
                    const ulonglong2 wr = *reinterpret_cast<const ulonglong2*>(w1rs + cc);
                    f32x2 p0 = fma2(vr2, wr.x, add2(hh.x, gg.x)), p1 = fma2(vr2, wr.y, add2(hh.y, gg.y));
                    silu4p<decltype(safe)::value>(p0, p1, qmax);
                    if (!rvalid) p0 = p1 = 0ull;
                    v[2 * j4] = p0;
                    v[2 * j4 + 1] = p1;
                }
            },
            lane_off + tA_hi, lane_off + tA_lo);
        a_ready();
        issue(dW2hi, dW2lo);
        mma_done();

        // ---- stage 2: mv = SiLU(D + b2v) -> shared tile and A ---------------------------------------------
        const float inv2 = tc16::encode_row2_tm(
            [&](int c, const uint32_t (&d)[16], f32x2 (&v)[8], bool first, auto safe, float& qmax) {
                const f32x2 is2 = bc2(inv1);
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    const int cc = 16 * c + 4 * j4;
                    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(b2s + cc);
                    f32x2 m0 = fma2(pk2u(d[4 * j4 + 0], d[4 * j4 + 1]), is2, bb.x);
                    f32x2 m1 = fma2(pk2u(d[4 * j4 + 2], d[4 * j4 + 3]), is2, bb.y);
                    silu4t<decltype(safe)::value>(m0, m1, qmax);
                    if (first && need_feat) *reinterpret_cast<ulonglong2*>(myrow + cc) = make_ulonglong2(m0, m1);
                    v[2 * j4] = m0;
                    v[2 * j4 + 1] = m1;
                }
            },
            lane_off + tD, lane_off + tA_hi, lane_off + tA_lo);
        a_ready();
        issue(dWxvhi, dWxvlo);
        // pools of mv (the tile in shared memory; MMA 2 wrote only D)
        if (need_feat) {
            // thread <-> (column pair, quarter): one LDS.64 + one pair add per two elements, two chains per sum
            const int c2 = 2 * (t & 31), q4 = t >> 5;
            auto ld2 = [](const float* p) { return *reinterpret_cast<const f32x2*>(p); };
            const f32x2 invC2 = bc2(SILU_T_OUT / (float)C);     // the tile holds mv' = SILU_T_IN·mv
            for (int n = q4; n < nvalid; n += 4) {          // mean over channels per node
                const float* base = tile_s + (n * C) * V16_ROW + c2;
                f32x2 s0 = 0ull, s1 = 0ull;
                int c = 0;
                for (; c + 1 < C; c += 2) {
                    s0 = add2(s0, ld2(base + c * V16_ROW));
                    s1 = add2(s1, ld2(base + (c + 1) * V16_ROW));
                }
                if (c < C) s0 = add2(s0, ld2(base + c * V16_ROW));
                *reinterpret_cast<f32x2*>(a.agg_v + (size_t)(n0 + n) * H + c2) = mul2(add2(s0, s1), invC2);
            }
            if (single) {                                    // sum over nodes per channel
                for (int c = q4; c < C; c += 4) {
                    const float* base = tile_s + c * V16_ROW + c2;
                    const int nstep = C * V16_ROW;
                    f32x2 s0 = 0ull, s1 = 0ull;
                    int n = 0;
                    for (; n + 1 < nvalid; n += 2) {
                        s0 = add2(s0, ld2(base + n * nstep));
                        s1 = add2(s1, ld2(base + (n + 1) * nstep));
                    }
                    if (n < nvalid) s0 = add2(s0, ld2(base + n * nstep));
                    f32x2* acc = reinterpret_cast<f32x2*>(accH + c * H + c2);
                    *acc = add2(*acc, add2(s0, s1));
                }
            } else {
                for (int n = q4; n < nvalid; n += 4) {
                    float* dst = a.vsum + (size_t)sgraph[n] * K + 4 + 3 * C + c2;
                    for (int c = 0; c < C; ++c) {
                        float v0, v1;
                        upk2(ld2(tile_s + (n * C + c) * V16_ROW + c2), v0, v1);
                        atomicAdd(dst + c * H, v0 * SILU_T_OUT);
                        atomicAdd(dst + c * H + 1, v1 * SILU_T_OUT);
                    }
                }
            }
        }
        mma_done();

        // ---- stage 3a: φ_xv = w3xv·SiLU(D + bxv) --------------------------------------------------------
        auto head_pass = [&](const float* bs, const float* ws, auto safe, float& qmax) {
            f32x2 ph01 = bc2(0.f), ph23 = bc2(0.f);
            const f32x2 is2 = bc2(inv2);
            auto head_math = [&](int c, const uint32_t (&d)[16]) {
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    const int cc = 16 * c + 4 * j4;
                    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(bs + cc);
                    const ulonglong2 ww = *reinterpret_cast<const ulonglong2*>(ws + cc);
                    f32x2 s0 = fma2(pk2u(d[4 * j4 + 0], d[4 * j4 + 1]), is2, bb.x);
                    f32x2 s1 = fma2(pk2u(d[4 * j4 + 2], d[4 * j4 + 3]), is2, bb.y);
                    silu4t<decltype(safe)::value>(s0, s1, qmax);
                    ph01 = fma2(s0, ww.x, ph01);
                    ph23 = fma2(s1, ww.y, ph23);
                }
            };
#pragma unroll 1
            for (int c = 0; c < 4; ++c) {
                uint32_t d[16];
                tm_ld16(lane_off + tD + 16 * c, d);
                head_math(c, d);
            }
            float p0, p1, p2, p3;
            upk2(ph01, p0, p1);
            upk2(ph23, p2, p3);
            return (p0 + p1) + (p2 + p3);
        };
        auto head = [&](const float* bs, const float* ws) {
            float qmax = 0.f;
            float phi = head_pass(bs, ws, tc16::kFast, qmax);
            if (__any_sync(FULL, silu_q_overflow(qmax))) phi = head_pass(bs, ws, tc16::kSafe, qmax);   // cold
            return phi;
        };
        phis[t] = head(bxvs, w3xvs);
        named_bar(bar_id, V16_GROUP);                  // D fully read (A still holds mv); nobody reads the mv tile any more
        issue(dWxhi, dWxlo);
        // trans_v[node] = mean_c(−ΔX_c·φ_xv,c)
        for (int i = t; i < nvalid * 3; i += V16_GROUP) {
            const int n = i / 3, d = i - 3 * n;
            float s = 0.f;
            for (int c = 0; c < C; ++c) s = fmaf(-dXs[4 * (n * C + c) + d], phis[n * C + c], s);
            a.trans_v[(size_t)(n0 + n) * 4 + d] = s / (float)C;
        }
        mma_done();

        // ---- stage 3b: φ_X = w3x·SiLU(D + bx); Σ_i ΔX_ic·φ_X,ic per graph [3][C] -----------------------------
        const float phiX = head(bxs, w3xs);
        if (single && pow2C) {
            // rows of one channel sit C lanes apart: butterfly over the lane bits above log2(C), then one shared-memory atomic per
            // (component, channel) and warp — no group barrier, no serial loop on the critical path of the tile
            const float4 d4 = *reinterpret_cast<const float4*>(dXs + 4 * t);      // own ΔX, written by this thread in stage 1
            float sx = rvalid ? d4.x * phiX : 0.f, sy = rvalid ? d4.y * phiX : 0.f, sz = rvalid ? d4.z * phiX : 0.f;
            for (int o = C; o < 32; o <<= 1) {
                sx += __shfl_xor_sync(FULL, sx, o);
                sy += __shfl_xor_sync(FULL, sy, o);
                sz += __shfl_xor_sync(FULL, sz, o);
            }
            if (lane < C) {
                atomicAdd(accX + lane, sx);
                atomicAdd(accX + C + lane, sy);
                atomicAdd(accX + 2 * C + lane, sz);
            }
        } else {
            phis[TILE_M + t] = phiX;
            named_bar(bar_id, V16_GROUP);
            if (t < 3 * C) {
                const int d = t / C, c = t - d * C;
                const float* phx = phis + TILE_M;
                if (single) {
                    float s = 0.f;
                    for (int n = 0; n < nvalid; ++n) s = fmaf(dXs[4 * (n * C + c) + d], phx[n * C + c], s);
                    accX[t] += s;
                } else {
                    for (int n = 0; n < nvalid; ++n)
                        atomicAdd(a.vsum + (size_t)sgraph[n] * K + 4 + t, dXs[4 * (n * C + c) + d] * phx[n * C + c]);
                }
            }
        }
        // dXs / phis / the mv tile are rewritten by the next tile only after ITS first group barrier, which the threads of the
        // loop above reach after their reads; sgraph is rewritten before that barrier, and read above only on the straddling path
        if (!single) named_bar(bar_id, V16_GROUP);
    }
    named_bar(bar_id, V16_GROUP);      // the last tile's shared-memory atomics into accX, before other threads flush them
    flush(cur_graph);
}

}  // namespace degnn

extern "C" int distegnn_virtual_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                          const int32_t* batch32, const float* x4, const float* Hn,
                                          const float* Xv, const float* G, const float* layer_params,
                                          float* agg_v, float* trans_v, float* vsum, void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(batch32 && x4 && Hn && Xv && G && layer_params && trans_v && vsum, "null pointer");
    DEGNN_CHECK_ARG((flags & DISTEGNN_FLAG_LAST) || agg_v, "null agg_v");
    Layout L = make_layout(A, C, Na);
    VirtT16Args a;
    a.N = n_nodes; a.B = n_graphs; a.C = C; a.flags = flags;
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
    // the G cache is taken when it fits next to the fixed layout
    const int g_bytes = V16_GROUPS * C * V16_ROW * 4;
    a.g_smem = (V16_SMEM_BYTES + g_bytes <= 232448 - 1024) ? 1 : 0;
    const int smem_bytes = V16_SMEM_BYTES + (a.g_smem ? g_bytes : 0);
    static_assert(V16_SMEM_BYTES + V16_GROUPS * V16_MAXC * V16_ROW * 4 <= 232448, "G cache of the widest C must fit");
    ensure_dynamic_smem((const void*)virtual_layer_t16_kernel, (int)V16_SMEM_BYTES + V16_GROUPS * V16_MAXC * V16_ROW * 4);
    const int TN = TILE_M / C;
    const int64_t tiles = (n_nodes + TN - 1) / TN;
    int64_t grid = (tiles + V16_GROUPS - 1) / V16_GROUPS;
    if (grid > sm_count()) grid = sm_count();
    virtual_layer_t16_kernel<<<(unsigned)grid, V16_THREADS, smem_bytes, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
