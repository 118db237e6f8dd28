// Backward of the real<->virtual stage on the tensor cores (wgmma) — production kernel behind
// distegnn_virtual_layer_bwd.  Its twin, the fp32-FMA kernel of csrc/testing/virtual_layer_bwd.cu behind
// distegnn_virtual_layer_bwd_simt, has the same contract and math (reference: autograd through models/FastEGNN.py:154-163,
// 180, 191-193, 207, 220-223, 252-253).  Per 128-row tile (rows = (node, channel)) the SIX row-wise tile GEMMs —
// recompute z2 = a1·W2vᵀ, zxv = mv·Wxvᵀ, zx = mv·Wxᵀ; data gradients g_mv = g_zxv·Wxv + g_zx·Wx (two MMAs into ONE accumulator, both rows encoded
// with a common scale), g_a1 = g_z2·W2v — run as wgmma f16 with the fp16 2-term split (tc16.cuh), A written to tile memory
// by the thread that owns the row; the three weight-gradient GEMMs stay on the CUDA cores (see edge_layer_bwd_tc.cu).
//
// Shared memory: six 64x64 B operands (hi + lo = 16 KB each) do not fit next to the two fp32 row tiles and the tile memory,
// so the weights are NOT resident: distegnn_virtual_bwd_prepare writes them once per call as fp16 hi/lo IMAGES already in
// the shared-memory operand layout, and the CTA streams them through two 16 KB slots with one TMA bulk copy per
// matrix, two matrices ahead of their use (mbarrier per slot; the order W2v, Wxv, Wx, Wxvᵀ, Wxᵀ, W2vᵀ repeats every tile).
// One CTA per SM, 128 threads = 1 warpgroup; thread r owns row r and holds whole 64-wide rows in registers.
// Tile memory (tile_mma.cuh, 192 columns): D 64 | A2_hi 32 | A2_lo 32 | z2 64, where the first 64 columns also
// hold the A operand (A_hi 32 | A_lo 32) that a GEMM writing D consumes: every D row is read into registers before its
// thread writes the next A there.  A2 holds mv for the two GEMMs that read it, then g_zx while D = g_zxv·Wxv is added to;
// z1 is recomputed from Hn, G and ‖ΔX‖ where it is needed again.  Every row is encoded with its own power-of-two scale
// (gradient rows span many orders of magnitude).  The row rules live in bwd_tc_common.cuh.
#include <cuda_fp16.h>

#include "bwd_common.cuh"
#include "bwd_tc_common.cuh"
#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct VirtBwdTcArgs {
    int64_t N;
    int B, C;
    unsigned flags;
    const int32_t* batch;
    const float* x4;
    const float* Hn;
    const float* Xv;
    const float* G;
    const float* w1r;
    const float* b2; const float* bxv; const float* w3xv; const float* bx; const float* w3x;
    const __half* wimg;       // [6][hi 4096 | lo 4096] operand images: W2v, Wxv, Wx, Wxvᵀ, Wxᵀ, W2vᵀ
    const float* g_aggv;
    const float* g_transv;
    const float* g_vsum;
    float* g_Hn;
    float* g_xv;
    float* g_G;
    float* g_Xv;
    float* g_w1r; float* g_w2; float* g_b2; float* g_wxv; float* g_bxv; float* g_w3xv;
    float* g_wx; float* g_bx; float* g_w3x;
};

constexpr int VT_THREADS = 128;
constexpr int VT_TM_COLS = 192;                                     // A / D 64 | A2 64 | z2 64
constexpr int VT_MAXC = DISTEGNN_MAX_CHANNELS;
constexpr int VT_IMG = 2 * 64 * 64;                                 // halfs per matrix image (hi + lo)
constexpr int VT_SMEM_BYTES = tmma::tm_bytes(VT_TM_COLS)
                              + 2 * VT_IMG * 2                      // two weight slots
                              + 2 * TILE_M * LDA * 4                // gradient tile + activation tile
                              + 6 * H * 4 + 6 * H * 4               // w1r, b2, bxv, w3xv, bx, w3x + gradient accumulators
                              + VT_MAXC * H * 4                     // Σ_i g_z1 per channel (-> g_G)
                              + 4 * VT_MAXC * 4                     // Σ_i gΔX per channel (-> g_Xv)
                              + TILE_M * 4 * 4                      // gΔX per row
                              + TILE_M * 4                          // ‖ΔX‖ per row
                              + TILE_M * 4                          // graph id per local node
                              + 256;                                // mbarriers

// fp16 hi/lo images of the six B operands in the shared-memory layout of tc16::stage_weight: forward matrices
// B[n][k] = W[n][k] = w_kmajor[k*64+n], transposed ones B[n][k] = W[k][n] = w_kmajor[n*64+k].
constexpr int VT_IMG_THREADS = 256;
__global__ void virtual_bwd_images_kernel(const float* w2, const float* wxv, const float* wx, __half* img) {
    const int m = blockIdx.x;                    // 0..5
    const float* src = (m == 0 || m == 5) ? w2 : ((m == 1 || m == 3) ? wxv : wx);
    __half* hi = img + (size_t)m * VT_IMG;
    if (m >= 3)
        tc16::stage_weight<VT_IMG_THREADS, true>(hi, hi + 64 * 64, src, 0, 64, threadIdx.x);
    else
        tc16::stage_weight<VT_IMG_THREADS>(hi, hi + 64 * 64, src, 0, 64, threadIdx.x);
}

__global__ void __launch_bounds__(VT_THREADS, 1) virtual_layer_bwd_tc_kernel(const VirtBwdTcArgs a) {
    using namespace tmma;
    uint8_t* const smem_raw = degnn_dyn_smem + tm_bytes(VT_TM_COLS);
    __half* slots = reinterpret_cast<__half*>(smem_raw);                     // [2 slots][VT_IMG]
    float* Gt = reinterpret_cast<float*>(slots + 2 * VT_IMG);                // gradient tile
    float* At = Gt + TILE_M * LDA;                                           // activation tile
    float* w1rs = At + TILE_M * LDA;
    float* b2s = w1rs + H;
    float* bxvs = b2s + H;
    float* w3xvs = bxvs + H;
    float* bxs = w3xvs + H;
    float* w3xs = bxs + H;
    float* gw1r = w3xs + H;
    float* gb2 = gw1r + H;
    float* gbxv = gb2 + H;
    float* gw3xv = gbxv + H;
    float* gbx = gw3xv + H;
    float* gw3x = gbx + H;
    float* accG = gw3x + H;                                                  // [C][64]
    float* accX = accG + VT_MAXC * H;                                        // [3][VT_MAXC] (pitch VT_MAXC, 4 rows)
    float* gdX = accX + 4 * VT_MAXC;                                         // [128][4]
    float* vrs = gdX + TILE_M * 4;                                           // [128]
    int* sgraph = reinterpret_cast<int*>(vrs + TILE_M);                      // [128]
    uint64_t* wbar = reinterpret_cast<uint64_t*>(sgraph + TILE_M);           // [2]: weight slot filled

    const int t = threadIdx.x, lane = t & 31, wq = t >> 5;
    const int C = a.C;
    const int K = 4 + 3 * C + H * C;
    const int TN = TILE_M / C;
    const float invC = 1.0f / (float)C;
    const bool need_feat = !(a.flags & DISTEGNN_FLAG_LAST) && a.g_aggv != nullptr;

    if (t < H) {
        w1rs[t] = a.w1r[t];
        b2s[t] = a.b2[t];
        bxvs[t] = a.bxv[t];
        w3xvs[t] = a.w3xv[t];
        bxs[t] = a.bx[t];
        w3xs[t] = a.w3x[t];
    }
    for (int i = t; i < 6 * H + VT_MAXC * H + 4 * VT_MAXC; i += VT_THREADS) gw1r[i] = 0.f;
    if (t == 0) {
        for (int i = 0; i < 2; ++i) mbar_init(&wbar[i], 1);
        fence_mbar_init();
    }
    fence_proxy_async_smem();
    __syncthreads();

    const uint32_t lane_off = ((uint32_t)(32 * wq)) << 16;
    const uint32_t tA_hi = lane_off, tA_lo = lane_off + 32, tD = lane_off;
    const uint32_t tA2_hi = lane_off + 64, tA2_lo = lane_off + 96, tZ2 = lane_off + 128;

    const int64_t num_tiles = (a.N + TN - 1) / TN;
    const int64_t my_tiles = blockIdx.x < num_tiles ? (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total_q = 6 * my_tiles;                        // matrices this CTA will consume, in order
    int64_t q_next = 0;                                          // next matrix to be requested (thread 0)
    auto request = [&]() {                                       // thread 0: stream matrix q_next into slot q_next & 1
        if (q_next < total_q) {
            const int slot = (int)(q_next & 1), m = (int)(q_next % 6);
            mbar_expect_tx(wbar + slot, VT_IMG * 2);
            bulk_g2s(slots + slot * VT_IMG, a.wimg + (size_t)m * VT_IMG, VT_IMG * 2, wbar + slot);
            ++q_next;
        }
    };
    if (t == 0) {
        request();
        request();
    }
    int64_t q_use = 0;                                           // next matrix to be used (same on all threads)
    // publish the A operand at tile-memory column `acol` (0: over D, 64: A2), wait for the weight slot, and run the
    // three split products over the whole tile: D (+)= A·Wᵀ
    auto issue = [&](uint32_t acol, bool accumulate) {
        fence_proxy_async_smem();
        __syncthreads();
        const int slot = (int)(q_use & 1);
        mbar_wait(wbar + slot, (uint32_t)((q_use >> 1) & 1));
        const __half* whi = slots + slot * VT_IMG;
        mma_f16x3_tile(0u, acol, acol + 32u, whi, whi + 64 * 64, accumulate);
        ++q_use;
    };
    auto mma_done = [&]() {                                      // D visible; the slot it read is refilled two matrices ahead
        __syncthreads();
        if (t == 0) request();
    };
    int cur_graph = -1;
    auto flush = [&](int g) {                                    // all threads; caller synchronises
        if (g >= 0) {
            for (int i = t; i < C * H; i += VT_THREADS) {
                atomicAdd(a.g_G + (size_t)g * C * H + i, accG[i]);
                accG[i] = 0.f;
            }
            if (t < 3 * C) {
                const int d = t / C, c = t - d * C;
                atomicAdd(a.g_Xv + (size_t)g * 3 * C + t, accX[d * VT_MAXC + c]);
                accX[d * VT_MAXC + c] = 0.f;
            }
        }
    };

    float gW2[8][4], gWxv[8][4], gWx[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) gW2[i][j] = gWxv[i][j] = gWx[i][j] = 0.f;

    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int64_t n0 = tile * TN;
        const int nvalid = (int)min((int64_t)TN, a.N - n0);
        const int rows = nvalid * C;
        if (t < TN) sgraph[t] = (t < nvalid) ? __ldg(a.batch + n0 + t) : -1;
        __syncthreads();
        const int g_first = sgraph[0];
        const bool single = (g_first == sgraph[nvalid - 1]);
        if (single && g_first != cur_graph) {
            flush(cur_graph);
            cur_graph = g_first;
            __syncthreads();
        }

        // ---- the thread's row: node, channel, geometry, upstream scalars -----------------------------------------------
        const bool rvalid = t < rows;
        const int nl = rvalid ? t / C : 0;
        const int ch = rvalid ? t - nl * C : 0;
        const int g = rvalid ? sgraph[nl] : g_first;
        const size_t node = (size_t)(n0 + nl);
        float dx, dy, dz, vr, gpxv = 0.f, gpx = 0.f;
        float4 gt = make_float4(0.f, 0.f, 0.f, 0.f);
        float gv0 = 0.f, gv1 = 0.f, gv2 = 0.f;
        {
            const float4 xi = ldg4(a.x4 + node * 4);
            const float* Xg = a.Xv + (size_t)g * 3 * C;
            dx = __ldg(Xg + ch) - xi.x; dy = __ldg(Xg + C + ch) - xi.y; dz = __ldg(Xg + 2 * C + ch) - xi.z;
            vr = sqrtf(dx * dx + dy * dy + dz * dz);
            if (rvalid) {
                gt = ldg4(a.g_transv + node * 4);
                const float* gv = a.g_vsum + (size_t)g * K + 4;
                gv0 = __ldg(gv + ch); gv1 = __ldg(gv + C + ch); gv2 = __ldg(gv + 2 * C + ch);
                gpxv = -(gt.x * dx + gt.y * dy + gt.z * dz) * invC;
                gpx = gv0 * dx + gv1 * dy + gv2 * dz;
            }
            vrs[t] = rvalid ? vr : 0.f;
        }

        // z1 = Hn[node] + G[graph,c] + w_r·‖ΔX‖ of the own row (stage 1, and again where SiLU(z1) / SiLU'(z1) are needed)
        auto z1_row = [&](float (&z1)[64]) {
            const float* hrow = a.Hn + node * H;
            const float* grow = a.G + ((size_t)g * C + ch) * H;
#pragma unroll
            for (int j4 = 0; j4 < 16; ++j4) {
                float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                if (rvalid) z = fma4(vr, *reinterpret_cast<const float4*>(w1rs + 4 * j4), add4(ldg4(hrow + 4 * j4), ldg4(grow + 4 * j4)));
                z1[4 * j4] = z.x; z1[4 * j4 + 1] = z.y; z1[4 * j4 + 2] = z.z; z1[4 * j4 + 3] = z.w;
            }
        };
        float v[64];
        // ---- stage 1: a1 = SiLU(z1) -> A;  MMA: z2 = a1·W2vᵀ ---------------------------------------------------------------
        {
            z1_row(v);
#pragma unroll
            for (int j = 0; j < 64; ++j) v[j] = rvalid ? silu(v[j]) : 0.f;
        }
        const float inv1 = encode_row_own_scale(v, tA_hi, tA_lo);
        issue(0u, false);                             // W2v
        mma_done();

        // ---- stage 2: z2 = D/s + b2v -> tile memory; mv = SiLU(z2) -> activation tile + A;  MMA: zxv = mv·Wxvᵀ --------------
        tm_load_row(tD, v);
#pragma unroll
        for (int j = 0; j < 64; ++j) v[j] = fmaf(v[j], inv1, b2s[j]);
        tm_store_row(tZ2, v);
#pragma unroll
        for (int j = 0; j < 64; ++j) v[j] = silu(v[j]);
        smem_store_row(At + t * LDA, v);
        const float inv2 = encode_row_own_scale(v, tA2_hi, tA2_lo);
        issue(64u, false);                            // Wxv
        mma_done();

        // ---- head xv: φ_xv, g_w3xv, g_zxv -> gradient tile; mv -> A again;  MMA: zx = mv·Wxᵀ -----------------------------------
        tm_load_row(tD, v);
        const float phixv = phi_head_bwd(v, inv2, bxvs, w3xvs, gpxv, gw3xv, lane);
        smem_store_row(Gt + t * LDA, v);
        float fm = row_absmax(v);                     // the two heads' gradient rows share one scale (one accumulator)
        issue(64u, false);                            // Wx (A2 unchanged: still mv); the barrier inside publishes both tiles
        wgrad128(gWxv, Gt, At, t);                    // g_Wxv += g_zxvᵀ·mv
        tile_colsum(gbxv, Gt, t);
        __syncthreads();                              // gradient tile fully read
        mma_done();

        // ---- head x: φ_X, g_w3x, g_zx;  MMAs: g_mv = g_zxv·Wxv + g_zx·Wx -----------------------------------------------------
        float gzx[64];
        tm_load_row(tD, gzx);
        const float phix = phi_head_bwd(gzx, inv2, bxs, w3xs, gpx, gw3x, lane);
        fm = row_absmax(gzx, fm);
        float sc, inv3;
        row_scale(fm, sc, inv3);
#pragma unroll
        for (int j4 = 0; j4 < 16; ++j4) {             // g_zxv back from the own row of the gradient tile (kept out of the
            const float4 q4 = *reinterpret_cast<const float4*>(Gt + t * LDA + 4 * j4);   // registers during the head)
            v[4 * j4] = q4.x; v[4 * j4 + 1] = q4.y; v[4 * j4 + 2] = q4.z; v[4 * j4 + 3] = q4.w;
        }
        encode_row(v, sc, tA_hi, tA_lo);              // A = g_zxv
        issue(0u, false);                             // Wxvᵀ
        smem_store_row(Gt + t * LDA, gzx);            // the gradient tile now holds g_zx (its readers passed the barrier above)
        mma_done();
        encode_row(gzx, sc, tA2_hi, tA2_lo);          // A2 = g_zx
        issue(64u, true);                             // Wxᵀ, accumulating; the barrier inside publishes the g_zx tile
        wgrad128(gWx, Gt, At, t);                     // g_Wx += g_zxᵀ·mv
        tile_colsum(gbx, Gt, t);
        __syncthreads();                              // both tiles fully read
        mma_done();

        // ---- g_z2 = (g_mv + upstream) ⊙ SiLU'(z2) -> gradient tile + A; a1 -> activation tile;  MMA: g_a1 = g_z2·W2v ------------
        float inv4;
        {
            tm_load_row(tD, v);
            tm_load_row(tZ2, gzx);                  // reuse as z2
            const bool up = need_feat && rvalid;
            const float* ga = a.g_aggv + node * H;
            const float* gs = a.g_vsum + (size_t)g * K + 4 + 3 * C + ch * H;
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                float gm = v[j] * inv3;
                if (up) gm += fmaf(__ldg(ga + j), invC, __ldg(gs + j));
                v[j] = gm * dsilu(gzx[j]);
            }
            smem_store_row(Gt + t * LDA, v);
            inv4 = encode_row_own_scale(v, tA_hi, tA_lo);
            z1_row(gzx);                            // z1 -> a1 row for the weight gradient
#pragma unroll
            for (int j = 0; j < 64; ++j) gzx[j] = rvalid ? silu(gzx[j]) : 0.f;
            smem_store_row(At + t * LDA, gzx);
        }
        issue(0u, false);                             // W2vᵀ
        wgrad128(gW2, Gt, At, t);                     // g_W2v += g_z2ᵀ·a1
        tile_colsum(gb2, Gt, t);
        __syncthreads();
        mma_done();

        // ---- g_z1 = D/s ⊙ SiLU'(z1) -> gradient tile; g_vr; geometry gradient ---------------------------------------------------
        {
            tm_load_row(tD, v);
            z1_row(gzx);
            float gr = 0.f;
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                v[j] = v[j] * inv4 * dsilu(gzx[j]);
                gr = fmaf(v[j], w1rs[j], gr);
            }
            smem_store_row(Gt + t * LDA, v);
            // gΔX = −g_trans_v·φ_xv/C + g_vsum·φ_X + g_vr·ΔX/‖ΔX‖
            const float s1 = -phixv * invC, s3 = vr > 0.f ? gr / vr : 0.f;
            float4 gd = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rvalid) gd = make_float4(fmaf(gt.x, s1, fmaf(gv0, phix, s3 * dx)), fmaf(gt.y, s1, fmaf(gv1, phix, s3 * dy)),
                                         fmaf(gt.z, s1, fmaf(gv2, phix, s3 * dz)), 0.f);
            *reinterpret_cast<float4*>(gdX + 4 * t) = gd;
        }
        __syncthreads();                              // g_z1 tile and gΔX visible

        // ---- reductions of the g_z1 tile and of gΔX ------------------------------------------------------------------------------
        {
            const int c64 = t & 63, h = t >> 6;
            for (int n = h; n < nvalid; n += 2) {           // g_Hn[node] = Σ_c g_z1
                float s = 0.f;
                for (int c = 0; c < C; ++c) s += Gt[(n * C + c) * LDA + c64];
                a.g_Hn[(size_t)(n0 + n) * H + c64] = s;
            }
            if (single) {                                    // Σ_i g_z1 per channel -> g_G
                for (int c = h; c < C; c += 2) {
                    float s = 0.f;
                    for (int n = 0; n < nvalid; ++n) s += Gt[(n * C + c) * LDA + c64];
                    accG[c * H + c64] += s;
                }
            } else {
                for (int n = h; n < nvalid; n += 2)
                    for (int c = 0; c < C; ++c)
                        atomicAdd(a.g_G + ((size_t)sgraph[n] * C + c) * H + c64, Gt[(n * C + c) * LDA + c64]);
            }
            float sr = 0.f;                                  // g_w_vr[n] += Σ_rows g_z1[row][n]·‖ΔX‖_row
            for (int q = 64 * h; q < 64 * h + 64; ++q) sr = fmaf(Gt[q * LDA + c64], vrs[q], sr);
            atomicAdd(gw1r + c64, sr);
        }
        if (t < nvalid) {                                    // g_x (virtual part) = −Σ_c gΔX
            float sx = 0.f, sy = 0.f, sz = 0.f;
            for (int c = 0; c < C; ++c) {
                const float4 gg = *reinterpret_cast<const float4*>(gdX + 4 * (t * C + c));
                sx += gg.x; sy += gg.y; sz += gg.z;
            }
            *reinterpret_cast<float4*>(a.g_xv + (size_t)(n0 + t) * 4) = make_float4(-sx, -sy, -sz, 0.f);
        }
        if (t >= 64 && t < 64 + 3 * C) {                     // g_Xv[b,d,c] += Σ_i gΔX_d
            const int k = t - 64, d = k / C, c = k - d * C;
            if (single) {
                float s = 0.f;
                for (int n = 0; n < nvalid; ++n) s += gdX[4 * (n * C + c) + d];
                accX[d * VT_MAXC + c] += s;
            } else {
                for (int n = 0; n < nvalid; ++n) atomicAdd(a.g_Xv + (size_t)sgraph[n] * 3 * C + k, gdX[4 * (n * C + c) + d]);
            }
        }
        __syncthreads();                              // tiles and per-row arrays are rewritten by the next iteration
    }
    flush(cur_graph);

    wgrad128_flush(a.g_w2, gW2, t);
    wgrad128_flush(a.g_wxv, gWxv, t);
    wgrad128_flush(a.g_wx, gWx, t);
    __syncthreads();
    if (t < H) {
        atomicAdd(a.g_w1r + t, gw1r[t]);
        atomicAdd(a.g_b2 + t, gb2[t]);
        atomicAdd(a.g_bxv + t, gbxv[t]);
        atomicAdd(a.g_w3xv + t, gw3xv[t]);
        atomicAdd(a.g_bx + t, gbx[t]);
        atomicAdd(a.g_w3x + t, gw3x[t]);
    }
}

}  // namespace degnn

extern "C" int distegnn_virtual_bwd_prepare(int A, int C, int Na, const float* layer_params, void* weight_images,
                                            void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    DEGNN_CHECK_ARG(layer_params && weight_images, "null pointer");
    Layout L = make_layout(A, C, Na);
    virtual_bwd_images_kernel<<<6, VT_IMG_THREADS, 0, (cudaStream_t)stream>>>(layer_params + L.off[DISTEGNN_P_V_W2],
                                                                              layer_params + L.off[DISTEGNN_P_V_WXV],
                                                                              layer_params + L.off[DISTEGNN_P_V_WX],
                                                                              reinterpret_cast<__half*>(weight_images));
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_virtual_layer_bwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                          const int32_t* batch32, const float* x4, const float* Hn, const float* Xv,
                                          const float* G, const float* layer_params, const void* weight_images,
                                          const float* g_agg_v, const float* g_trans_v, const float* g_vsum,
                                          float* g_Hn, float* g_xv, float* g_G, float* g_Xv, float* g_layer_params,
                                          void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(batch32 && x4 && Hn && Xv && G && layer_params && weight_images && g_trans_v && g_vsum && g_Hn && g_xv &&
                        g_G && g_Xv && g_layer_params,
                    "null pointer");
    Layout L = make_layout(A, C, Na);
    VirtBwdTcArgs a;
    a.N = n_nodes; a.B = n_graphs; a.C = C; a.flags = flags;
    a.batch = batch32; a.x4 = x4; a.Hn = Hn; a.Xv = Xv; a.G = G;
    a.w1r = layer_params + L.off[DISTEGNN_P_V_W1R];
    a.b2 = layer_params + L.off[DISTEGNN_P_V_B2];
    a.bxv = layer_params + L.off[DISTEGNN_P_V_BXV];
    a.w3xv = layer_params + L.off[DISTEGNN_P_V_W3XV];
    a.bx = layer_params + L.off[DISTEGNN_P_V_BX];
    a.w3x = layer_params + L.off[DISTEGNN_P_V_W3X];
    a.wimg = reinterpret_cast<const __half*>(weight_images);
    a.g_aggv = g_agg_v; a.g_transv = g_trans_v; a.g_vsum = g_vsum;
    a.g_Hn = g_Hn; a.g_xv = g_xv; a.g_G = g_G; a.g_Xv = g_Xv;
    a.g_w1r = g_layer_params + L.off[DISTEGNN_P_V_W1R];
    a.g_w2 = g_layer_params + L.off[DISTEGNN_P_V_W2];
    a.g_b2 = g_layer_params + L.off[DISTEGNN_P_V_B2];
    a.g_wxv = g_layer_params + L.off[DISTEGNN_P_V_WXV];
    a.g_bxv = g_layer_params + L.off[DISTEGNN_P_V_BXV];
    a.g_w3xv = g_layer_params + L.off[DISTEGNN_P_V_W3XV];
    a.g_wx = g_layer_params + L.off[DISTEGNN_P_V_WX];
    a.g_bx = g_layer_params + L.off[DISTEGNN_P_V_BX];
    a.g_w3x = g_layer_params + L.off[DISTEGNN_P_V_W3X];
    ensure_dynamic_smem((const void*)virtual_layer_bwd_tc_kernel, (int)VT_SMEM_BYTES);
    const int TN = TILE_M / C;
    int64_t grid = (n_nodes + TN - 1) / TN;
    if (grid > sm_count()) grid = sm_count();
    virtual_layer_bwd_tc_kernel<<<(unsigned)grid, VT_THREADS, VT_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
