// Node update of one E_GCL_vel layer on the tensor cores — production kernel behind distegnn_node_layer_fwd.
// Replaces reference models/FastEGNN.py:177-183 (sum of the three coordinate terms, φ_v) and :203-217
// (node_model) and emits the per-node operands of the NEXT layer's fused stages (P, Q, Hn; SURVEY §7 "W1 split").
// Same math/outputs as node_layer.cu's fp32-FMA kernel (kept as ..._simt for cross-checks).
//
// One CTA per SM, NT_WG warpgroups, each an independent pipeline: a warpgroup grid-strides over its own 64-node tiles and,
// once set up, shares no barrier with the other warpgroups.  Warp w of a warpgroup owns nodes 16w .. 16w+15 of its tile,
// which are exactly the rows of the m64n64 accumulator fragment it holds (tile_mma.cuh); thread (g = lane/4, q = lane%4)
// owns rows g and g+8 of the warp, columns 8j + 2q + {0,1}, and reads and writes the rows of h, agg_m, agg_v, h', P, Q, Hn
// in that layout (a quad covers one 32-byte sector of a row per column block j).  All eight 64x64 GEMMs take their A
// operand from registers (fp16 2-term split, tc16.cuh) and keep the accumulator there; the weights (hi/lo, 128 KB) stay
// resident in shared memory, shared by the four pipelines.  Sequence per tile:
//                      h -> A;                                MMA: D = h·Lᵀ;  φ_v per row (quad shuffles)
//                      x' and Σ(x',1) from φ_v (lane q <-> coordinate q of the thread's rows)
//                      MMA: D = h·N1aᵀ;   agg_m/deg -> A; MMA: D += ·N1bᵀ;   agg_v -> A; MMA: D += ·N1cᵀ  (one row scale)
//                      t1 = SiLU(D + attr·N1d + b1) -> A;     MMA: D = t1·N2ᵀ
//                      h' = h + D + b2 -> HBM, -> A;          3 x (MMA: D = h'·W'ᵀ, W' = W1a', W1b', W1vh'; D -> P / Q / Hn)
// FLAG_LAST runs the first line and x' only.
#include "common.cuh"
#include "tc16.cuh"
#include "tile_mma.cuh"

namespace degnn {

struct NodeTcArgs {
    int64_t N;
    int B, Na, K;
    unsigned flags;
    const int32_t* rowptr; const int32_t* batch;
    const float* h; const float* x4; const float* vel; const float* attr;
    const float* agg_m; const float* agg_x; const float* agg_v; const float* trans_v;
    const float* lw; const float* lb; const float* lw3; const float* lb3;          // φ_v
    const float* n1; const float* nb1; const float* n2; const float* nb2;          // node MLP
    const float* nw1a; const float* nxb1; const float* nw1b; const float* nw1h;    // next layer
    float* h_out; float* x4_out; float* P; float* Q; float* Hn; float* loc_out; float* vsum;
};

// 4 warpgroups = 16 warps per SM
constexpr int NT_WG = 4;
constexpr int NT_THREADS = 128 * NT_WG, NT_WARPS = NT_THREADS / 32;
constexpr int NT_TILE = 64;                                   // nodes per warpgroup tile
constexpr int NT_W = H * H;                                   // fp16 elements per 64x64 weight matrix
constexpr uint32_t NT_LBO64 = tc16::lbo_bytes(64), NT_LBO192 = tc16::lbo_bytes(192);
constexpr uint64_t NT_DESC_N64 = (64 / 8 * 128) >> 4;         // descriptor step to B row n + 64 (8-row groups 128 B apart)
// weights L, N1a-c, N2, NEXT (hi+lo) | lb, lw3, nb1, nb2, nxb1, N1d [Na][64] | Σ(x,1) per warp
constexpr int NT_SMEM_BYTES = 16 * NT_W * 2 + (5 * H + DISTEGNN_MAX_NODE_ATTR * H + NT_WARPS * 4) * 4;
// weights NEXT (hi+lo) | embedding [F][64], bias, nxb1 | Σ(x,1) per warp
constexpr int ET_SMEM_BYTES = 6 * NT_W * 2 + ((DISTEGNN_MAX_NODE_FEAT + 2) * H + NT_WARPS * 4) * 4;

// The calling thread's two rows of its warpgroup's tile: a = row 16w + g, b = a + 8 (valid: < N), their node ids (a valid
// node for rows past N, never read for them) and q = lane % 4: its column pairs are 8j + 2q, +1.
struct Rows {
    int q;
    bool va, vb;
    size_t na, nb;
};
__device__ __forceinline__ f32x2 ld_pair(const float* p) { return *reinterpret_cast<const f32x2*>(p); }
__device__ __forceinline__ void st_pair(float* p, f32x2 v) { *reinterpret_cast<f32x2*>(p) = v; }
// Pull bytes [p, p + n) towards L2: one 128-byte line per thread of a warpgroup (t < 128) and step
__device__ __forceinline__ void prefetch_l2_range(const void* p, size_t n, int t) {
    const uintptr_t b = (uintptr_t)p, e = b + n;
    for (uintptr_t l = (b & ~(uintptr_t)127) + 128u * (uintptr_t)t; l < e; l += 128u * 128u)
        tmma::prefetch_l2((const void*)l);
}

// Σ(x, 1) per graph into vsum[:, 0:4].  Lane q of a quad holds entry q of its rows a and b.  Tiles inside one graph add to
// per-warp sums in shared memory, flushed by the warpgroup (one atomic per entry) when its graph changes and at the end;
// tiles that straddle graphs add their rows to vsum directly.
struct XSum {
    float* vsum;
    int K;
    float* acc_w;      // this warp's four sums
    float* acc_g;      // the four warps' sums of the group
    uint32_t bar;      // the group's named barrier
    int t, lane;
    int cur;           // graph of the sums (group-uniform)
    __device__ __forceinline__ void flush() {
        if (cur >= 0 && t < 4) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s += acc_g[4 * k + t];
                acc_g[4 * k + t] = 0.f;
            }
            atomicAdd(vsum + (size_t)cur * K + t, s);
        }
    }
    __device__ __forceinline__ void start_tile(int g_first, bool single) {   // group-uniform; rare: once per graph
        if (single && g_first != cur) {
            tmma::named_bar(bar, 128);         // every warp is done with its sums
            flush();
            cur = g_first;
            tmma::named_bar(bar, 128);
        }
    }
    __device__ __forceinline__ void add(bool single, const Rows& r, float xa, float xb, int ga, int gb) {
        if (single) {
            float s = (r.va ? xa : 0.f) + (r.vb ? xb : 0.f);
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) s += __shfl_xor_sync(FULL, s, o);
            if (lane < 4) acc_w[lane] += s;
        } else {
            if (r.va) atomicAdd(vsum + (size_t)ga * K + r.q, xa);
            if (r.vb) atomicAdd(vsum + (size_t)gb * K + r.q, xb);
        }
    }
    __device__ __forceinline__ void finish() {
        tmma::named_bar(bar, 128);
        flush();
    }
};

// h rows -> h_out (rows < N) and A; P, Q, Hn = h·[W1a; W1b; W1vh]ᵀ, 64 columns at a time, with E_B1 added to P.
// hrow(j, xa, xb) gives column pair j of rows a and b.  Rows out of the fp16 range are re-encoded from what was stored to
// h_out (which may be the kernel's h input, so h cannot be read again).
template <class Hrow>
__device__ __forceinline__ void store_h_project(Hrow&& hrow, const Rows& r, float* h_out, float* P, float* Q, float* Hn,
                                                uint64_t b_hi, uint64_t b_lo, const float* nxb1s, float (&d)[32],
                                                uint32_t (&ahi)[16], uint32_t (&alo)[16]) {
    tc16::RowScales s;
    tc16::encode_rows<true>(
        [&](int j, f32x2& xa, f32x2& xb, auto pass) {
            const int col = 8 * j + 2 * r.q;
            if constexpr (decltype(pass)::value == tc16::FAST_PASS) {
                hrow(j, xa, xb);
                if (r.va) st_pair(h_out + r.na * H + col, xa);
                if (r.vb) st_pair(h_out + r.nb * H + col, xb);
            } else {
                xa = r.va ? ld_pair(h_out + r.na * H + col) : 0ull;
                xb = r.vb ? ld_pair(h_out + r.nb * H + col) : 0ull;
            }
        },
        ahi, alo, s);
    const float ia = s.a == 1.0f ? 1.0f : 1.0f / s.a, ib = s.b == 1.0f ? 1.0f : 1.0f / s.b;
#pragma unroll 1
    for (int o = 0; o < 3; ++o) {
        tc16::mma_f16x3_rA<NT_LBO192>(d, ahi, alo, b_hi + o * NT_DESC_N64, b_lo + o * NT_DESC_N64);
        tc16::mma_f16x3_rA_wait(d, ahi, alo);
        float* dst = o == 0 ? P : (o == 1 ? Q : Hn);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int col = 8 * j + 2 * r.q;
            float ya0 = d[4 * j + 0] * ia, ya1 = d[4 * j + 1] * ia, yb0 = d[4 * j + 2] * ib, yb1 = d[4 * j + 3] * ib;
            if (o == 0) {
                const float b0 = nxb1s[col], b1 = nxb1s[col + 1];
                ya0 += b0; ya1 += b1; yb0 += b0; yb1 += b1;
            }
            if (r.va) st_pair(dst + r.na * H + col, pk2(ya0, ya1));
            if (r.vb) st_pair(dst + r.nb * H + col, pk2(yb0, yb1));
        }
    }
}

__global__ void __launch_bounds__(NT_THREADS, 1) node_layer_tc_kernel(const NodeTcArgs a) {
    using namespace tmma;
    __half* Lhi = reinterpret_cast<__half*>(degnn_dyn_smem);
    __half* Llo = Lhi + NT_W;
    __half* N1hi = Llo + NT_W;            // [3][4096]
    __half* N1lo = N1hi + 3 * NT_W;
    __half* N2hi = N1lo + 3 * NT_W;
    __half* N2lo = N2hi + NT_W;
    __half* NXhi = N2lo + NT_W;           // 192 x 64
    __half* NXlo = NXhi + 3 * NT_W;
    float* lbs = reinterpret_cast<float*>(NXlo + 3 * NT_W);
    float* lw3s = lbs + H;
    float* nb1s = lw3s + H;
    float* nb2s = nb1s + H;
    float* nxb1s = nb2s + H;
    float* n1ds = nxb1s + H;              // [Na][64]
    float* accx_all = n1ds + DISTEGNN_MAX_NODE_ATTR * H;          // [warps][4]: Σ(x',1)

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int wg = warp >> 2, w = warp & 3, t = tid & 127;
    const int q = lane & 3;
    const bool last = a.flags & DISTEGNN_FLAG_LAST;
    const bool zero_agg = a.flags & DISTEGNN_FLAG_ZERO_AGG;   // leave agg_m / agg_x zeroed for the next edge stage
    const int Na = a.Na;

    // ---- one-time setup ---------------------------------------------------------------------------
    tc16::stage_weight<NT_THREADS>(Lhi, Llo, a.lw, 0, 64, tid);
    if (!last) {
        for (int c = 0; c < 3; ++c) tc16::stage_weight<NT_THREADS>(N1hi + c * NT_W, N1lo + c * NT_W, a.n1 + c * H * H, 0, 64, tid);
        tc16::stage_weight<NT_THREADS>(N2hi, N2lo, a.n2, 0, 64, tid);
        tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1a, 0, 192, tid);
        tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1b, 64, 192, tid);
        tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1h, 128, 192, tid);
    }
    if (tid < H) {
        lbs[tid] = a.lb[tid];
        lw3s[tid] = a.lw3[tid];
        if (!last) {
            nb1s[tid] = a.nb1[tid];
            nb2s[tid] = a.nb2[tid];
            nxb1s[tid] = a.nxb1[tid];
        }
    }
    if (!last)
        for (int i = tid; i < Na * H; i += NT_THREADS) n1ds[i] = a.n1[(size_t)3 * H * H + i];
    if (tid < NT_WARPS * 4) accx_all[tid] = 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    auto desc = [&](const __half* p, uint32_t lbo) { return make_desc(smem_u32(p), lbo, 128); };
    const uint64_t dLhi = desc(Lhi, NT_LBO64), dLlo = desc(Llo, NT_LBO64);
    const uint64_t dN2hi = desc(N2hi, NT_LBO64), dN2lo = desc(N2lo, NT_LBO64);
    const uint64_t dNXhi = desc(NXhi, NT_LBO192), dNXlo = desc(NXlo, NT_LBO192);
    XSum xs{a.vsum, a.K, accx_all + 4 * warp, accx_all + 16 * wg, 1u + (uint32_t)wg, t, lane, -1};
    const int ra = 16 * w + (lane >> 2), rb = ra + 8;             // the thread's tile rows

    const int64_t num_tiles = (a.N + NT_TILE - 1) / NT_TILE;
    for (int64_t tile = (int64_t)blockIdx.x * NT_WG + wg; tile < num_tiles; tile += (int64_t)gridDim.x * NT_WG) {
        const int64_t n0 = tile * NT_TILE;
        const int nvalid = (int)min((int64_t)NT_TILE, a.N - n0);
        Rows r;
        r.q = q;
        r.va = ra < nvalid;
        r.vb = rb < nvalid;
        r.na = (size_t)(n0 + (r.va ? ra : 0));
        r.nb = (size_t)(n0 + (r.vb ? rb : 0));
        {   // pull the next tile's inputs towards L2: a tile takes many DRAM round trips, each of them waited for
            const int64_t m0 = n0 + (int64_t)gridDim.x * NT_WG * NT_TILE;
            if (m0 < a.N) {
                const size_t mv = (size_t)min((int64_t)NT_TILE, a.N - m0), m = (size_t)m0;
                prefetch_l2_range(a.h + m * H, mv * H * 4, t);
                if (!last) {
                    prefetch_l2_range(a.agg_m + m * H, mv * H * 4, t);
                    prefetch_l2_range(a.agg_v + m * H, mv * H * 4, t);
                    if (Na) prefetch_l2_range(a.attr + m * Na, mv * Na * 4, t);
                }
                prefetch_l2_range(a.x4 + m * 4, mv * 16, t);
                prefetch_l2_range(a.agg_x + m * 4, mv * 16, t);
                prefetch_l2_range(a.trans_v + m * 4, mv * 16, t);
                prefetch_l2_range(a.vel + m * 3, mv * 12, t);
                prefetch_l2_range(a.rowptr + m, (mv + 1) * 4, t);
                prefetch_l2_range(a.batch + m, mv * 4, t);
            }
        }
        const int g_first = __ldg(a.batch + n0), g_last = __ldg(a.batch + n0 + nvalid - 1);
        const bool single = g_first == g_last;
        xs.start_tile(g_first, single);
        // plain (coherent) loads of the rows: h is also this kernel's h_out in FastEGNN's layer loop, and agg_m is cleared
        auto rows_of = [&](const float* src, int j, f32x2& xa, f32x2& xb) {
            xa = r.va ? ld_pair(src + r.na * H + 8 * j + 2 * q) : 0ull;
            xb = r.vb ? ld_pair(src + r.nb * H + 8 * j + 2 * q) : 0ull;
        };

        // ---- h -> A (fp16 hi/lo);  D = h·Lᵀ -------------------------------------------------------------------
        uint32_t ahi[16], alo[16];
        tc16::RowScales sh;
        tc16::encode_rows<true>([&](int j, f32x2& xa, f32x2& xb, auto) { rows_of(a.h, j, xa, xb); }, ahi, alo, sh);
        float d[32];
        tc16::mma_f16x3_rA<NT_LBO64>(d, ahi, alo, dLhi, dLlo);
        float inv_deg_a = 0.f, inv_deg_b = 0.f;
        if (r.va) inv_deg_a = 1.0f / (float)max(__ldg(a.rowptr + r.na + 1) - __ldg(a.rowptr + r.na), 1);
        if (r.vb) inv_deg_b = 1.0f / (float)max(__ldg(a.rowptr + r.nb + 1) - __ldg(a.rowptr + r.nb), 1);
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- φ_v(h) (FastEGNN.py:183: the OLD h) per row --------------------------------------------------------
        float phia = 0.f, phib = 0.f;
        {
            const float iha = 1.0f / sh.a, ihb = 1.0f / sh.b;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + 2 * q + e;
                    phia = fmaf(silu(fmaf(d[4 * j + e], iha, lbs[col])), lw3s[col], phia);
                    phib = fmaf(silu(fmaf(d[4 * j + 2 + e], ihb, lbs[col])), lw3s[col], phib);
                }
            const float lb3 = __ldg(a.lb3);
            phia = lb3 + tc16::quad_sum(phia);
            phib = lb3 + tc16::quad_sum(phib);
        }

        // ---- x' = x + agg_x/deg + trans_v + φ_v·v, entry q of the thread's rows (q = 3: x' has 0, Σ(x',1) counts 1) ------
        {
            // every load of both rows before the first store (the stores may alias the loaded rows)
            const bool v[2] = {r.va, r.vb};
            const size_t node[2] = {r.na, r.nb};
            float x[2], ax[2], tv[2], vel[2], xn[2];
            int gr[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                x[i] = ax[i] = tv[i] = vel[i] = 0.f;
                gr[i] = g_first;
                if (v[i]) {
                    x[i] = a.x4[node[i] * 4 + q];                     // plain loads: x4 may be x4_out, agg_x is cleared
                    ax[i] = a.agg_x[node[i] * 4 + q];
                    tv[i] = __ldg(a.trans_v + node[i] * 4 + q);
                    if (q < 3) vel[i] = __ldg(a.vel + node[i] * 3 + q);
                    if (!single) gr[i] = __ldg(a.batch + node[i]);
                }
            }
            const float phi[2] = {phia, phib}, inv_deg[2] = {inv_deg_a, inv_deg_b};
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                xn[i] = q < 3 ? x[i] + ax[i] * inv_deg[i] + tv[i] + phi[i] * vel[i] : 0.f;
                if (v[i]) {
                    if (zero_agg) const_cast<float*>(a.agg_x)[node[i] * 4 + q] = 0.f;
                    if (q < 3 && a.loc_out) a.loc_out[node[i] * 3 + q] = xn[i];
                    a.x4_out[node[i] * 4 + q] = xn[i];
                }
                if (q == 3) xn[i] = 1.0f;
            }
            xs.add(single, r, xn[0], xn[1], gr[0], gr[1]);
        }
        if (last) continue;

        // ---- node MLP layer 1: h·N1aᵀ + (agg_m / deg)·N1bᵀ + agg_v·N1cᵀ  (D accumulates with one row scale) -----------
        // The first GEMM is not issued before the coordinate update above: with it in flight there, ptxas serialises the
        // kernel's wgmma (C7518).
        tc16::mma_f16x3_rA<NT_LBO64>(d, ahi, alo, desc(N1hi, NT_LBO64), desc(N1lo, NT_LBO64));   // A still holds h
        tc16::mma_f16x3_rA_wait(d, ahi, alo);
        float s2a = sh.a, s2b = sh.b;                 // the scales the D rows currently carry
        auto l1_chunk = [&](const float* src, float rsa, float rsb, int c, bool zero_src) {
            tc16::RowScales sn{s2a, s2b};
            tc16::encode_rows<true>(
                [&](int j, f32x2& xa, f32x2& xb, auto) {
                    rows_of(src, j, xa, xb);
                    xa = mul2(xa, bc2(rsa));
                    xb = mul2(xb, bc2(rsb));
                },
                ahi, alo, sn);
            if (zero_src)                             // after the last read of the rows
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (r.va) st_pair(const_cast<float*>(src) + r.na * H + 8 * j + 2 * q, 0ull);
                    if (r.vb) st_pair(const_cast<float*>(src) + r.nb * H + 8 * j + 2 * q, 0ull);
                }
            if (__any_sync(FULL, sn.a != s2a || sn.b != s2b)) {   // cold: bring the partial sums in D to the new row scales
                const float fa = sn.a / s2a, fb = sn.b / s2b;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    d[4 * j + 0] *= fa; d[4 * j + 1] *= fa;
                    d[4 * j + 2] *= fb; d[4 * j + 3] *= fb;
                }
                s2a = sn.a;
                s2b = sn.b;
            }
            tc16::mma_f16x3_rA<NT_LBO64, true>(d, ahi, alo, desc(N1hi + c * NT_W, NT_LBO64), desc(N1lo + c * NT_W, NT_LBO64));
            tc16::mma_f16x3_rA_wait(d, ahi, alo);
        };
        l1_chunk(a.agg_m, inv_deg_a, inv_deg_b, 1, zero_agg);
        l1_chunk(a.agg_v, 1.0f, 1.0f, 2, false);

        // ---- t1 = SiLU(D/s + attr·N1d + b1) -> A;  D = t1·N2ᵀ ----------------------------------------------
        float attra[DISTEGNN_MAX_NODE_ATTR], attrb[DISTEGNN_MAX_NODE_ATTR];
#pragma unroll
        for (int k = 0; k < DISTEGNN_MAX_NODE_ATTR; ++k) {
            attra[k] = (k < Na && r.va) ? __ldg(a.attr + r.na * Na + k) : 0.f;
            attrb[k] = (k < Na && r.vb) ? __ldg(a.attr + r.nb * Na + k) : 0.f;
        }
        tc16::RowScales st;
        {
            const float i2a = 1.0f / s2a, i2b = 1.0f / s2b;
            tc16::encode_rows<true>(
                [&](int j, f32x2& xa, f32x2& xb, auto) {
                    float za[2], zb[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * j + 2 * q + e;
                        za[e] = fmaf(d[4 * j + e], i2a, nb1s[col]);
                        zb[e] = fmaf(d[4 * j + 2 + e], i2b, nb1s[col]);
#pragma unroll
                        for (int k = 0; k < DISTEGNN_MAX_NODE_ATTR; ++k)
                            if (k < Na) {
                                za[e] = fmaf(attra[k], n1ds[k * H + col], za[e]);
                                zb[e] = fmaf(attrb[k], n1ds[k * H + col], zb[e]);
                            }
                    }
                    xa = pk2(silu(za[0]), silu(za[1]));
                    xb = pk2(silu(zb[0]), silu(zb[1]));
                },
                ahi, alo, st);
        }
        tc16::mma_f16x3_rA<NT_LBO64>(d, ahi, alo, dN2hi, dN2lo);
        tc16::mma_f16x3_rA_wait(d, ahi, alo);

        // ---- h' = h + D/s + b2 -> HBM and -> A;  P, Q, Hn = h'·[W1a';W1b';W1vh']ᵀ -----------------------------------
        const float ita = st.a == 1.0f ? 1.0f : 1.0f / st.a, itb = st.b == 1.0f ? 1.0f : 1.0f / st.b;
        store_h_project(
            [&](int j, f32x2& xa, f32x2& xb) {
                const int col = 8 * j + 2 * q;
                f32x2 ha, hb;
                rows_of(a.h, j, ha, hb);
                float h0, h1;
                upk2(ha, h0, h1);
                xa = pk2(h0 + fmaf(d[4 * j + 0], ita, nb2s[col]), h1 + fmaf(d[4 * j + 1], ita, nb2s[col + 1]));
                upk2(hb, h0, h1);
                xb = pk2(h0 + fmaf(d[4 * j + 2], itb, nb2s[col]), h1 + fmaf(d[4 * j + 3], itb, nb2s[col + 1]));
            },
            r, a.h_out, a.P, a.Q, a.Hn, dNXhi, dNXlo, nxb1s, d, ahi, alo);
    }
    xs.finish();
}

// =================================================================================================
// embedding prologue on the tensor cores (FastEGNN.forward, reference models/FastEGNN.py:298-302):
// h0 = embedding_in(node_feat) per node (F <= 16 inputs: plain FMAs, straight into the A fragments), then P/Q/Hn of
// layer 0 as three N = 64 GEMMs (store_h_project); also node_loc -> x4, data_batch -> int32, and Σ(x,1) per graph into
// vsum.  Same CTA layout as the node kernel.
// =================================================================================================
struct EmbedTcArgs {
    int64_t N;
    int B, F, K;
    const float* feat; const float* loc; const int64_t* batch64;
    const float* wt; const float* bias;                                  // [F][64], [64]
    const float* nw1a; const float* nxb1; const float* nw1b; const float* nw1h;
    float* h; float* x4; int32_t* batch32; float* P; float* Q; float* Hn; float* vsum;
    int32_t* n_invalid;                                                   // device counter of bad data_batch entries (or null)
};

__global__ void __launch_bounds__(NT_THREADS, 1) embed_tc_kernel(const EmbedTcArgs a) {
    using namespace tmma;
    __half* NXhi = reinterpret_cast<__half*>(degnn_dyn_smem);
    __half* NXlo = NXhi + 3 * NT_W;
    float* wts = reinterpret_cast<float*>(NXlo + 3 * NT_W);     // [F][64]
    float* bs = wts + DISTEGNN_MAX_NODE_FEAT * H;
    float* nxb1s = bs + H;
    float* accx_all = nxb1s + H;                                // [warps][4]: Σ(x,1)
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int wg = warp >> 2, w = warp & 3, t = tid & 127;
    const int q = lane & 3;
    const int F = a.F;

    tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1a, 0, 192, tid);
    tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1b, 64, 192, tid);
    tc16::stage_weight<NT_THREADS>(NXhi, NXlo, a.nw1h, 128, 192, tid);
    for (int i = tid; i < F * H; i += NT_THREADS) wts[i] = a.wt[i];
    if (tid < H) {
        bs[tid] = a.bias[tid];
        nxb1s[tid] = a.nxb1[tid];
    }
    if (tid < NT_WARPS * 4) accx_all[tid] = 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    const uint64_t dNXhi = make_desc(smem_u32(NXhi), NT_LBO192, 128), dNXlo = make_desc(smem_u32(NXlo), NT_LBO192, 128);
    XSum xs{a.vsum, a.K, accx_all + 4 * warp, accx_all + 16 * wg, 1u + (uint32_t)wg, t, lane, -1};
    const int ra = 16 * w + (lane >> 2), rb = ra + 8;
    // precondition of every per-graph reduction downstream: ids sorted and inside [0,B) (PyG batches are; the reference
    // takes B from data_batch[-1]+1, FastEGNN.py:298).  Violations are counted for the host and clamped.
    auto graph_of = [&](size_t node) {
        const int64_t gi = a.batch64[node];
        return (int)(gi < 0 ? 0 : (gi >= a.B ? a.B - 1 : gi));
    };

    const int64_t num_tiles = (a.N + NT_TILE - 1) / NT_TILE;
    for (int64_t tile = (int64_t)blockIdx.x * NT_WG + wg; tile < num_tiles; tile += (int64_t)gridDim.x * NT_WG) {
        const int64_t n0 = tile * NT_TILE;
        const int nvalid = (int)min((int64_t)NT_TILE, a.N - n0);
        Rows r;
        r.q = q;
        r.va = ra < nvalid;
        r.vb = rb < nvalid;
        r.na = (size_t)(n0 + (r.va ? ra : 0));
        r.nb = (size_t)(n0 + (r.vb ? rb : 0));
        {   // pull the next tile's inputs towards L2
            const int64_t m0 = n0 + (int64_t)gridDim.x * NT_WG * NT_TILE;
            if (m0 < a.N) {
                const size_t mv = (size_t)min((int64_t)NT_TILE, a.N - m0), m = (size_t)m0;
                prefetch_l2_range(a.feat + m * F, mv * F * 4, t);
                prefetch_l2_range(a.loc + m * 3, mv * 12, t);
                prefetch_l2_range(a.batch64 + m, mv * 8, t);
            }
        }
        const int g_first = graph_of((size_t)n0), g_last = graph_of((size_t)(n0 + nvalid - 1));
        const bool single = g_first == g_last;
        xs.start_tile(g_first, single);

        // per node: graph id (lane 0 of the quad validates and stores it), coordinate q -> x4, Σ(x,1)
        auto node_scalars = [&](bool v, size_t node, int& gr) {
            gr = g_first;
            if (!v) return 0.f;
            gr = graph_of(node);
            if (q == 0) {
                const int64_t gi = a.batch64[node];
                const bool bad = gi < 0 || gi >= a.B || (node > 0 && a.batch64[node - 1] > gi);
                if (bad && a.n_invalid) atomicAdd(a.n_invalid, 1);
                a.batch32[node] = gr;
            }
            const float x = q < 3 ? __ldg(a.loc + node * 3 + q) : 0.f;
            a.x4[node * 4 + q] = x;
            return q < 3 ? x : 1.0f;
        };
        int ga, gb;
        const float xa = node_scalars(r.va, r.na, ga), xb = node_scalars(r.vb, r.nb, gb);
        xs.add(single, r, xa, xb, ga, gb);

        float fa[DISTEGNN_MAX_NODE_FEAT], fb[DISTEGNN_MAX_NODE_FEAT];
#pragma unroll
        for (int k = 0; k < DISTEGNN_MAX_NODE_FEAT; ++k) {
            fa[k] = (r.va && k < F) ? __ldg(a.feat + r.na * F + k) : 0.f;
            fb[k] = (r.vb && k < F) ? __ldg(a.feat + r.nb * F + k) : 0.f;
        }
        uint32_t ahi[16], alo[16];
        float d[32];
        store_h_project(
            [&](int j, f32x2& ya, f32x2& yb) {
                float za[2], zb[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + 2 * q + e;
                    za[e] = zb[e] = bs[col];
#pragma unroll
                    for (int k = 0; k < DISTEGNN_MAX_NODE_FEAT; ++k)
                        if (k < F) {
                            za[e] = fmaf(fa[k], wts[k * H + col], za[e]);
                            zb[e] = fmaf(fb[k], wts[k * H + col], zb[e]);
                        }
                }
                ya = r.va ? pk2(za[0], za[1]) : 0ull;
                yb = r.vb ? pk2(zb[0], zb[1]) : 0ull;
            },
            r, a.h, a.P, a.Q, a.Hn, dNXhi, dNXlo, nxb1s, d, ahi, alo);
    }
    xs.finish();
}

}  // namespace degnn

extern "C" int distegnn_node_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                       const int32_t* rowptr, const int32_t* batch32, const float* h, const float* x4,
                                       const float* node_vel, const float* node_attr, const float* agg_m,
                                       const float* agg_x, const float* agg_v, const float* trans_v,
                                       const float* layer_params, const float* next_layer_params, float* h_out,
                                       float* x4_out, float* P, float* Q, float* Hn, float* node_loc_out, float* vsum,
                                       void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    const bool last = flags & DISTEGNN_FLAG_LAST;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(rowptr && batch32 && h && x4 && node_vel && agg_x && trans_v && layer_params && x4_out && vsum,
                    "null pointer");
    DEGNN_CHECK_ARG(Na == 0 || last || node_attr, "null node_attr with node_attr_nf > 0");
    DEGNN_CHECK_ARG(last || (agg_m && agg_v && next_layer_params && h_out && P && Q && Hn),
                    "null pointer (non-last layer)");
    Layout L = make_layout(A, C, Na);
    NodeTcArgs a;
    a.N = n_nodes; a.B = n_graphs; a.Na = Na; a.K = 4 + 3 * C + H * C; a.flags = flags;
    a.rowptr = rowptr; a.batch = batch32; a.h = h; a.x4 = x4; a.vel = node_vel; a.attr = node_attr;
    a.agg_m = agg_m; a.agg_x = agg_x; a.agg_v = agg_v; a.trans_v = trans_v;
    a.lw = layer_params + L.off[DISTEGNN_P_L_W];
    a.lb = layer_params + L.off[DISTEGNN_P_L_B];
    a.lw3 = layer_params + L.off[DISTEGNN_P_L_W3];
    a.lb3 = layer_params + L.off[DISTEGNN_P_L_B3];
    a.n1 = layer_params + L.off[DISTEGNN_P_N_W1];
    a.nb1 = layer_params + L.off[DISTEGNN_P_N_B1];
    a.n2 = layer_params + L.off[DISTEGNN_P_N_W2];
    a.nb2 = layer_params + L.off[DISTEGNN_P_N_B2];
    const float* nx = next_layer_params ? next_layer_params : layer_params;
    a.nw1a = nx + L.off[DISTEGNN_P_E_W1A];
    a.nxb1 = nx + L.off[DISTEGNN_P_E_B1];
    a.nw1b = nx + L.off[DISTEGNN_P_E_W1B];
    a.nw1h = nx + L.off[DISTEGNN_P_V_W1H];
    a.h_out = h_out; a.x4_out = x4_out; a.P = P; a.Q = Q; a.Hn = Hn; a.loc_out = node_loc_out; a.vsum = vsum;
    ensure_dynamic_smem((const void*)node_layer_tc_kernel, (int)NT_SMEM_BYTES);
    const int64_t tiles = (n_nodes + NT_TILE - 1) / NT_TILE;
    int64_t grid = (tiles + NT_WG - 1) / NT_WG;
    if (grid > sm_count()) grid = sm_count();
    node_layer_tc_kernel<<<(unsigned)grid, NT_THREADS, NT_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_embed_fwd(int64_t n_nodes, int n_graphs, int F, int A, int C, int Na, const float* node_feat,
                                  const float* node_loc, const int64_t* data_batch, const float* emb_wt,
                                  const float* emb_b, const float* layer0_params, float* h, float* x4,
                                  int32_t* batch32, float* P, float* Q, float* Hn, float* vsum, int32_t* n_invalid,
                                  void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(F >= 1 && F <= DISTEGNN_MAX_NODE_FEAT, "node_feat_nf out of range");
    DEGNN_CHECK_ARG(node_feat && node_loc && data_batch && emb_wt && emb_b && layer0_params && h && x4 && batch32 &&
                        P && Q && Hn && vsum, "null pointer");
    Layout L = make_layout(A, C, Na);
    EmbedTcArgs a;
    a.N = n_nodes; a.B = n_graphs; a.F = F; a.K = 4 + 3 * C + H * C;
    a.feat = node_feat; a.loc = node_loc; a.batch64 = data_batch; a.wt = emb_wt; a.bias = emb_b;
    a.nw1a = layer0_params + L.off[DISTEGNN_P_E_W1A];
    a.nxb1 = layer0_params + L.off[DISTEGNN_P_E_B1];
    a.nw1b = layer0_params + L.off[DISTEGNN_P_E_W1B];
    a.nw1h = layer0_params + L.off[DISTEGNN_P_V_W1H];
    a.h = h; a.x4 = x4; a.batch32 = batch32; a.P = P; a.Q = Q; a.Hn = Hn; a.vsum = vsum;
    a.n_invalid = n_invalid;
    ensure_dynamic_smem((const void*)embed_tc_kernel, (int)ET_SMEM_BYTES);
    const int64_t tiles = (n_nodes + NT_TILE - 1) / NT_TILE;
    int64_t grid = (tiles + NT_WG - 1) / NT_WG;
    if (grid > sm_count()) grid = sm_count();
    embed_tc_kernel<<<(unsigned)grid, NT_THREADS, ET_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
