// Backward of the real<->real edge stage (SURVEY §8 f-1) — fp32 FMA on the CUDA cores: the first, correctness-first
// kernel, now behind distegnn_edge_layer_bwd_simt as the twin of the tensor-core kernel (edge_layer_bwd_tc.cu).
// Differentiates what distegnn_edge_layer_fwd computes (reference models/FastEGNN.py:237-246 coord2radial,
// :144-150 edge_model, :169-177 edge part of coord_model_vel, :206 edge part of node_model, scatter_add_ :322-337;
// in the reference this is autograd through ~20 [E,64] tensors):
//     z1 = P[i] + Q[j] + w_r·r + W_e·a,  a1 = SiLU(z1),  z2 = W2·a1 + b2,  m = SiLU(z2),
//     zc = Wc·m + bc,  φ = w3·SiLU(zc),   agg_m[i] += m,   agg_x[i] += Δ·φ        (i = row, j = col)
// Nothing of size [E,·] is kept from the forward pass: each 128-edge tile is recomputed (2 tile GEMMs), then
//     gφ = g_aggx[i]·Δ,  g_zc = gφ·w3 ⊙ SiLU'(zc),  g_m = g_aggm[i] + Wcᵀ·g_zc,  g_z2 = g_m ⊙ SiLU'(z2),
//     g_z1 = (W2ᵀ·g_z2) ⊙ SiLU'(z1)                                               (2 tile GEMMs)
//     g_P[i] += g_z1,  g_Q[j] += g_z1,  g_r = w_r·g_z1,  gΔ_raw = g_aggx[i]·φ/norm + 2·g_r·Δ_raw,
//     g_x[i] += gΔ_raw,  g_x[j] −= gΔ_raw                                          (norm detached, :243)
// and the weight gradients g_Wc += g_zcᵀ·m, g_W2 += g_z2ᵀ·a1 (2 more tile GEMMs, accumulated in registers over all
// tiles of the CTA), g_b2, g_bc, g_w3, g_w_r, g_W_e (accumulated in shared memory), all added to `g_params`, a
// buffer with the layout of the parameter block (distegnn_param_layout).
#include "bwd_common.cuh"
#include "common.cuh"

namespace degnn {

struct EdgeBwdArgs {
    int64_t N, E;
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
    const float* g_aggm;   // [N,64] gradient w.r.t. the SUM agg_m (null with FLAG_LAST)
    const float* g_aggx;   // [N,4]  gradient w.r.t. the SUM agg_x
    float* g_P;            // [N,64] +=
    float* g_Q;            // [N,64] +=
    float* g_x;            // [N,4]  +=
    float* g_w1r; float* g_w1e; float* g_w2; float* g_b2; float* g_wc; float* g_bc; float* g_w3;   // += (param layout)
};

constexpr int EB_SMEM_FLOATS = 4 * TILE_M * LDA          // Z1, Z2, W (A operand), G (gradient operand)
                               + 4 * H * H               // W2, Wc (k-major) and their transposes
                               + 4 * H + DISTEGNN_MAX_EDGE_ATTR * H          // b2, bc, w3, w1r, w1e
                               + 4 * H + DISTEGNN_MAX_EDGE_ATTR * H          // gradient accumulators of the same
                               + TILE_M * DISTEGNN_MAX_EDGE_ATTR             // edge attrs of the tile
                               + TILE_M * 4              // Δ_raw (xyz) + radial
                               + 5 * TILE_M;             // 1/norm, gφ, φ, g_r, (row, col as int: 2)  -> 6, see below
constexpr size_t EB_SMEM_BYTES = (EB_SMEM_FLOATS + TILE_M) * sizeof(float);

__global__ void __launch_bounds__(NTHREADS, 1) edge_layer_bwd_kernel(const EdgeBwdArgs a) {
    extern __shared__ __align__(16) float smem[];
    float* Z1 = smem;
    float* Z2 = Z1 + TILE_M * LDA;
    float* Wt = Z2 + TILE_M * LDA;          // current A operand: a1, then m, then a1 again
    float* Gt = Wt + TILE_M * LDA;          // current gradient operand: g_zc, then g_z2
    float* W2s = Gt + TILE_M * LDA;
    float* Wcs = W2s + H * H;
    float* W2T = Wcs + H * H;
    float* WcT = W2T + H * H;
    float* b2s = WcT + H * H;
    float* bcs = b2s + H;
    float* w3s = bcs + H;
    float* w1rs = w3s + H;
    float* w1es = w1rs + H;
    float* gb2 = w1es + DISTEGNN_MAX_EDGE_ATTR * H;
    float* gbc = gb2 + H;
    float* gw3 = gbc + H;
    float* gw1r = gw3 + H;
    float* gw1e = gw1r + H;
    float* eas = gw1e + DISTEGNN_MAX_EDGE_ATTR * H;
    float* dxs = eas + TILE_M * DISTEGNN_MAX_EDGE_ATTR;      // Δ_raw xyz, radial
    float* invn = dxs + TILE_M * 4;
    float* gphis = invn + TILE_M;
    float* phis = gphis + TILE_M;
    float* grs = phis + TILE_M;
    int* srow = reinterpret_cast<int*>(grs + TILE_M);
    int* scol = srow + TILE_M;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;
    const int A = a.A;
    const bool normalize = a.flags & DISTEGNN_FLAG_NORMALIZE;
    const bool need_m = !(a.flags & DISTEGNN_FLAG_LAST) && a.g_aggm != nullptr;

    load_w64(W2s, a.w2, tid);
    load_w64(Wcs, a.wc, tid);
    load_w64_t(W2T, a.w2, tid);
    load_w64_t(WcT, a.wc, tid);
    if (tid < H) {
        b2s[tid] = a.b2[tid];
        bcs[tid] = a.bc[tid];
        w3s[tid] = a.w3[tid];
        w1rs[tid] = a.w1r[tid];
    }
    for (int i = tid; i < A * H; i += NTHREADS) w1es[i] = a.w1e[i];
    for (int i = tid; i < 4 * H + DISTEGNN_MAX_EDGE_ATTR * H; i += NTHREADS) gb2[i] = 0.f;
    float gW2[4][4], gWc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) gW2[i][j] = gWc[i][j] = 0.f;
    __syncthreads();

    const float4 b2v = *reinterpret_cast<const float4*>(b2s + 4 * tx);
    const float4 bcv = *reinterpret_cast<const float4*>(bcs + 4 * tx);
    const float4 w3v = *reinterpret_cast<const float4*>(w3s + 4 * tx);
    const float4 wrv = *reinterpret_cast<const float4*>(w1rs + 4 * tx);

    const int64_t num_tiles = (a.E + TILE_M - 1) / TILE_M;
    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int64_t e0 = tile * TILE_M;
        // ---- 1. edge metadata -----------------------------------------------------------------------------------
        if (tid < TILE_M) {
            const int64_t e = e0 + tid;
            const bool ok = e < a.E;
            srow[tid] = ok ? __ldg(a.row + e) : -1;
            scol[tid] = ok ? __ldg(a.col + e) : 0;
        }
        for (int i = tid; i < TILE_M * A; i += NTHREADS) {
            const int64_t g = e0 * A + i;
            eas[i] = (g < a.E * A) ? __ldg(a.ea + g) : 0.f;
        }
        __syncthreads();

        // ---- 2. gather + first layer (half-warp per edge): Z1 = z1, Wt = a1, geometry, gφ ----------------------------
        {
            const int l = lane & 15;
            const float4 wr4 = *reinterpret_cast<const float4*>(w1rs + 4 * l);
#pragma unroll 2
            for (int it = 0; it < 8; ++it) {
                const int el = 16 * warp + 2 * it + (lane >> 4);
                const int r = srow[el];
                float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
                if (r >= 0) {
                    const int c = scol[el];
                    const float4 p = ldg4(a.P + (size_t)r * H + 4 * l);
                    const float4 q = ldg4(a.Q + (size_t)c * H + 4 * l);
                    const float4 xi = ldg4(a.x4 + (size_t)r * 4);
                    const float4 xj = ldg4(a.x4 + (size_t)c * 4);
                    const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
                    const float radial = dx * dx + dy * dy + dz * dz;
                    pre = fma4(radial, wr4, add4(p, q));
                    for (int k = 0; k < A; ++k)
                        pre = fma4(eas[el * A + k], *reinterpret_cast<const float4*>(w1es + k * H + 4 * l), pre);
                    if (l == 0) {
                        const float inv = normalize ? 1.0f / (sqrtf(radial) + 1e-8f) : 1.0f;
                        const float4 gx = ldg4(a.g_aggx + (size_t)r * 4);
                        *reinterpret_cast<float4*>(dxs + 4 * el) = make_float4(dx, dy, dz, radial);
                        invn[el] = inv;
                        gphis[el] = (gx.x * dx + gx.y * dy + gx.z * dz) * inv;
                    }
                } else if (l == 0) {
                    *reinterpret_cast<float4*>(dxs + 4 * el) = make_float4(0.f, 0.f, 0.f, 0.f);
                    invn[el] = 0.f;
                    gphis[el] = 0.f;
                }
                *reinterpret_cast<float4*>(Z1 + el * LDA + 4 * l) = pre;
                *reinterpret_cast<float4*>(Wt + el * LDA + 4 * l) = silu4(pre);
            }
        }
        __syncthreads();

        // ---- 3. z2 = a1·W2 + b2 -> Z2;  Wt = m = SiLU(z2) --------------------------------------------------------
        float acc[8][4];
        zero_acc(acc);
        gemm_tile(acc, Wt, W2s, ty, tx);
        __syncthreads();                       // everyone finished reading a1
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 z = make_float4(acc[i][0] + b2v.x, acc[i][1] + b2v.y, acc[i][2] + b2v.z, acc[i][3] + b2v.w);
            *reinterpret_cast<float4*>(Z2 + (ty + 16 * i) * LDA + 4 * tx) = z;
            *reinterpret_cast<float4*>(Wt + (ty + 16 * i) * LDA + 4 * tx) = silu4(z);
        }
        __syncthreads();

        // ---- 4. zc = m·Wc + bc;  φ;  g_zc = gφ·w3 ⊙ SiLU'(zc) -> Gt;  g_w3, g_bc ---------------------------------------
        zero_acc(acc);
        gemm_tile(acc, Wt, Wcs, ty, tx);
        {
            float gw[4] = {0.f, 0.f, 0.f, 0.f}, gb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = ty + 16 * i;
                const float gp = gphis[e];
                const float zc[4] = {acc[i][0] + bcv.x, acc[i][1] + bcv.y, acc[i][2] + bcv.z, acc[i][3] + bcv.w};
                const float w3a[4] = {w3v.x, w3v.y, w3v.z, w3v.w};
                float ph = 0.f, g[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float s = sigmoid_f(zc[j]);
                    const float ac = zc[j] * s;
                    ph = fmaf(ac, w3a[j], ph);
                    gw[j] = fmaf(gp, ac, gw[j]);
                    g[j] = gp * w3a[j] * (s * fmaf(zc[j], 1.0f - s, 1.0f));
                    gb[j] += g[j];
                }
                ph += __shfl_xor_sync(FULL, ph, 1);
                ph += __shfl_xor_sync(FULL, ph, 2);
                ph += __shfl_xor_sync(FULL, ph, 4);
                ph += __shfl_xor_sync(FULL, ph, 8);
                if (tx == 0) phis[e] = ph;
                *reinterpret_cast<float4*>(Gt + e * LDA + 4 * tx) = make_float4(g[0], g[1], g[2], g[3]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                atomicAdd(gw3 + 4 * tx + j, gw[j]);
                atomicAdd(gbc + 4 * tx + j, gb[j]);
            }
        }
        __syncthreads();

        // ---- 5. g_Wc += g_zcᵀ·m;  g_m = g_zc·Wc + g_aggm[row];  g_z2 = g_m ⊙ SiLU'(z2) ------------------------------
        wgrad_tile(gWc, Gt, Wt, tid);
        zero_acc(acc);
        gemm_tile(acc, Gt, WcT, ty, tx);
        __syncthreads();                       // Gt and Wt fully read
        {
            float gb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = ty + 16 * i;
                const int r = srow[e];
                float4 gm = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
                if (need_m && r >= 0) gm = add4(gm, ldg4(a.g_aggm + (size_t)r * H + 4 * tx));
                const float4 z = *reinterpret_cast<const float4*>(Z2 + e * LDA + 4 * tx);
                const float4 g = make_float4(gm.x * dsilu(z.x), gm.y * dsilu(z.y), gm.z * dsilu(z.z), gm.w * dsilu(z.w));
                gb[0] += g.x; gb[1] += g.y; gb[2] += g.z; gb[3] += g.w;
                *reinterpret_cast<float4*>(Gt + e * LDA + 4 * tx) = g;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) atomicAdd(gb2 + 4 * tx + j, gb[j]);
        }
        silu_tile(Wt, Z1, tid);                // Wt = a1 again
        __syncthreads();

        // ---- 6. g_W2 += g_z2ᵀ·a1;  g_z1 = (g_z2·W2) ⊙ SiLU'(z1) -> g_P, g_Q, g_w_r, g_W_e, g_r ------------------------
        wgrad_tile(gW2, Gt, Wt, tid);
        zero_acc(acc);
        gemm_tile(acc, Gt, W2T, ty, tx);
        {
            float gwr[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = ty + 16 * i;
                const int r = srow[e];
                const float4 z = *reinterpret_cast<const float4*>(Z1 + e * LDA + 4 * tx);
                const float4 g = make_float4(acc[i][0] * dsilu(z.x), acc[i][1] * dsilu(z.y), acc[i][2] * dsilu(z.z),
                                             acc[i][3] * dsilu(z.w));
                float gr = g.x * wrv.x + g.y * wrv.y + g.z * wrv.z + g.w * wrv.w;
                gr += __shfl_xor_sync(FULL, gr, 1);
                gr += __shfl_xor_sync(FULL, gr, 2);
                gr += __shfl_xor_sync(FULL, gr, 4);
                gr += __shfl_xor_sync(FULL, gr, 8);
                if (tx == 0) grs[e] = gr;
                if (r >= 0) {
                    red_add_v4(a.g_P + (size_t)r * H + 4 * tx, g);
                    red_add_v4(a.g_Q + (size_t)scol[e] * H + 4 * tx, g);
                    const float rad = dxs[4 * e + 3];
                    gwr[0] = fmaf(g.x, rad, gwr[0]); gwr[1] = fmaf(g.y, rad, gwr[1]);
                    gwr[2] = fmaf(g.z, rad, gwr[2]); gwr[3] = fmaf(g.w, rad, gwr[3]);
                    for (int k = 0; k < A; ++k) {
                        const float ev = eas[e * A + k];
                        atomicAdd(gw1e + k * H + 4 * tx + 0, g.x * ev);
                        atomicAdd(gw1e + k * H + 4 * tx + 1, g.y * ev);
                        atomicAdd(gw1e + k * H + 4 * tx + 2, g.z * ev);
                        atomicAdd(gw1e + k * H + 4 * tx + 3, g.w * ev);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) atomicAdd(gw1r + 4 * tx + j, gwr[j]);
        }
        __syncthreads();

        // ---- 7. geometry: gΔ_raw = g_aggx[i]·φ/norm + 2·g_r·Δ_raw (none for a self loop: +gΔ − gΔ on one node) ---------
        if (tid < TILE_M) {
            const int r = srow[tid], c = scol[tid];
            if (r >= 0 && r != c) {
                const float4 d = *reinterpret_cast<const float4*>(dxs + 4 * tid);
                const float4 gx = ldg4(a.g_aggx + (size_t)r * 4);
                const float s = phis[tid] * invn[tid], t2 = 2.0f * grs[tid];
                const float gdx = fmaf(gx.x, s, t2 * d.x), gdy = fmaf(gx.y, s, t2 * d.y), gdz = fmaf(gx.z, s, t2 * d.z);
                atomicAdd(a.g_x + (size_t)r * 4 + 0, gdx);
                atomicAdd(a.g_x + (size_t)r * 4 + 1, gdy);
                atomicAdd(a.g_x + (size_t)r * 4 + 2, gdz);
                atomicAdd(a.g_x + (size_t)c * 4 + 0, -gdx);
                atomicAdd(a.g_x + (size_t)c * 4 + 1, -gdy);
                atomicAdd(a.g_x + (size_t)c * 4 + 2, -gdz);
            }
        }
        __syncthreads();                       // tile buffers are rewritten by the next iteration
    }

    // ---- flush the CTA's parameter gradients ------------------------------------------------------------------------
    wgrad_flush(a.g_w2, gW2, tid);
    wgrad_flush(a.g_wc, gWc, tid);
    if (tid < H) {
        atomicAdd(a.g_b2 + tid, gb2[tid]);
        atomicAdd(a.g_bc + tid, gbc[tid]);
        atomicAdd(a.g_w3 + tid, gw3[tid]);
        atomicAdd(a.g_w1r + tid, gw1r[tid]);
    }
    for (int i = tid; i < A * H; i += NTHREADS) atomicAdd(a.g_w1e + i, gw1e[i]);
}

}  // namespace degnn

extern "C" int distegnn_edge_layer_bwd_simt(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                       const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                       const float* x4, const float* P, const float* Q, const float* layer_params,
                                       const float* g_agg_m, const float* g_agg_x, float* g_P, float* g_Q, float* g_x4,
                                       float* g_layer_params, void* stream) {
    using namespace degnn;
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_edges == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_edges > 0, "negative size");
    DEGNN_CHECK_ARG(row && col && x4 && P && Q && layer_params && g_agg_x && g_P && g_Q && g_x4 && g_layer_params,
                    "null pointer");
    DEGNN_CHECK_ARG(A == 0 || edge_attr_sorted, "null edge_attr with edge_attr_nf > 0");
    Layout L = make_layout(A, C, Na);
    EdgeBwdArgs a;
    a.N = n_nodes; a.E = n_edges; a.A = A; a.flags = flags;
    a.row = row; a.col = col; a.ea = edge_attr_sorted; a.x4 = x4; a.P = P; a.Q = Q;
    a.w1r = layer_params + L.off[DISTEGNN_P_E_W1R];
    a.w1e = layer_params + L.off[DISTEGNN_P_E_W1E];
    a.w2 = layer_params + L.off[DISTEGNN_P_E_W2];
    a.b2 = layer_params + L.off[DISTEGNN_P_E_B2];
    a.wc = layer_params + L.off[DISTEGNN_P_E_WC];
    a.bc = layer_params + L.off[DISTEGNN_P_E_BC];
    a.w3 = layer_params + L.off[DISTEGNN_P_E_W3];
    a.g_aggm = g_agg_m; a.g_aggx = g_agg_x; a.g_P = g_P; a.g_Q = g_Q; a.g_x = g_x4;
    a.g_w1r = g_layer_params + L.off[DISTEGNN_P_E_W1R];
    a.g_w1e = g_layer_params + L.off[DISTEGNN_P_E_W1E];
    a.g_w2 = g_layer_params + L.off[DISTEGNN_P_E_W2];
    a.g_b2 = g_layer_params + L.off[DISTEGNN_P_E_B2];
    a.g_wc = g_layer_params + L.off[DISTEGNN_P_E_WC];
    a.g_bc = g_layer_params + L.off[DISTEGNN_P_E_BC];
    a.g_w3 = g_layer_params + L.off[DISTEGNN_P_E_W3];
    ensure_dynamic_smem((const void*)edge_layer_bwd_kernel, (int)EB_SMEM_BYTES);
    const int64_t tiles = (n_edges + TILE_M - 1) / TILE_M;
    int64_t grid = sm_count();
    if (grid > tiles) grid = tiles;
    edge_layer_bwd_kernel<<<(unsigned)grid, NTHREADS, EB_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
