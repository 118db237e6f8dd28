// Backward of the real<->real edge stage on the tensor cores (wgmma) — production kernel behind
// distegnn_edge_layer_bwd.  Its twin, the fp32-FMA kernel of csrc/testing/edge_layer_bwd.cu behind
// distegnn_edge_layer_bwd_simt, has the same contract and math (reference: autograd through models/FastEGNN.py:144-150,
// 169-177, 206, 237-246, 322-337); what changes is where the six tile GEMMs of a 128-edge tile run:
//   * the four ROW-WISE GEMMs (recompute z2 = a1·W2ᵀ, zc = m·Wcᵀ; data gradients g_m = g_zc·Wc, g_a1 = g_z2·W2) run as
//     wgmma f16 with the fp16 2-term split of both operands (tc16.cuh), A written to tile memory by the thread that owns
//     the row, B (W and Wᵀ, hi/lo) resident in shared memory, D read back row-per-thread;
//   * the two WEIGHT-GRADIENT GEMMs (g_Wc += g_zcᵀ·m, g_W2 += g_z2ᵀ·a1; contraction over the 128 edges) stay on the CUDA
//     cores for now: they need the operands edge-major ("MN-major"), which the K-major machinery of the forward kernels
//     does not provide; they read the two fp32 row tiles the row threads leave in shared memory.
// One CTA per SM, 128 threads = 1 warpgroup; thread r owns edge r of the tile end to end and holds a whole 64-wide row in
// registers.  Tile memory (tile_mma.cuh, 128 columns): A_hi 32 | A_lo 32 | z2 64, and D overwrites the A operand it was
// computed from (every D row is read into registers before its thread writes the next A).  z2 is parked in tile memory
// between the forward recompute and the SiLU' factors of the backward chain; z1 is recomputed from P, Q and the edge
// geometry where it is needed again.
// Gradient rows span many orders of magnitude, so EVERY row is encoded with its own power-of-two scale (row maximum
// taken from the registers), not only the rows that would overflow; D rows are multiplied by 1/scale on the way out.
// The row rules (encoding, row-tile GEMM, φ-head backward, column sums, weight gradients) live in bwd_tc_common.cuh.
// Edge order: g_P is summed over runs of equal destination row, so the edges of a row must be contiguous; the rows may
// come in any order (the cached graph's spatial order, DESIGN §3).
#include "edge_layer_bwd_tc.cuh"

namespace degnn {

void launch_edge_layer_bwd_tc_inputs(const EdgeBwdTcArgs& a, unsigned grid, cudaStream_t stream);   // _inputs.cu

static int edge_layer_bwd_launch(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                 const int32_t* row, const int32_t* col, const float* edge_attr_sorted, const float* x4,
                                 const float* P, const float* Q, const float* layer_params, const float* g_agg_m,
                                 const float* g_agg_x, float* g_P, float* g_Q, float* g_x4, float* g_layer_params,
                                 const int32_t* n_edges_dev, float* g_edge_attr_sorted, void* stream) {
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_edges == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(n_nodes > 0 && n_edges > 0, "negative size");
    DEGNN_CHECK_ARG(row && col && x4 && P && Q && layer_params && g_agg_x && g_P && g_Q && g_x4 && g_layer_params,
                    "null pointer");
    DEGNN_CHECK_ARG(A == 0 || edge_attr_sorted, "null edge_attr with edge_attr_nf > 0");
    Layout L = make_layout(A, C, Na);
    EdgeBwdTcArgs a;
    a.N = n_nodes; a.E = n_edges; a.E_dev = n_edges_dev; a.A = A; a.flags = flags;
    a.row = row; a.col = col; a.ea = edge_attr_sorted; a.x4 = x4; a.P = P; a.Q = Q;
    a.w1r = layer_params + L.off[DISTEGNN_P_E_W1R];
    a.w1e = layer_params + L.off[DISTEGNN_P_E_W1E];
    a.w2 = layer_params + L.off[DISTEGNN_P_E_W2];
    a.b2 = layer_params + L.off[DISTEGNN_P_E_B2];
    a.wc = layer_params + L.off[DISTEGNN_P_E_WC];
    a.bc = layer_params + L.off[DISTEGNN_P_E_BC];
    a.w3 = layer_params + L.off[DISTEGNN_P_E_W3];
    a.g_aggm = g_agg_m; a.g_aggx = g_agg_x; a.g_P = g_P; a.g_Q = g_Q; a.g_x = g_x4; a.g_ea = g_edge_attr_sorted;
    a.g_w1r = g_layer_params + L.off[DISTEGNN_P_E_W1R];
    a.g_w1e = g_layer_params + L.off[DISTEGNN_P_E_W1E];
    a.g_w2 = g_layer_params + L.off[DISTEGNN_P_E_W2];
    a.g_b2 = g_layer_params + L.off[DISTEGNN_P_E_B2];
    a.g_wc = g_layer_params + L.off[DISTEGNN_P_E_WC];
    a.g_bc = g_layer_params + L.off[DISTEGNN_P_E_BC];
    a.g_w3 = g_layer_params + L.off[DISTEGNN_P_E_W3];
    int64_t grid = (n_edges + TILE_M - 1) / TILE_M;
    if (grid > sm_count()) grid = sm_count();
    if (g_edge_attr_sorted != nullptr && A > 0) {
        launch_edge_layer_bwd_tc_inputs(a, (unsigned)grid, (cudaStream_t)stream);
    } else {
        ensure_dynamic_smem((const void*)edge_layer_bwd_tc_kernel<false>, (int)BT_SMEM_BYTES);
        edge_layer_bwd_tc_kernel<false><<<(unsigned)grid, BT_THREADS, BT_SMEM_BYTES, (cudaStream_t)stream>>>(a);
    }
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" int distegnn_edge_layer_bwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                       const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                       const float* x4, const float* P, const float* Q, const float* layer_params,
                                       const float* g_agg_m, const float* g_agg_x, float* g_P, float* g_Q, float* g_x4,
                                       float* g_layer_params, const int32_t* n_edges_dev, void* stream) {
    return degnn::edge_layer_bwd_launch(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q,
                                        layer_params, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_layer_params, n_edges_dev,
                                        nullptr, stream);
}

extern "C" int distegnn_edge_layer_bwd_inputs(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                              const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                              const float* x4, const float* P, const float* Q, const float* layer_params,
                                              const float* g_agg_m, const float* g_agg_x, float* g_P, float* g_Q,
                                              float* g_x4, float* g_layer_params, const int32_t* n_edges_dev,
                                              float* g_edge_attr_sorted, void* stream) {
    return degnn::edge_layer_bwd_launch(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q,
                                        layer_params, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_layer_params, n_edges_dev,
                                        g_edge_attr_sorted, stream);
}
