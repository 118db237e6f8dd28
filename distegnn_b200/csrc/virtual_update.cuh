// Arguments of the virtual-node update fused with the cross-partition SUM all-reduce (virtual_update.cu), and their
// checks.  Shared by the product entry point distegnn_virtual_update_fwd (one CTA per graph) and the testing library's
// W-rank twin (testing/comm_ranks.cu, one CTA per graph and rank); the update itself is virtual_update_graph.cuh.
#pragma once
#include "comm.cuh"
#include "common.cuh"

namespace degnn {

struct VUpdArgs {
    int B, C, K;
    unsigned flags;
    float* vsum;
    float* Xv;   // [B,3,C]
    float* Hv;   // [B,C,64]
    const float* m1; const float* mb1; const float* m2; const float* mb2;   // node_mlp_virtual
    const float* nv1v; const float* nv1m; const float* nvb1;                 // next layer's W1v_V, W1v_M, b1v
    float* G;    // [B,C,64]
    const float* init_loc_mean;   // [B,3]   (FLAG_INIT: Xv := loc_mean broadcast over channels, FastEGNN.py:300)
    const float* init_hv0;        // [C,64]  (FLAG_INIT: Hv := virtual_node_feat, FastEGNN.py:299)
};

constexpr int VU_KMAX = 4 + 3 * DISTEGNN_MAX_CHANNELS + H * DISTEGNN_MAX_CHANNELS;
constexpr int VU_THREADS = 512;          // one (channel, column) output per thread at C = 8: the kernel is pure latency

// Argument checks of distegnn_virtual_update_fwd past check_dims and n_graphs == 0, and the arguments of the update from
// the parameter layout.  Errors name `who`.
inline int virtual_update_args(const char* who, int n_graphs, int A, int C, int Na, unsigned flags, float* vsum, float* Xv,
                               float* Hv, const float* layer_params, const float* next_layer_params, float* G,
                               const float* init_loc_mean, const float* init_hv0, VUpdArgs* out) {
#define VU_CHECK_ARG(cond, msg)                     \
    do {                                            \
        if (!(cond)) {                              \
            ::degnn::set_error("%s: %s", who, msg); \
            return DISTEGNN_EINVAL;                 \
        }                                           \
    } while (0)
    const bool last = flags & DISTEGNN_FLAG_LAST, init = flags & DISTEGNN_FLAG_INIT;
    VU_CHECK_ARG(n_graphs > 0, "bad size");
    VU_CHECK_ARG(vsum && Xv, "null pointer");
    VU_CHECK_ARG(last || (Hv && next_layer_params && G), "null pointer (non-last)");
    VU_CHECK_ARG(last || init || layer_params, "null layer_params");
    VU_CHECK_ARG(init || (!init_loc_mean && !init_hv0), "init_loc_mean / init_hv0 need FLAG_INIT");
    VU_CHECK_ARG(!(flags & DISTEGNN_FLAG_INIT_CENTROID) || (init && !init_loc_mean),
                 "FLAG_INIT_CENTROID needs FLAG_INIT and no init_loc_mean");
#undef VU_CHECK_ARG
    Layout L = make_layout(A, C, Na);
    VUpdArgs& a = *out;
    a.B = n_graphs; a.C = C; a.K = 4 + 3 * C + H * C; a.flags = flags;
    a.vsum = vsum; a.Xv = Xv; a.Hv = Hv;
    const float* lp = layer_params ? layer_params : next_layer_params;
    a.m1 = lp ? lp + L.off[DISTEGNN_P_M_W1] : nullptr;
    a.mb1 = lp ? lp + L.off[DISTEGNN_P_M_B1] : nullptr;
    a.m2 = lp ? lp + L.off[DISTEGNN_P_M_W2] : nullptr;
    a.mb2 = lp ? lp + L.off[DISTEGNN_P_M_B2] : nullptr;
    a.nv1v = next_layer_params ? next_layer_params + L.off[DISTEGNN_P_V_W1V] : nullptr;
    a.nv1m = next_layer_params ? next_layer_params + L.off[DISTEGNN_P_V_W1M] : nullptr;
    a.nvb1 = next_layer_params ? next_layer_params + L.off[DISTEGNN_P_V_B1] : nullptr;
    a.G = G;
    a.init_loc_mean = init_loc_mean; a.init_hv0 = init_hv0;
    return DISTEGNN_OK;
}

}  // namespace degnn
