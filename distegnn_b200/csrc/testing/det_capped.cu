// Grid-capped twins of the deterministic mode's entry points (include/distegnn_b200_testing_det.h).  The kernels are the
// production ones: build.py links edge_layer_cs, virtual_layer_tc16 and deterministic into this library too.
#include "../../../include/distegnn_b200_testing_det.h"
#include "common.cuh"
#include "det.cuh"

extern "C" {

int distegnn_edge_layer_fwd_det_capped(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                       const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                       const float* x4, const float* P, const float* Q, const float* layer_params,
                                       float* agg_m, float* agg_x, const int32_t* n_edges_dev, void* workspace,
                                       int64_t workspace_bytes, void* stream, int max_ctas) {
    using namespace degnn;
    DEGNN_CHECK_ARG(max_ctas >= 0, "negative grid cap");
    return edge_layer_fwd_det(n_nodes, n_edges, A, C, Na, flags, row, col, edge_attr_sorted, x4, P, Q, layer_params,
                              agg_m, agg_x, n_edges_dev, workspace, workspace_bytes, stream, max_ctas);
}

int distegnn_edge_combine_det_capped(int64_t n_nodes, int64_t n_edges, int C, const int32_t* row,
                                     const int32_t* n_edges_dev, float* agg_m, float* agg_x, void* workspace,
                                     int64_t workspace_bytes, void* stream, int max_ctas) {
    using namespace degnn;
    DEGNN_CHECK_ARG(max_ctas >= 0, "negative grid cap");
    return edge_combine_det(n_nodes, n_edges, C, row, n_edges_dev, agg_m, agg_x, workspace, workspace_bytes, stream,
                            max_ctas);
}

int distegnn_virtual_layer_fwd_det_capped(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                          const int32_t* batch32, const float* x4, const float* Hn, const float* Xv,
                                          const float* G, const float* layer_params, float* agg_v, float* trans_v,
                                          float* vsum, void* workspace, int64_t workspace_bytes, void* stream,
                                          int max_ctas) {
    using namespace degnn;
    DEGNN_CHECK_ARG(max_ctas >= 0, "negative grid cap");
    return virtual_layer_fwd_det(n_nodes, n_graphs, A, C, Na, flags, batch32, x4, Hn, Xv, G, layer_params, agg_v,
                                 trans_v, vsum, workspace, workspace_bytes, stream, max_ctas);
}

int distegnn_vsum_combine_det_capped(int64_t n_nodes, int n_graphs, int C, unsigned flags, const int32_t* batch32,
                                     const float* x4, float* vsum, void* workspace, int64_t workspace_bytes,
                                     void* stream, int max_ctas) {
    using namespace degnn;
    DEGNN_CHECK_ARG(max_ctas >= 0, "negative grid cap");
    return vsum_combine_det(n_nodes, n_graphs, C, flags, batch32, x4, vsum, workspace, workspace_bytes, stream,
                            max_ctas);
}

}  // extern "C"
