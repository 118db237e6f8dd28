// The <true> instantiation of the edge-stage backward kernel (gradient w.r.t. edge_attr as well), in a translation unit of
// its own so that the weights-only kernel in edge_layer_bwd_tc.cu compiles exactly as without it.
#include "edge_layer_bwd_tc.cuh"

namespace degnn {

void launch_edge_layer_bwd_tc_inputs(const EdgeBwdTcArgs& a, unsigned grid, cudaStream_t stream) {
    ensure_dynamic_smem((const void*)edge_layer_bwd_tc_kernel<true>, (int)BT_SMEM_BYTES);
    edge_layer_bwd_tc_kernel<true><<<grid, BT_THREADS, BT_SMEM_BYTES, stream>>>(a);
}

}  // namespace degnn
