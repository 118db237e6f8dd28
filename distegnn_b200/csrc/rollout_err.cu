// The per-step error of a rollout against recorded targets (distegnn_rollout_sq_err, DESIGN §19):
//   sq_err[t, b] = Σ over the nodes of graph b of Σ_d (pred − targets[t])², t the step on the device counter,
// fp32 differences, fp64 squares and sums (`target_sq_dist`), added by `graph_chunk_sum` (rollout_err.cuh) in an order
// fixed by N and the graph sizes: the same bits in either mode, eager or captured, at any capacity, and on a rerun step.
#include "common.cuh"
#include "rollout_err.cuh"

namespace degnn {

__global__ void __launch_bounds__(DET_RED) rollout_sq_err_kernel(int64_t N, int B, int steps, const float* pred,
                                                                 const float* targets, const int64_t* batch,
                                                                 const int32_t* counter, double* sq_err, double* slots,
                                                                 unsigned* ticket) {
    const int t = __ldcg(counter);             // this step: the advance moves the counter on after this launch
    const bool keep = t >= 0 && t < steps;
    const float* tg = targets + (keep ? (int64_t)t * N * 3 : 0);
    graph_chunk_sum<1>(N, B, batch, keep, sq_err + (keep ? (int64_t)t * B : 0), slots, ticket,
                       [&](int64_t k, double (&s)[1]) {
                           s[0] += target_sq_dist([&](int d) { return __ldg(pred + k * 3 + d); },
                                                  [&](int d) { return __ldg(tg + k * 3 + d); });
                       });
}

// workspace: [slots: one double per chunk | ticket].  The caller zeroes it once; every launch leaves the ticket at 0.
static int64_t sq_err_ticket_at(int64_t N) { return (int64_t)align256((size_t)err_chunks(N) * 8); }
static int64_t sq_err_workspace(int64_t N) { return sq_err_ticket_at(N) + 256; }

}  // namespace degnn

extern "C" {

int distegnn_rollout_sq_err_workspace_bytes(int64_t n_nodes, int64_t* bytes_host) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes_host, "null output pointer");
    DEGNN_CHECK_ARG(n_nodes >= 0, "negative size");
    *bytes_host = sq_err_workspace(n_nodes);
    return DISTEGNN_OK;
}

int distegnn_rollout_sq_err(int64_t n_nodes, int n_graphs, int steps, const float* pred, const float* targets,
                            const int64_t* data_batch, const int32_t* counter, double* sq_err, void* workspace,
                            int64_t workspace_bytes, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0 && steps >= 1, "bad size");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    DEGNN_CHECK_ARG(counter && sq_err, "null pointer");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(pred && targets && workspace, "null pointer");
    DEGNN_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace not 16-byte aligned");
    if (workspace_bytes < sq_err_workspace(n_nodes)) {
        set_error("distegnn_rollout_sq_err: workspace %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)sq_err_workspace(n_nodes));
        return DISTEGNN_EWORKSPACE;
    }
    double* slots = reinterpret_cast<double*>(workspace);
    unsigned* ticket = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(workspace) + sq_err_ticket_at(n_nodes));
    rollout_sq_err_kernel<<<(unsigned)err_chunks(n_nodes), DET_RED, 0, (cudaStream_t)stream>>>(
        n_nodes, n_graphs, steps, pred, targets, data_batch, counter, sq_err, slots, ticket);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

}  // extern "C"
