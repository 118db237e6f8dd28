// Multi-step rollout: the per-step state update on the device (distegnn_b200/rollout.py).
//
// A rollout feeds the model's prediction back in as the next step's input, restating the reference's data pipeline on
// predicted positions (datasets/process_dataset.py:345, vel = pos[f+1] − pos[f]; the |v| node feature of :107, :190, :346,
// :505).  Per step, after graph build and forward:
//   distegnn_rollout_advance   v ← (x' − x)/tau, feat[:, speed_col] ← ‖v‖, x ← x', trajectory[step] ← x', n_edges[step],
//                              sticky overflow flag of the graph build — one launch, the step index lives on the device so
//                              the same launch replays from a CUDA graph
//   distegnn_edge_lengths_csr  fixed-graph mode (N-body, fully connected): edge_attr ← ‖x_row − x_col‖ in every column
// and once at the end
//   distegnn_rollout_centroid  per-graph Σx and node count in fp64 (the caller all-reduces over the partitions and
//                              divides).
// The backward of a differentiable rollout adds, per step in reverse:
//   distegnn_rollout_advance_bwd  the advance's gradient: upstream of the step's prediction and the −g_v/tau part of x_t
//   distegnn_edge_lengths_bwd     g_edge_attr (CSR order) -> positions
#include "common.cuh"

namespace degnn {

struct AdvanceArgs {
    int64_t N;
    int F, speed_col, steps;
    float tau;
    const float* pred;          // [N,3] the forward's output x_{t+1}
    float* loc;                 // [N,3] state x_t, overwritten with x_{t+1}
    float* vel;                 // [N,3]
    float* feat;                // [N,F] (speed column written) or null
    float* traj;                // [steps,N,3] or null
    const int32_t* edge_count;  // [1] edges of this step's graph
    const int32_t* overflow;    // [1] nonzero if this step's graph build overflowed, or null
    int32_t* n_edges;           // [steps]
    int32_t* counter;           // [8] see include/distegnn_b200.h
};

__global__ void __launch_bounds__(256) rollout_advance_kernel(const AdvanceArgs a) {
    // every block reads the step before the last block to finish advances it (ticket in counter[4])
    const int step = __ldcg(a.counter);
    const bool keep = step >= 0 && step < a.steps;
    const float inv_tau = 1.0f / a.tau;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.N; i += (int64_t)gridDim.x * blockDim.x) {
        float x[3], v[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            x[d] = __ldg(a.pred + i * 3 + d);
            v[d] = (x[d] - a.loc[i * 3 + d]) * inv_tau;
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            a.vel[i * 3 + d] = v[d];
            a.loc[i * 3 + d] = x[d];
            if (a.traj && keep) a.traj[((int64_t)step * a.N + i) * 3 + d] = x[d];
        }
        if (a.feat) a.feat[i * a.F + a.speed_col] = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const int e = __ldcg(a.edge_count);
        if (keep) a.n_edges[step] = e;
        if (a.overflow && __ldcg(a.overflow) && a.counter[1] == 0) {
            a.counter[1] = 1;
            a.counter[2] = step;
        }
        a.counter[3] = max(a.counter[3], e);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(a.counter + 4), 1u);
        if (t == gridDim.x - 1) {
            a.counter[4] = 0;
            a.counter[0] = step + 1;
            __threadfence();
        }
    }
}

__global__ void __launch_bounds__(256) edge_lengths_kernel(int64_t E, int A, const int32_t* row, const int32_t* col,
                                                           const float* pos, const int32_t* n_edges_dev, float* ea) {
    const int64_t nE = n_edges_dev ? min((int64_t)__ldg(n_edges_dev), E) : E;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nE; e += (int64_t)gridDim.x * blockDim.x) {
        const int i = __ldg(row + e), j = __ldg(col + e);
        float ddx, ddy, ddz;
        edge_delta(pos, i, j, ddx, ddy, ddz);
        const float dd = sqrtf(edge_len2(ddx, ddy, ddz));
        for (int c = 0; c < A; ++c) ea[e * A + c] = dd;
    }
}

// fp64 accumulation: the count stays exact and Σx carries no fp32 rounding at millions of nodes per graph
__global__ void __launch_bounds__(256) centroid_kernel(int64_t N, int B, const float* pos, const int64_t* batch,
                                                       double* sums) {
    const int lane = threadIdx.x & 31;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < N; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const bool ok = i < N;
        const int b = ok ? graph_id(batch, i, B) : 0;
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        if (ok) {
            s[0] = __ldg(pos + i * 3); s[1] = __ldg(pos + i * 3 + 1); s[2] = __ldg(pos + i * 3 + 2); s[3] = 1.0;
        }
        // whole warp in one graph (the common case: batches are sorted): one atomic per component and warp
        const int b0 = __shfl_sync(FULL, b, 0);
        if (__all_sync(FULL, !ok || b == b0)) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(FULL, s[k], o);
            if (lane == 0)
                for (int k = 0; k < 4; ++k) atomicAdd(sums + b0 * 4 + k, s[k]);
        } else if (ok) {
            for (int k = 0; k < 4; ++k) atomicAdd(sums + b * 4 + k, s[k]);
        }
    }
}

// ---- backward of a differentiable rollout (distegnn_b200/rollout.py: differentiable_rollout) -------------------------------
// d‖x_i − x_j‖ / dx_i = u = (x_i − x_j)/‖x_i − x_j‖, and −u for x_j.  One thread per edge; the row side is a segmented
// warp sum over the CSR runs (rows are sorted) with one RED per run, the col side one RED per edge.  A zero-length edge
// (self loop, coincident points) contributes exactly 0, like torch's norm backward.
__global__ void __launch_bounds__(256) edge_lengths_bwd_kernel(int64_t E, int A, const int32_t* row, const int32_t* col,
                                                               const float* pos, const int32_t* n_edges_dev,
                                                               const float* g_ea, float* g_pos) {
    const int64_t nE = n_edges_dev ? min((int64_t)__ldg(n_edges_dev), E) : E;
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < nE; base += n_warps * 32) {
        const int64_t e = base + lane;
        int i = -1;
        float c[3] = {0.f, 0.f, 0.f};
        if (e < nE) {
            i = __ldg(row + e);
            const int j = __ldg(col + e);
            float ddx, ddy, ddz;
            edge_delta(pos, i, j, ddx, ddy, ddz);
            const float dd = sqrtf(edge_len2(ddx, ddy, ddz));
            if (dd > 0.f) {
                float g = 0.f;
                for (int k = 0; k < A; ++k) g += __ldg(g_ea + e * A + k);
                const float s = g / dd;
                c[0] = s * ddx; c[1] = s * ddy; c[2] = s * ddz;
                if (s != 0.f) {
#pragma unroll
                    for (int d = 0; d < 3; ++d) atomicAdd(g_pos + (int64_t)j * 3 + d, -c[d]);
                }
            }
        }
        // suffix sums within runs of equal row: lane k ends up with the sum of its run from k on
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int io = __shfl_down_sync(FULL, i, o);
            float co[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) co[d] = __shfl_down_sync(FULL, c[d], o);
            if (lane + o < 32 && io == i) {
#pragma unroll
                for (int d = 0; d < 3; ++d) c[d] += co[d];
            }
        }
        const int prev = __shfl_up_sync(FULL, i, 1);
        if (i >= 0 && (lane == 0 || prev != i) && (c[0] != 0.f || c[1] != 0.f || c[2] != 0.f)) {
#pragma unroll
            for (int d = 0; d < 3; ++d) atomicAdd(g_pos + (int64_t)i * 3 + d, c[d]);
        }
    }
}

// v = (x' − x)·(1/tau) with the forward's arithmetic; g_v = g_v' + g_speed·v/‖v‖ (0 at v = 0);
// g_pred = g_traj + g_x' + g_v/tau;  g_x = −g_v/tau;  g_feat'[:, speed_col] is consumed (set to 0).
__global__ void __launch_bounds__(256) rollout_advance_bwd_kernel(int64_t N, int F, int speed_col, float tau,
                                                                  const float* x_next, const float* x,
                                                                  const float* g_traj, const float* g_x_next,
                                                                  const float* g_v_next, float* g_feat_next,
                                                                  float* g_pred, float* g_x) {
    const float inv_tau = 1.0f / tau;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        float v[3], gv[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            v[d] = (__ldg(x_next + i * 3 + d) - __ldg(x + i * 3 + d)) * inv_tau;
            gv[d] = g_v_next ? __ldg(g_v_next + i * 3 + d) : 0.f;
        }
        if (g_feat_next) {
            const float gs = g_feat_next[i * F + speed_col];
            g_feat_next[i * F + speed_col] = 0.f;
            const float s = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            if (s > 0.f) {
#pragma unroll
                for (int d = 0; d < 3; ++d) gv[d] += gs * (v[d] / s);
            }
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float a = gv[d] * inv_tau;
            float p = a;
            if (g_traj) p += __ldg(g_traj + i * 3 + d);
            if (g_x_next) p += __ldg(g_x_next + i * 3 + d);
            g_pred[i * 3 + d] = p;
            g_x[i * 3 + d] = -a;
        }
    }
}

static unsigned grid_for(int64_t n) {
    const int64_t cap = 4 * (int64_t)sm_count();
    const int64_t g = (n + 255) / 256;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace degnn

extern "C" int distegnn_rollout_advance(int64_t n_nodes, int F, int speed_col, float tau, int steps, const float* pred,
                                        float* loc, float* vel, float* feat, float* trajectory,
                                        const int32_t* edge_count, const int32_t* overflow, int32_t* n_edges,
                                        int32_t* counter, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && steps >= 1, "bad size");
    DEGNN_CHECK_ARG(tau > 0.f, "tau must be > 0");
    DEGNN_CHECK_ARG(pred && loc && vel && edge_count && n_edges && counter, "null pointer");
    DEGNN_CHECK_ARG(!feat || (speed_col >= 0 && speed_col < F), "speed_col outside [0, F)");
    AdvanceArgs a;
    a.N = n_nodes; a.F = F; a.speed_col = speed_col; a.steps = steps; a.tau = tau;
    a.pred = pred; a.loc = loc; a.vel = vel; a.feat = feat; a.traj = trajectory;
    a.edge_count = edge_count; a.overflow = overflow; a.n_edges = n_edges; a.counter = counter;
    rollout_advance_kernel<<<grid_for(n_nodes), 256, 0, (cudaStream_t)stream>>>(a);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_edge_lengths_csr(int64_t n_edges, int edge_attr_nf, const int32_t* row, const int32_t* col,
                                         const float* pos, const int32_t* n_edges_dev, float* edge_attr, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_edges >= 0 && edge_attr_nf >= 0 && edge_attr_nf <= DISTEGNN_MAX_EDGE_ATTR, "bad size");
    if (n_edges == 0 || edge_attr_nf == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(row && col && pos && edge_attr, "null pointer");
    edge_lengths_kernel<<<grid_for(n_edges), 256, 0, (cudaStream_t)stream>>>(n_edges, edge_attr_nf, row, col, pos,
                                                                              n_edges_dev, edge_attr);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_edge_lengths_bwd(int64_t n_edges, int edge_attr_nf, const int32_t* row, const int32_t* col,
                                         const float* pos, const int32_t* n_edges_dev, const float* g_edge_attr,
                                         float* g_pos, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_edges >= 0 && edge_attr_nf >= 0 && edge_attr_nf <= DISTEGNN_MAX_EDGE_ATTR, "bad size");
    if (n_edges == 0 || edge_attr_nf == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(row && col && pos && g_edge_attr && g_pos, "null pointer");
    edge_lengths_bwd_kernel<<<grid_for(n_edges), 256, 0, (cudaStream_t)stream>>>(n_edges, edge_attr_nf, row, col, pos,
                                                                                  n_edges_dev, g_edge_attr, g_pos);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_rollout_advance_bwd(int64_t n_nodes, int F, int speed_col, float tau, const float* x_next,
                                            const float* x, const float* g_traj, const float* g_x_next,
                                            const float* g_v_next, float* g_feat_next, float* g_pred, float* g_x,
                                            void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0, "bad size");
    DEGNN_CHECK_ARG(tau > 0.f, "tau must be > 0");
    DEGNN_CHECK_ARG(!g_feat_next || (speed_col >= 0 && speed_col < F), "speed_col outside [0, F)");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(x_next && x && g_pred && g_x, "null pointer");
    rollout_advance_bwd_kernel<<<grid_for(n_nodes), 256, 0, (cudaStream_t)stream>>>(
        n_nodes, F, speed_col, tau, x_next, x, g_traj, g_x_next, g_v_next, g_feat_next, g_pred, g_x);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_rollout_centroid(int64_t n_nodes, int n_graphs, const float* pos, const int64_t* data_batch,
                                         double* sums, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_nodes >= 0 && n_graphs > 0, "bad size");
    DEGNN_CHECK_ARG(n_graphs == 1 || data_batch, "data_batch needed for more than one graph");
    if (n_nodes == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(pos && sums, "null pointer");
    centroid_kernel<<<grid_for(n_nodes), 256, 0, (cudaStream_t)stream>>>(n_nodes, n_graphs, pos, data_batch, sums);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
