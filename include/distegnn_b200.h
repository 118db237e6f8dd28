/*
 * distegnn_b200.h — C ABI of libdistegnn_b200.so: the sm_100a implementation of the DistEGNN hot
 * path (FastEGNN per-layer equivariant message passing + the packed virtual-node statistics that are
 * all-reduced across graph partitions).
 *
 * The reference (GLAD-RUC/DistEGNN) is pure Python/PyTorch and has no FFI of its own; the entry
 * points below are what a binding for this path has to expose.  Each one cites the reference code it
 * replaces (paths relative to the reference repo root).  The only caller in this repo is
 * distegnn_b200/fast_egnn.py (ctypes); INTEGRATION.md shows the stub a maintainer of the reference
 * would add.
 *
 * Conventions
 *   - every function returns 0 on success or a negative DISTEGNN_E* code; distegnn_last_error()
 *     returns a thread-local human-readable message for the last failure;
 *   - all pointers are DEVICE pointers unless the name ends in _host; the caller owns every buffer
 *     (inputs, outputs, workspaces); the library never allocates, frees or synchronises — the one
 *     exception is the communicator (distegnn_comm_init / _destroy), which owns its peer-mapped segment;
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*); the call returns as soon as
 *     the work is enqueued; it is safe inside CUDA-graph capture;
 *   - fp32 everywhere, node ids int32 after distegnn_build_csr (int64 at the reference boundary);
 *   - hidden width H is fixed at 64 (every shipped config: config/ *.yaml `hidden_nf: 64`);
 *   - preconditions the kernels rely on and the host mirror validates (fast_egnn.py): data_batch is
 *     non-decreasing with ids in [0, n_graphs) (FastEGNN.py:298 takes B from data_batch[-1]+1 and PyG batches are
 *     sorted); edge ids lie in [0, n_nodes) (distegnn_build_csr returns DISTEGNN_EINVAL otherwise);
 *   - cross-check twins of these entry points (fp32 FMA on the CUDA cores) live in
 *     distegnn_b200_testing.h / libdistegnn_b200_testing.so and are not part of the product.
 *
 * Internal data layout (all row-major, contiguous)
 *   h      [N,64]   node features                x4     [N,4]  coordinates (xyz, w unused)
 *   P,Q    [N,64]   first edge-MLP layer split per node: P = W1[:, 0:64]·h + b1, Q = W1[:,64:128]·h
 *   Hn     [N,64]   first virtual-MLP layer node part:  W1v[:, 0:64]·h
 *   Xv     [B,3,C]  virtual coordinates (reference layout)
 *   Hv     [B,C,64] virtual features (reference layout is [B,64,C]; transposed once on the host)
 *   G      [B,C,64] per-graph/channel constant of the first virtual-MLP layer:
 *                   W1v[:,64:128]·Hv[b,:,c] + W1v[:,129:129+C]·m_X[b,:,c] + b1v
 *   vsum   [B,K]    packed per-graph partial sums that are all-reduced (SUM) once per layer,
 *                   K = 4 + 3C + 64C:  [0:3] Σ_i x_i   [3] node count   [4 : 4+3C] Σ_i ΔX_ic·φ_X as
 *                   [3][C]   [4+3C : K] Σ_i mv_ic as [C][64]
 */
#ifndef DISTEGNN_B200_H
#define DISTEGNN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DISTEGNN_ABI_VERSION 3

#if defined(__GNUC__)
#define DISTEGNN_API __attribute__((visibility("default")))
#else
#define DISTEGNN_API
#endif

enum {
    DISTEGNN_OK = 0,
    DISTEGNN_EINVAL = -1,   /* bad argument (null pointer, unsupported size)              */
    DISTEGNN_ECUDA = -2,    /* a CUDA runtime call or kernel launch failed                 */
    DISTEGNN_EWORKSPACE = -3 /* caller-provided workspace too small                        */
};

/* limits of the compiled kernels */
#define DISTEGNN_HIDDEN 64
#define DISTEGNN_MAX_CHANNELS 16   /* virtual_channels C            */
#define DISTEGNN_MAX_EDGE_ATTR 8   /* edge_attr_nf A                */
#define DISTEGNN_MAX_NODE_ATTR 8   /* node_attr_nf Na               */
#define DISTEGNN_MAX_NODE_FEAT 16  /* node_feat_nf F                */

/* flags */
#define DISTEGNN_FLAG_NORMALIZE 1u  /* E_GCL_vel(normalize=True), FastEGNN.py:242-244                  */
#define DISTEGNN_FLAG_LAST 2u       /* last layer: h'/Hv' are dead (FastEGNN.py:307) — skip them        */
#define DISTEGNN_FLAG_INIT 4u       /* virtual_update before layer 0: no X / Hv update, only x̄, m_X, G */
#define DISTEGNN_FLAG_ZERO_VSUM 8u  /* virtual_update: leave vsum zeroed (ready for the next layer's accumulation)  */
#define DISTEGNN_FLAG_ZERO_AGG 16u  /* node_layer: leave agg_m / agg_x zeroed (ready for the next edge stage)       */
#define DISTEGNN_FLAG_INIT_CENTROID 32u /* virtual_update with FLAG_INIT: X_0 := the summed x̄ (inference / rollout only) */

DISTEGNN_API int distegnn_abi_version(void);
DISTEGNN_API const char *distegnn_last_error(void);

/* ---- per-layer parameter block -------------------------------------------------------------------
 * One flat fp32 buffer per E_GCL_vel layer; every matrix is stored k-major ([in][out], i.e. the
 * transpose of nn.Linear.weight) so a thread reads 4 consecutive outputs with one 16-byte load.
 * Field order / source tensors (state_dict keys under gcl_<i>., SURVEY §8b):
 */
enum {
    DISTEGNN_P_E_W1A = 0,  /* [64][64]  edge_mlp.0.weight[:, 0:64]^T   (h[row])            FastEGNN.py:69-74 */
    DISTEGNN_P_E_W1B,      /* [64][64]  edge_mlp.0.weight[:, 64:128]^T (h[col])                              */
    DISTEGNN_P_E_W1R,      /* [64]      edge_mlp.0.weight[:, 128]      (radial)                              */
    DISTEGNN_P_E_W1E,      /* [A][64]   edge_mlp.0.weight[:, 129:129+A]^T (edge_attr)                        */
    DISTEGNN_P_E_B1,       /* [64]      edge_mlp.0.bias                                                      */
    DISTEGNN_P_E_W2,       /* [64][64]  edge_mlp.2.weight^T                                                  */
    DISTEGNN_P_E_B2,       /* [64]                                                                            */
    DISTEGNN_P_E_WC,       /* [64][64]  coord_mlp_r.0.weight^T                                 :96-110       */
    DISTEGNN_P_E_BC,       /* [64]                                                                            */
    DISTEGNN_P_E_W3,       /* [64]      coord_mlp_r.2.weight[0]                                               */
    DISTEGNN_P_V_W1H,      /* [64][64]  edge_mlp_virtual.0.weight[:, 0:64]^T (h)                :76-81        */
    DISTEGNN_P_V_W1V,      /* [64][64]  edge_mlp_virtual.0.weight[:, 64:128]^T (Hv)                           */
    DISTEGNN_P_V_W1R,      /* [64]      edge_mlp_virtual.0.weight[:, 128] (‖ΔX‖)                              */
    DISTEGNN_P_V_W1M,      /* [C][64]   edge_mlp_virtual.0.weight[:, 129:129+C]^T (m_X)                       */
    DISTEGNN_P_V_B1,       /* [64]                                                                            */
    DISTEGNN_P_V_W2,       /* [64][64]  edge_mlp_virtual.2.weight^T                                           */
    DISTEGNN_P_V_B2,       /* [64]                                                                            */
    DISTEGNN_P_V_WXV,      /* [64][64]  coord_mlp_r_virtual.0.weight^T                          :111          */
    DISTEGNN_P_V_BXV,      /* [64]                                                                            */
    DISTEGNN_P_V_W3XV,     /* [64]      coord_mlp_r_virtual.2.weight[0]                                       */
    DISTEGNN_P_V_WX,       /* [64][64]  coord_mlp_v_virtual.0.weight^T                          :112          */
    DISTEGNN_P_V_BX,       /* [64]                                                                            */
    DISTEGNN_P_V_W3X,      /* [64]      coord_mlp_v_virtual.2.weight[0]                                       */
    DISTEGNN_P_L_W,        /* [64][64]  coord_mlp_vel.0.weight^T                                :115-119      */
    DISTEGNN_P_L_B,        /* [64]                                                                            */
    DISTEGNN_P_L_W3,       /* [64]      coord_mlp_vel.2.weight[0]                                             */
    DISTEGNN_P_L_B3,       /* [4]       coord_mlp_vel.2.bias (1 value, padded)                                */
    DISTEGNN_P_N_W1,       /* [192+Na][64] node_mlp.0.weight^T  (h | agg | agg_v | node_attr)   :130-135      */
    DISTEGNN_P_N_B1,       /* [64]                                                                            */
    DISTEGNN_P_N_W2,       /* [64][64]  node_mlp.2.weight^T                                                   */
    DISTEGNN_P_N_B2,       /* [64]                                                                            */
    DISTEGNN_P_M_W1,       /* [128][64] node_mlp_virtual.0.weight^T (Hv | agg)                  :137-141      */
    DISTEGNN_P_M_B1,       /* [64]                                                                            */
    DISTEGNN_P_M_W2,       /* [64][64]  node_mlp_virtual.2.weight^T                                           */
    DISTEGNN_P_M_B2,       /* [64]                                                                            */
    DISTEGNN_P_NUM_FIELDS
};

/* Fills offsets_host[DISTEGNN_P_NUM_FIELDS] (in floats, each a multiple of 4) and *total_floats for a
 * layer with edge_attr_nf=A, virtual_channels=C, node_attr_nf=Na.  Host-only, no CUDA call. */
DISTEGNN_API int distegnn_param_layout(int A, int C, int Na, int64_t *offsets_host, int64_t *total_floats_host);

/* ---- graph preprocessing (cached per edge_index by the caller) -----------------------------------
 * Replaces the implicit "scatter by edge_index[0]" of unsorted_segment_sum/mean
 * (models/FastEGNN.py:322-337, twins models/basic.py:50-66): the COO list [2,E] int64 (row =
 * edge_index[0] = aggregation destination, col = edge_index[1] = neighbour; FastEGNN.py:238,250) is
 * stably sorted by row into int32 CSR.  perm[e'] = original position of sorted edge e' (to permute
 * edge_attr).  Self loops, duplicate edges and isolated nodes are legal (equivariant_test.py:26-27).
 * Ids outside [0, n_nodes) — on which the reference dies with a device-side index assert — are counted into the device
 * counter *n_invalid (may be NULL) and clamped, so that nothing indexes out of bounds; the caller reads the counter once
 * per graph (the build is cached) and raises.
 */
DISTEGNN_API int distegnn_csr_workspace_bytes(int64_t n_nodes, int64_t n_edges, int64_t *bytes_host);
DISTEGNN_API int distegnn_build_csr(const int64_t *edge_index, int64_t n_nodes, int64_t n_edges,
                       int32_t *rowptr /*[N+1]*/, int32_t *row /*[E]*/, int32_t *col /*[E]*/,
                       int32_t *perm /*[E]*/, void *workspace, int64_t workspace_bytes,
                       int32_t *n_invalid /*[1], device, may be NULL*/, void *stream);

/* dst[i,:] = src[perm[i],:] for i < n_rows, rows of `width` floats (edge_attr into CSR order). */
DISTEGNN_API int distegnn_gather_rows(const float *src, const int32_t *perm, int64_t n_rows, int width, float *dst,
                         void *stream);

/* The inverse of distegnn_gather_rows: dst[perm[i],:] = src[i,:] for i < n_rows (gradients w.r.t. edge_attr in CSR order
 * back into the caller's edge order).  perm must be a permutation of [0, n_rows). */
DISTEGNN_API int distegnn_scatter_rows(const float *src, const int32_t *perm, int64_t n_rows, int width, float *dst,
                                       void *stream);

/* ---- embedding + per-forward setup ---------------------------------------------------------------
 * FastEGNN.forward prologue (FastEGNN.py:298-302): h0 = embedding_in(node_feat); also converts
 * node_loc [N,3] → x4, data_batch int64 → batch32, computes P/Q/Hn of layer 0 from `layer0_params`,
 * and accumulates Σx and the node count of every graph into vsum[:,0:4] (caller zeroes vsum).
 * emb_wt is embedding_in.weight^T [F][64], emb_b [64].
 * data_batch must be non-decreasing with ids in [0, n_graphs): the per-graph reductions of every later stage rely on
 * it.  Violations are counted into the device counter *n_invalid (may be NULL; the caller zeroes it) and the ids clamped.
 */
DISTEGNN_API int distegnn_embed_fwd(int64_t n_nodes, int n_graphs, int F, int A, int C, int Na,
                       const float *node_feat, const float *node_loc, const int64_t *data_batch,
                       const float *emb_wt, const float *emb_b, const float *layer0_params,
                       float *h, float *x4, int32_t *batch32, float *P, float *Q, float *Hn,
                       float *vsum, int32_t *n_invalid, void *stream);

/* ---- real↔real edge stage ------------------------------------------------------------------------
 * coord2radial + edge_model + the edge part of coord_model_vel + the edge part of node_model
 * (FastEGNN.py:237-246, 144-150, 169-177, 206): for every CSR edge (i=row, j=col)
 *   Δx = x_i − x_j, r = ‖Δx‖² (Δx /= sqrt(r)+1e-8 if NORMALIZE)
 *   m  = SiLU(W2·SiLU(P_i + Q_j + w_r·r + W_e·a_ij) + b2),  φ = w3·SiLU(Wc·m + bc)
 *   agg_m[i] += m   (skipped with FLAG_LAST),   agg_x[i].xyz += Δx·φ
 * Sums, not means: the division by max(deg,1) happens in distegnn_node_layer_fwd.  The caller zeroes
 * agg_m [N,64] and agg_x [N,4] before the call.  For graphs built on the device without a host round trip
 * (distegnn_radius_graph_csr with a capacity) n_edges is the CAPACITY of row/col/edge_attr and n_edges_dev points to the
 * true count, which the kernel reads itself.
 */
DISTEGNN_API int distegnn_edge_layer_fwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                            const int32_t *row, const int32_t *col, const float *edge_attr_sorted,
                            const float *x4, const float *P, const float *Q,
                            const float *layer_params, float *agg_m, float *agg_x,
                            const int32_t *n_edges_dev /*NULL, or the edge count on the device (<= n_edges)*/,
                            void *stream);

/* Backward of distegnn_edge_layer_fwd (SURVEY §8 f-1; in the reference: autograd through models/FastEGNN.py:144-150,
 * 169-177, 206, 237-246, 322-337).  Nothing of size [E,.] is kept from the forward pass: every 128-edge tile is
 * recomputed.  Inputs: the forward inputs plus g_agg_m [N,64] (gradient w.r.t. the SUM agg_m; may be NULL with
 * FLAG_LAST) and g_agg_x [N,4] (w.r.t. the SUM agg_x).  Outputs are ACCUMULATED (+=): g_P, g_Q [N,64], g_x4 [N,4]
 * (both edge endpoints; the normalisation norm is detached as in :243) and g_layer_params, a buffer with the layout
 * of the parameter block (fields E_W1R, E_W1E, E_W2, E_B2, E_WC, E_BC, E_W3 are written). */
DISTEGNN_API int distegnn_edge_layer_bwd(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                         const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                         const float* x4, const float* P, const float* Q, const float* layer_params,
                                         const float* g_agg_m, const float* g_agg_x, float* g_P, float* g_Q,
                                         float* g_x4, float* g_layer_params, const int32_t* n_edges_dev, void* stream);
/* distegnn_edge_layer_bwd plus the gradient w.r.t. the edge attributes (model input edge_attr, in CSR order):
 * g_edge_attr_sorted [E,A] is ACCUMULATED (+=), so one buffer collects every layer.  NULL (or A = 0) is exactly
 * distegnn_edge_layer_bwd. */
DISTEGNN_API int distegnn_edge_layer_bwd_inputs(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                                const int32_t* row, const int32_t* col, const float* edge_attr_sorted,
                                                const float* x4, const float* P, const float* Q, const float* layer_params,
                                                const float* g_agg_m, const float* g_agg_x, float* g_P, float* g_Q,
                                                float* g_x4, float* g_layer_params, const int32_t* n_edges_dev,
                                                float* g_edge_attr_sorted, void* stream);

/* Backward of distegnn_virtual_layer_fwd (SURVEY §8 f-1; in the reference: autograd through models/FastEGNN.py:154-163,
 * 180, 191-193, 207, 220-223, 252-253).  Rows are recomputed tile by tile; the six row-wise tile GEMMs run on the tensor cores (wgmma).
 * `weight_images` (96 KB, device): the stage's three 64x64 matrices and their transposes as fp16 hi/lo images in the
 * shared-memory operand layout, written by distegnn_virtual_bwd_prepare(layer_params) — once per layer and call; the
 * kernel streams them through shared memory with TMA.  Upstream gradients: g_agg_v [N,64] (NULL with FLAG_LAST), g_trans_v
 * [N,4], g_vsum [B,K] (entries [4:] are read; already summed over the partitions).  g_Hn [N,64] and g_xv [N,4] are WRITTEN;
 * g_G [B,C,64], g_Xv [B,3,C] and the parameter gradients (V_W1R, V_W2, V_B2, V_WXV, V_BXV, V_W3XV, V_WX, V_BX, V_W3X of a
 * parameter-layout buffer) are accumulated. */
DISTEGNN_API int distegnn_virtual_bwd_prepare(int A, int C, int Na, const float* layer_params, void* weight_images,
                                              void* stream);
DISTEGNN_API int distegnn_virtual_layer_bwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                            const int32_t* batch32, const float* x4, const float* Hn, const float* Xv,
                                            const float* G, const float* layer_params, const void* weight_images,
                                            const float* g_agg_v, const float* g_trans_v, const float* g_vsum,
                                            float* g_Hn, float* g_xv, float* g_G, float* g_Xv, float* g_layer_params,
                                            void* stream);

/* On-device radius graph, CSR out, in ONE call and without a host round trip (csrc/radius_csr.cu; SURVEY §8 f-2): the
 * reference-boundary tensors in (pos [N,3] fp32, data_batch int64 [N] sorted, may be NULL for one graph), int32 CSR by
 * destination out (rowptr [N+1], row / col [capacity]) plus edge_attr [capacity, edge_attr_nf] = the edge length in every
 * column (datasets/distribute_graphs.py:43-44).  Pairs with |x_i - x_j| < radius (strict, as torch_cluster), j != i unless
 * `loop`, same graph only.  Bounding box, grid sizing (cell >= radius*(1 + 2^-10), grown until graphs x cells + 1 <=
 * table_cells; needs n_graphs + 1 <= table_cells), cell keys, sort, counts and prefix sums all happen on the device;
 * info [4] (device): [0] edges found, [1] 1 if that exceeds `capacity` (then only rowptr is complete), [2] cells used.
 * capacity = 0 runs the count only (row/col may be NULL).  Any position is accepted: a node with an inf or NaN
 * coordinate gets no edges, the others their normal ones. */
DISTEGNN_API int distegnn_radius_csr_workspace_bytes(int64_t n_nodes, int64_t table_cells, int64_t *bytes_host);
DISTEGNN_API int distegnn_radius_graph_csr(int64_t n_nodes, int n_graphs, const float *pos, const int64_t *data_batch,
                                           float radius, int loop, int edge_attr_nf, int64_t capacity,
                                           int64_t table_cells, int32_t *rowptr, int32_t *row, int32_t *col,
                                           float *edge_attr, int32_t *info, void *workspace, int64_t workspace_bytes,
                                           void *stream);

/* Lloyd iterations of the k-means node partitioner (datasets/distribute_graphs.py:118-143, 188-198: sklearn KMeans on the
 * host) with sklearn's stopping rules evaluated on the device: `iters` iterations are enqueued; once no label changes, or
 * the squared centre shift is <= tol (then after one more assignment pass), the remaining ones are no-ops.  centers [K,3]
 * in/out (seeded by the caller, k-means++), labels int32 [N] in/out (−1 initially), sums float64 [K,4] zeroed once by the
 * caller, state int32 [4] zeroed once: [0] 0 running / 1 final pass pending / 2 converged, [1] iterations done. */
/* ---- multi-step rollout (csrc/rollout.cu; distegnn_b200/rollout.py) ----------------------------------------------------
 * distegnn_rollout_advance: one step's state update after the forward, in one launch, no host synchronisation:
 *   v = (pred − loc)/tau -> vel [N,3];  ‖v‖ -> feat[:, speed_col] (feat [N,F], NULL = no speed feature);  pred -> loc;
 *   pred -> trajectory[step] ([steps,N,3], NULL = not kept);  *edge_count -> n_edges[step] (int32 [steps]).
 * counter int32 [8], zeroed by the caller except [2] = −1: [0] step (read by every block, advanced by one per launch, so
 * the same launch can be replayed from a CUDA graph), [1] sticky: 1 once *overflow was nonzero (overflow may be NULL),
 * [2] first step that overflowed, [3] largest *edge_count seen, [4] internal (block ticket; keep 0).
 * distegnn_edge_lengths_csr: edge_attr[e, :] = ‖pos[row[e]] − pos[col[e]]‖ for e < min(*n_edges_dev, n_edges) (NULL: all),
 * with the arithmetic of distegnn_radius_graph_csr's fill pass (fixed-graph rollouts).
 * distegnn_rollout_centroid: sums [n_graphs,4] fp64 += (Σx, Σy, Σz, count) per graph (data_batch int64, NULL for one
 * graph); fp64, so the count is exact and Σx keeps full precision at any graph size. */
DISTEGNN_API int distegnn_rollout_advance(int64_t n_nodes, int F, int speed_col, float tau, int steps, const float *pred,
                                          float *loc, float *vel, float *feat, float *trajectory,
                                          const int32_t *edge_count, const int32_t *overflow, int32_t *n_edges,
                                          int32_t *counter, void *stream);
DISTEGNN_API int distegnn_edge_lengths_csr(int64_t n_edges, int edge_attr_nf, const int32_t *row, const int32_t *col,
                                           const float *pos, const int32_t *n_edges_dev, float *edge_attr, void *stream);
DISTEGNN_API int distegnn_rollout_centroid(int64_t n_nodes, int n_graphs, const float *pos, const int64_t *data_batch,
                                           double *sums, void *stream);
/* Backward of a differentiable rollout (differentiable_rollout), one step at a time in reverse.  Caller-owned buffers,
 * nothing allocated, no host synchronisation; negative error codes like every entry point.
 * distegnn_edge_lengths_bwd: backward of distegnn_edge_lengths_csr (and of the radius fill pass's edge_attr).  For
 *   e < min(*n_edges_dev, n_edges) (n_edges_dev NULL: all): g = Σ_k g_edge_attr[e,k], u = Δx/‖Δx‖ with Δx = pos[row[e]] −
 *   pos[col[e]] computed as in the forward; g_pos[row[e]] += g·u, g_pos[col[e]] −= g·u (accumulated; g_pos [N,3]).  A
 *   zero-length edge (self loop, coincident points) contributes exactly 0.  Rows must be sorted (CSR); edges at and
 *   beyond the count are never read.
 * distegnn_rollout_advance_bwd: backward of distegnn_rollout_advance for one step.  Recomputes v = (x_next − x)/tau with
 *   the forward's arithmetic, then g_v = g_v_next + g_feat_next[:, speed_col]·v/‖v‖ (0 at v = 0; g_feat_next NULL = no
 *   speed feature, else that column is set to 0 after it is read), writes g_pred = g_traj + g_x_next + g_v/tau (the
 *   upstream of the step's model output) and g_x = −g_v/tau.  g_traj, g_x_next, g_v_next may be NULL (zero). */
DISTEGNN_API int distegnn_edge_lengths_bwd(int64_t n_edges, int edge_attr_nf, const int32_t *row, const int32_t *col,
                                           const float *pos, const int32_t *n_edges_dev, const float *g_edge_attr,
                                           float *g_pos, void *stream);
DISTEGNN_API int distegnn_rollout_advance_bwd(int64_t n_nodes, int F, int speed_col, float tau, const float *x_next,
                                              const float *x, const float *g_traj, const float *g_x_next,
                                              const float *g_v_next, float *g_feat_next, float *g_pred, float *g_x,
                                              void *stream);

/* ---- edge cutoff (csrc/cutoff_csr.cu; FastEGNN's cutoff_edges mode, datasets/process_dataset.py:300-305) --------------
 * Keeps the shortest edges of every graph of a CSR graph, on the device, without a host round trip.  Candidates: the edges
 * of the input CSR (rowptr_in [N+1], row_in / col_in [capacity]) below *n_edges_in (NULL: rowptr_in[N]), never past
 * `capacity`; graph b's candidates are the CSR range of its nodes (data_batch int64 [N] sorted, NULL for one graph).  Per
 * graph, k_b = floor((double)E_b * (1.0 - cutoff_rate)) in fp64 (= Python's int(E * (1 - cutoff_rate))) and the kept set
 * is the k_b smallest candidates by (fp32 length with the fill pass's arithmetic, CSR position): a stable selection, NaN
 * last.  Output: a sub-sequence of the candidates in CSR order (row_out / col_out [capacity]), edge_attr_out
 * [capacity, edge_attr_nf] = the length in every column, rowptr_out [N+1] = kept candidates before rowptr_in[i].
 * info [4] (device): [0] kept edges (the output's n_edges_dev), [1] 1 if the candidate build overflowed (count above
 * `capacity`, or *overflow_in nonzero; overflow_in may be NULL) — the output is then not valid, but nothing past the
 * capacity is read, [2] candidate count, [3] 0.  cutoff_rate in [0, 1].  Deterministic bit for bit, capturable. */
DISTEGNN_API int distegnn_cutoff_csr_workspace_bytes(int64_t n_nodes, int n_graphs, int64_t capacity, int64_t *bytes_host);
DISTEGNN_API int distegnn_cutoff_csr(int64_t n_nodes, int n_graphs, const float *pos, const int64_t *data_batch,
                                     double cutoff_rate, int edge_attr_nf, const int32_t *rowptr_in, const int32_t *row_in,
                                     const int32_t *col_in, const int32_t *n_edges_in, int64_t capacity,
                                     const int32_t *overflow_in, int32_t *rowptr_out, int32_t *row_out, int32_t *col_out,
                                     float *edge_attr_out, int32_t *info, void *workspace, int64_t workspace_bytes,
                                     void *stream);

DISTEGNN_API int distegnn_kmeans_lloyd(int64_t n_nodes, int n_clusters, const float *pos, float *centers,
                                       int32_t *labels, double *sums, int32_t *state, float tol, int iters, void *stream);

/* ---- real↔virtual stage --------------------------------------------------------------------------
 * Virtual geometry + edge_mode_virtual + the virtual parts of coord_model_vel, coord_model_virtual,
 * node_model and node_model_virtual (FastEGNN.py:252-253, 154-163, 180, 191-193, 207, 220-223):
 * for every node i (graph b) and channel c
 *   ΔX = Xv[b,:,c] − x_i,  mv = SiLU(W2v·SiLU(Hn_i + G[b,c] + w_vr·‖ΔX‖) + b2v)
 *   trans_v[i] = mean_c(−ΔX·φ_xv(mv)),  agg_v[i] = mean_c mv                       (per node)
 *   vsum[b, 4:4+3C] += ΔX·φ_X(mv),      vsum[b, 4+3C:] += mv                       (per graph)
 * With FLAG_LAST agg_v and the Σmv block are skipped.  Caller zeroes vsum.
 */
DISTEGNN_API int distegnn_virtual_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                               const int32_t *batch32, const float *x4, const float *Hn,
                               const float *Xv, const float *G, const float *layer_params,
                               float *agg_v, float *trans_v /*[N,4]*/, float *vsum, void *stream);

/* ---- node update ---------------------------------------------------------------------------------
 * The rest of coord_model_vel and node_model (FastEGNN.py:177-183, 203-217):
 *   x' = x + agg_x/max(deg,1) + trans_v + φ_v(h)·v
 *   h' = h + W2n·SiLU(W1n·[h; agg_m/max(deg,1); agg_v; node_attr] + b1n) + b2n
 * plus P/Q/Hn of the NEXT layer from next_layer_params, and vsum[b,0:4] += (x', 1).
 * With FLAG_LAST only x' is produced and additionally written as [N,3] to node_loc_out (the model
 * output); h_out/P/Q/Hn/next_layer_params may be null.  h_out may alias h, x4_out may alias x4.
 * With FLAG_ZERO_AGG the kernel clears agg_m and agg_x after consuming them (they are written although declared
 * const), so the caller needs no memset before the next edge stage.
 */
DISTEGNN_API int distegnn_node_layer_fwd(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                            const int32_t *rowptr, const int32_t *batch32, const float *h,
                            const float *x4, const float *node_vel, const float *node_attr,
                            const float *agg_m, const float *agg_x, const float *agg_v,
                            const float *trans_v, const float *layer_params,
                            const float *next_layer_params, float *h_out, float *x4_out, float *P,
                            float *Q, float *Hn, float *node_loc_out, float *vsum, void *stream);

/* Backward of distegnn_node_layer_fwd and of the embedding prologue (SURVEY §8 f-1; in the reference: autograd through
 * models/FastEGNN.py:177-183, 203-217, 302) — fp32 FMA tile GEMMs, everything recomputed from N-sized tensors.
 * Upstream: g_x_out [N,3] (w.r.t. x'), g_vsum [B,K] (optional; its [b,0:3] entries add to g_x' of the nodes of graph b —
 * x' feeds the next layer's Σ x'), g_h_out / g_P / g_Q / g_Hn [N,64] (w.r.t. h' and the next layer's projections; NULL with
 * FLAG_LAST).  WRITTEN: g_h [N,64], g_x [N,3], g_agg_x / g_trans_v [N,4], g_agg_m / g_agg_v [N,64] (not with FLAG_LAST).
 * ACCUMULATED: fields L_W, L_B, L_W3, L_B3, N_W1, N_B1, N_W2, N_B2 of g_layer_params and E_W1A, E_B1, E_W1B, V_W1H of
 * g_next_layer_params (parameter-layout buffers).  distegnn_embed_bwd: h0 = the forward's h of layer 0; accumulates
 * g_emb_wt [F][64], g_emb_b [64] and the same four projection fields of layer 0's gradient block. */
DISTEGNN_API int distegnn_node_layer_bwd(int64_t n_nodes, int A, int C, int Na, unsigned flags, const int32_t *rowptr,
                                         const float *h, const float *node_vel, const float *node_attr,
                                         const float *agg_m, const float *agg_v, const float *layer_params,
                                         const float *next_layer_params, const float *g_x_out, const float *g_vsum,
                                         const int32_t *batch32, const float *g_h_out, const float *g_P, const float *g_Q,
                                         const float *g_Hn, float *g_h, float *g_x, float *g_agg_x, float *g_trans_v,
                                         float *g_agg_m, float *g_agg_v, float *g_layer_params,
                                         float *g_next_layer_params, void *stream);
DISTEGNN_API int distegnn_embed_bwd(int64_t n_nodes, int F, int A, int C, int Na, const float *node_feat, const float *h0,
                                    const float *layer0_params, const float *g_h, const float *g_P, const float *g_Q,
                                    const float *g_Hn, float *g_emb_wt, float *g_emb_b, float *g_layer0_params,
                                    void *stream);
/* The same two backward passes plus the gradients w.r.t. the model inputs.  distegnn_node_layer_bwd_inputs ACCUMULATES
 * (+=) g_node_vel [N,3] (φ_v·g_x') and g_node_attr [N,Na] (the attr rows of N_W1; no term with FLAG_LAST), so one buffer
 * each collects every layer; either may be NULL.  distegnn_embed_bwd_inputs WRITES g_node_feat [N,F] = g_h0·emb_wtᵀ
 * (emb_wt [F][64] as in distegnn_embed_fwd) and g_node_loc [N,3] = g_x0 + g_vsum0[batch32[i], 0:3], where g_x0 [N,3] is
 * the gradient w.r.t. layer 0's coordinates and g_vsum0 [B,K] (may be NULL) the gradient of the initial statistics
 * (Σx of the initial centroid; already summed over the partitions); either output may be NULL.  With all extra outputs
 * NULL both are exactly their plain counterparts. */
DISTEGNN_API int distegnn_node_layer_bwd_inputs(int64_t n_nodes, int A, int C, int Na, unsigned flags,
                                                const int32_t *rowptr, const float *h, const float *node_vel,
                                                const float *node_attr, const float *agg_m, const float *agg_v,
                                                const float *layer_params, const float *next_layer_params,
                                                const float *g_x_out, const float *g_vsum, const int32_t *batch32,
                                                const float *g_h_out, const float *g_P, const float *g_Q,
                                                const float *g_Hn, float *g_h, float *g_x, float *g_agg_x,
                                                float *g_trans_v, float *g_agg_m, float *g_agg_v, float *g_layer_params,
                                                float *g_next_layer_params, float *g_node_vel, float *g_node_attr,
                                                void *stream);
DISTEGNN_API int distegnn_embed_bwd_inputs(int64_t n_nodes, int F, int A, int C, int Na, const float *node_feat,
                                           const float *h0, const float *layer0_params, const float *g_h,
                                           const float *g_P, const float *g_Q, const float *g_Hn, float *g_emb_wt,
                                           float *g_emb_b, float *g_layer0_params, const float *emb_wt,
                                           const int32_t *batch32, const float *g_x0, const float *g_vsum0,
                                           float *g_node_feat, float *g_node_loc, void *stream);

/* ---- virtual-node sync: packed SUM all-reduce over NVLink peer memory ------------------------------------------------
 * Replaces weighted_average_reduce / _AllReduce (models/FastEGNN.py:10-43, 310-319; call sites :195-197, 225-227,
 * 259-261 — six NCCL calls behind host syncs per layer) with ONE exchange of the packed statistics vsum [B,K] per layer.
 * One process per GPU; every rank owns a segment of device memory that all peers map through CUDA IPC.  A call pushes the
 * rank's values into every peer's segment, raises a per-slot flag, waits for the peers' flags and sums the `world`
 * contributions in RANK ORDER, so the result is bit-identical on all ranks (the property the reference relies on NCCL
 * for, FastEGNN.py:29-31) and independent of arrival order.  No host synchronisation, safe under CUDA-graph capture (the
 * per-slot epoch lives in device memory).  All ranks must issue the same sequence of calls with the same sizes.
 *
 *   distegnn_comm_init     allocate + clear this rank's segment for calls of at most max_slots x slot_floats floats (for
 *                          the model: max_slots >= B graphs, slot_floats >= K); returns the opaque communicator and this
 *                          rank's IPC handle (distegnn_comm_handle_bytes() bytes, host memory).  Synchronises the device.
 *   (caller)               all-gathers the handles over any host transport (the mirror uses torch.distributed)
 *   distegnn_comm_connect  all_handles_host = world handles in rank order; maps the peers' segments
 *   distegnn_allreduce_packed  in-place SUM of buf[0:count] over the ranks, enqueued on `stream`
 *   distegnn_comm_status   *status_host != 0 if a wait timed out (a peer never arrived; default 10 s, see _set_timeout_ms)
 *   distegnn_comm_disconnect  unmap the peers' segments (own segment stays: peers may still map it)
 *   distegnn_comm_destroy  unmap + free.  Teardown across ranks: no calls in flight -> every rank disconnects -> host
 *                          barrier -> every rank destroys (an exported allocation must outlive its importers' mappings)
 * The fused form — all-reduce of vsum[b,:] followed by the virtual-node update in the same kernel — is
 * distegnn_virtual_update_fwd with a non-null `comm`.
 */
DISTEGNN_API int distegnn_comm_handle_bytes(void);
DISTEGNN_API int distegnn_comm_init(int rank, int world, int max_slots, int slot_floats, void **comm_out,
                                    void *handle_out_host);
DISTEGNN_API int distegnn_comm_connect(void *comm, const void *all_handles_host);
DISTEGNN_API int distegnn_comm_set_timeout_ms(void *comm, int64_t milliseconds);
DISTEGNN_API int distegnn_comm_status(void *comm, int *status_host);
DISTEGNN_API int distegnn_comm_disconnect(void *comm);
DISTEGNN_API int distegnn_comm_destroy(void *comm);
DISTEGNN_API int distegnn_allreduce_packed(void *comm, float *buf, int64_t count, void *stream);

/* ---- virtual-node update, fused with the all-reduce of vsum ---------------------------------------------------------
 * The global halves of coord_model_virtual / node_model_virtual and the next layer's m_X
 * (FastEGNN.py:199, 229-233, 258-264) from the *summed* statistics (weighted_average_reduce,
 * FastEGNN.py:310-319, is Σ_r n_r·mean_r / Σ_r n_r = Σ_r sum_r / Σ_r n_r).  One CTA per graph:
 *   [comm != NULL]  vsum[b,:] := Σ over the partitions (the exchange described above, slot = graph)
 *   n = max(vsum[b,3],1);  Xv += vsum[b,4:4+3C]/n;  Hv += MLP_hv([Hv; vsum[b,4+3C:]/n])
 *   x̄ = vsum[b,0:3]/n;  m_X = (Xv−x̄)ᵀ(Xv−x̄);  G_next = W1v_V·Hv + W1v_M·m_X + b1v (next layer's)
 * FLAG_INIT: skip the Xv/Hv updates (before layer 0); if init_loc_mean [B,3] / init_hv0 [C,64] are given, Xv / Hv are
 * first initialised from them (FastEGNN.py:299-300) instead of being read.  FLAG_LAST: only Xv is updated.
 * FLAG_INIT | FLAG_INIT_CENTROID: X_0 := x̄ = vsum[b,0:3]/n, the per-graph centroid over all partitions of the positions
 * the embedding summed (init_loc_mean must be NULL) — loc_mean of a rollout step without an exchange of its own.  The
 * backward rejects the flag.
 * FLAG_ZERO_VSUM: vsum is left zeroed for the next layer's accumulation; otherwise it holds the summed statistics on
 * return (the training path keeps them for the backward pass).
 * layer_params: this layer's block (node_mlp_virtual); next_layer_params: the block whose virtual MLP
 * consumes G (null with FLAG_LAST).  With FLAG_INIT pass layer 0's block as next_layer_params.
 */
DISTEGNN_API int distegnn_virtual_update_fwd(int n_graphs, int A, int C, int Na, unsigned flags, float *vsum,
                                float *Xv, float *Hv, const float *layer_params,
                                const float *next_layer_params, float *G, const float *init_loc_mean,
                                const float *init_hv0, void *comm, void *stream);

/* Backward of distegnn_virtual_update_fwd (per graph; in the reference: autograd through models/FastEGNN.py:193-199,
 * 222-234, 258-264).  vsum = the SUMMED statistics the forward consumed, Xv / Hv = the forward's inputs (with FLAG_INIT: the
 * initial loc_mean / virtual_node_feat broadcasts).  Upstream g_Xn [B,3,C], g_Hn, g_G [B,C,64] (NULL = zero).  WRITTEN:
 * g_vsum [B,K] (entry 3, the node count, gets 0), g_Xv [B,3,C], g_Hv [B,C,64] (not with FLAG_LAST).  ACCUMULATED: M_W1, M_B1,
 * M_W2, M_B2 of g_layer_params (regular layers) and V_W1V, V_W1M, V_B1 of g_next_layer_params. */
DISTEGNN_API int distegnn_virtual_update_bwd(int n_graphs, int A, int C, int Na, unsigned flags, const float *vsum,
                                             const float *Xv, const float *Hv, const float *layer_params,
                                             const float *next_layer_params, const float *g_Xn, const float *g_Hn,
                                             const float *g_G, float *g_vsum, float *g_Xv, float *g_Hv,
                                             float *g_layer_params, float *g_next_layer_params, void *stream);

/* ---- loss side of the training step (SURVEY §8 f-3) -------------------------------------------------------------------
 * Replaces utils/train.py:98-147: node-count weighted MSE (:98-110), the MMD regulariser between the virtual
 * coordinates and S = samples·C sampled target positions per graph (:119-147, kernel k(x,y) = exp(−‖x−y‖₂/(2σ²)), :11-14)
 * and the per-step scalar collectives (:104, :109 and the loc_mean all_gather check :52-61), folded into ONE packed SUM
 * all-reduce issued by the caller between the two calls (distegnn_allreduce_packed or any SUM all-reduce).
 *   packed [2 + world·3B]  (zeroed by the caller)  [0] n_r, [1] n_r·MSE_r, [2 + r·3B ...] rank r's loc_mean
 *   acc    [3]             (zeroed by the caller)  Σ_b l_vv, Σ_b l_rv, n_r·MSE_r (local copies for the finalize)
 *   graph_ptr [B+1] int64: first node of every graph (data_batch is sorted); samples [B,S] int32: node indices LOCAL to
 *   the graph drawn by the caller (the reference uses torch.randperm(num_node)[:S] per graph; −1 pads graphs with fewer
 *   than S nodes — the reference still divides by S)
 * distegnn_loss_finalize (after the all-reduce): out[0] = loss to back-propagate = world·n_r/Σn·(MSE_r + weight·MMD_r) /
 * accumulation_steps, out[1] = logged loss Σ_r n_r/Σn·MSE_r, out[2] = MMD_r, out[3] = max |loc_mean_r − loc_mean_0|, and
 * the gradients of out[0]: g_pred [N,3], g_Xv [B,3,C] (cdist's convention: zero gradient at coincident points). */
DISTEGNN_API int distegnn_loss_packed_floats(int n_graphs, int world);
DISTEGNN_API int distegnn_loss_partials(int64_t n_nodes, int n_graphs, int C, int S, int world, int rank, float sigma,
                                        const float *pred, const float *target, const float *Xv, const float *loc_mean,
                                        const int64_t *graph_ptr, const int32_t *samples, float *acc, float *packed,
                                        float *gV_raw, void *stream);
DISTEGNN_API int distegnn_loss_finalize(int64_t n_nodes, int n_graphs, int C, int S, int world, int rank, float sigma,
                                        float weight, int accumulation_steps, const float *pred, const float *target,
                                        const float *loc_mean, const float *acc, const float *packed, const float *gV_raw,
                                        float *g_pred, float *g_Xv, float *out, void *stream);

/* ---- deterministic mode (csrc/deterministic.cu, csrc/det.cuh; DESIGN §17) ----------------------------------------------
 * Bitwise-reproducible forward: every floating-point sum is taken in an order fixed by the sizes, never by the grid, the
 * stream, concurrent work or the device-side edge count against the capacity.  The *_det entry points never allocate and
 * never synchronise (capturable); they take one caller-owned workspace of distegnn_deterministic_workspace_bytes(n_nodes,
 * edge_capacity, C) bytes (16-byte aligned; reused across layers and steps).  A forward layer in this mode is
 *   distegnn_edge_layer_fwd_det, then distegnn_edge_combine_det      (agg_m / agg_x complete only after the combine)
 *   distegnn_virtual_layer_fwd_det
 *   distegnn_node_layer_fwd
 *   distegnn_vsum_combine_det on the node layer's x4_out              (vsum complete only after the combine)
 *   distegnn_virtual_update_fwd
 * and the embedding is distegnn_embed_fwd followed by distegnn_vsum_combine_det with DISTEGNN_FLAG_INIT on its x4.
 * distegnn_edge_layer_fwd_det: arguments as distegnn_edge_layer_fwd.  Stores, rather than adds, the partial sums of agg_m
 *   and agg_x: rows whose first edge lies in a 16-edge slice get the slice's partial; later slices of a row fill their
 *   slots.  Rows without an edge are not written (they keep the zeros of a cleared buffer).
 * distegnn_edge_combine_det: adds the slots of every row spanning slices to the row, in slice order (agg_m NULL: last
 *   layer, agg_x only).
 * distegnn_virtual_layer_fwd_det: arguments as distegnn_virtual_layer_fwd.  vsum[:, 4:K] is stored per graph (the chunk
 *   of 16 tiles that holds the graph's first node) and the later chunks' partials go to slots; vsum[:, 0:4] is left to the
 *   combine.
 * distegnn_vsum_combine_det: vsum[b, 0:3] = Σx of x4 over graph b, summed per chunk in node order and the chunks in
 *   chunk order (replacing what the embedding / node kernel added), vsum[b, 3] = the node count; without
 *   DISTEGNN_FLAG_INIT also vsum[b, 4:K] += the graph's slots, in chunk order.  data_batch sorted (int32, as the embedding
 *   writes it).
 *   With DISTEGNN_FLAG_LAST (after a last layer's real<->virtual kernel) only vsum[b, 4:4+3C] takes slots: the rest was
 *   not written in that layer.
 * distegnn_rollout_centroid_det: distegnn_rollout_centroid in a fixed order (no workspace). */
DISTEGNN_API int distegnn_deterministic_workspace_bytes(int64_t n_nodes, int64_t edge_capacity, int C,
                                                        int64_t *bytes_host);
DISTEGNN_API int distegnn_edge_layer_fwd_det(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags,
                                             const int32_t *row, const int32_t *col, const float *edge_attr_sorted,
                                             const float *x4, const float *P, const float *Q, const float *layer_params,
                                             float *agg_m, float *agg_x, const int32_t *n_edges_dev, void *workspace,
                                             int64_t workspace_bytes, void *stream);
DISTEGNN_API int distegnn_edge_combine_det(int64_t n_nodes, int64_t n_edges, int C, const int32_t *row,
                                           const int32_t *n_edges_dev, float *agg_m, float *agg_x, void *workspace,
                                           int64_t workspace_bytes, void *stream);
DISTEGNN_API int distegnn_virtual_layer_fwd_det(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags,
                                                const int32_t *batch32, const float *x4, const float *Hn, const float *Xv,
                                                const float *G, const float *layer_params, float *agg_v, float *trans_v,
                                                float *vsum, void *workspace, int64_t workspace_bytes, void *stream);
DISTEGNN_API int distegnn_vsum_combine_det(int64_t n_nodes, int n_graphs, int C, unsigned flags, const int32_t *batch32,
                                           const float *x4, float *vsum, void *workspace, int64_t workspace_bytes,
                                           void *stream);
DISTEGNN_API int distegnn_rollout_centroid_det(int64_t n_nodes, int n_graphs, const float *pos,
                                               const int64_t *data_batch, double *sums, void *stream);
/* distegnn_rollout_sq_err (csrc/rollout_err.cu): a rollout step's error against recorded targets, between the forward
 * and distegnn_rollout_advance.  With t = counter[0] (the advance's step counter, see distegnn_rollout_advance; nothing is
 * written unless 0 <= t < steps):
 *   sq_err[t, b] = Σ_{i in graph b} ‖pred_i − targets[t, i]‖²     (sq_err float64 [steps, n_graphs], targets [steps, N, 3])
 * with the differences in fp32 (round-to-nearest) and the squares and sums in fp64, in an order fixed by n_nodes and the
 * graph sizes alone: chunks of 2048 rows, each graph's rows in a chunk summed as distegnn_rollout_centroid_det sums, the
 * chunks added in order.  Every entry of row t is stored (0 for a graph without nodes), never accumulated, so a rerun step
 * overwrites its row.  data_batch int64 [N] sorted (NULL for one graph).  One launch, no allocation, no host
 * synchronisation; capturable.  The workspace (distegnn_rollout_sq_err_workspace_bytes, 16-byte aligned) must be zeroed
 * once before the first call; the kernel leaves it fit for the next.  n_nodes 0: nothing is launched. */
DISTEGNN_API int distegnn_rollout_sq_err_workspace_bytes(int64_t n_nodes, int64_t *bytes_host);
DISTEGNN_API int distegnn_rollout_sq_err(int64_t n_nodes, int n_graphs, int steps, const float *pred,
                                         const float *targets, const int64_t *data_batch, const int32_t *counter,
                                         double *sq_err, void *workspace, int64_t workspace_bytes, void *stream);
/* distegnn_rollout_chamfer: the Chamfer distance of a rollout step against its recorded frame (DESIGN §20), launched
 * beside distegnn_rollout_sq_err.  With t = counter[0] (nothing is written unless 0 <= t < steps) and, for graph b, its
 * rows I_b:
 *   chamfer[t, b, 0] = Σ_{i in I_b} min_{j in I_b} d(pred_i, targets[t, j])      (prediction -> record)
 *   chamfer[t, b, 1] = Σ_{j in I_b} min_{i in I_b} d(targets[t, j], pred_i)      (record -> prediction)
 * (chamfer float64 [steps, n_graphs, 2]), d the per-node term of distegnn_rollout_sq_err, every minimum exact.  The sums
 * take that entry point's order, so chamfer[t, b, k] <= sq_err[t, b] bit for bit.  A graph without nodes gets 0, a graph
 * with a non-finite coordinate in pred or targets[t] NaN in both entries.  Row t is stored, never accumulated.
 * data_batch int64 [N] sorted (NULL for one graph); n_nodes + n_graphs <= 2^29.  A fixed number of launches, no
 * allocation, no host synchronisation; capturable.  The workspace (distegnn_rollout_chamfer_workspace_bytes, 16-byte
 * aligned) needs no initialisation.  n_nodes 0: nothing is launched. */
DISTEGNN_API int distegnn_rollout_chamfer_workspace_bytes(int64_t n_nodes, int n_graphs, int64_t *bytes_host);
DISTEGNN_API int distegnn_rollout_chamfer(int64_t n_nodes, int n_graphs, int steps, const float *pred,
                                          const float *targets, const int64_t *data_batch, const int32_t *counter,
                                          double *chamfer, void *workspace, int64_t workspace_bytes, void *stream);

/* ---- frame assembly (csrc/frames.cu; distegnn_b200/frames.py: training batches from raw trajectories) ----------------
 * For a batch of n_samples samples, from the staged frames of each sample's WHOLE scene — frames float32 [3, n_frame_nodes,
 * 3] = (pos[f], x1, pos[f+Δ]) with x1 = pos[f+1] for DISTEGNN_FRAMES_WATER3D and vel[f] otherwise, scenes concatenated at
 * scene_ptr int64 [n_samples+1] — and the static fields statics float32 [n_frame_nodes, S] (S = 1: particle type or
 * charge; S = 2 for DISTEGNN_FRAMES_LARGEFLUID: viscosity, mass), writes this rank's nodes: output node k of sample b
 * (out_ptr int64 [n_samples+1]) is scene node index[k] (int32, scene-local; NULL = every node in order, then n_out ==
 * n_frame_nodes):
 *   node_loc = pos[f], target = pos[f+Δ], node_vel = x1 − pos[f] (Water-3D) or x1   (copies / one fp32 subtraction)
 *   NBODY, WATER3D:  node_feat [n_out,2] = [‖v‖, s / scene_max[b]], node_attr [n_out,1] = s
 *   LARGEFLUID:      node_feat [n_out,3] = [viscosity, mass, ‖v‖], node_attr [n_out,2] = [viscosity, mass]
 *   data_batch int64 [n_out] = b;  ‖v‖ = sqrt((vx·vx + vy·vy) + vz·vz), every operation round-to-nearest, no contraction
 * and per sample, over the whole scene before any split: loc_mean [n_samples,3] = fp32(Σx / n) with Σx in fp64 in a fixed
 * order (deterministic bit for bit), scene_max [n_samples] = max of static column 0.  An index outside its scene yields NaN
 * rows (nothing outside the scene is read).  No workspace, no allocation, no host synchronisation; capturable. */
enum {
    DISTEGNN_FRAMES_NBODY = 0,
    DISTEGNN_FRAMES_WATER3D = 1,
    DISTEGNN_FRAMES_LARGEFLUID = 2,
};
DISTEGNN_API int distegnn_frames_assemble(int recipe, int n_samples, int64_t n_frame_nodes, int64_t n_out,
                                          const float *frames, const float *statics, const int64_t *scene_ptr,
                                          const int64_t *out_ptr, const int32_t *index, float *node_feat,
                                          float *node_loc, float *node_vel, float *node_attr, float *target,
                                          int64_t *data_batch, float *loc_mean, float *scene_max, void *stream);
/* distegnn_frames_targets: multi-step targets.  frames float32 [2 + horizon, n_frame_nodes, 3] = (pos[f], x1, pos[f+Δ],
 * pos[f+2Δ], .., pos[f+horizon·Δ]) per scene (the first three as for distegnn_frames_assemble, which reads only those);
 * writes targets float32 [horizon, n_out, 3] rows 1..horizon−1: targets[t, k] = pos[f+(t+1)Δ] of output node k, with the
 * assembly's scene_ptr, out_ptr and index (NULL = every node in order; an index outside its scene yields NaN rows).
 * Row 0 is not written: pass targets[0] as the assembly's `target`.  Copies only; horizon 1 launches nothing.  No
 * workspace, no allocation, no host synchronisation; capturable. */
DISTEGNN_API int distegnn_frames_targets(int n_samples, int64_t n_frame_nodes, int64_t n_out, int horizon,
                                         const float *frames, const int64_t *scene_ptr, const int64_t *out_ptr,
                                         const int32_t *index, float *targets, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DISTEGNN_B200_H */
