// Deterministic mode (DESIGN §17): the workspace of the *_det entry points and the fixed units its slots belong to.
//
// Every floating-point sum of the forward is taken in an order fixed by the input sizes alone:
//   edge stage   the edges are cut into slices of 16 (warp w of tile t owns edges 16(4t + w) .. +15, whatever the grid);
//                a slice sums its runs of equal destination row in edge order and stores each partial.  A row's first
//                slice writes it to the row, every later slice of the row to its slot; distegnn_edge_combine_det adds
//                the slots in slice order.
//   vsum         the real<->virtual kernel's tiles are grouped into chunks of 2^det_chunk_shift(N, C) consecutive tiles
//                (16 or more, a power of two: at most DET_MAX_CHUNKS chunks); a chunk is summed in tile order by one
//                pipeline.  A graph's first chunk writes its partial to vsum, every later chunk of the graph to the
//                chunk's slot.  distegnn_vsum_combine_det sums the coordinates of each chunk's nodes in node order the
//                same way (entries 0..2), then adds the slots in chunk order.
// Workspace: [vsum slots: chunks x K floats | edge slots: ceil(E_capacity / 16) x DET_EDGE_SLOT floats], each part
// 256-byte aligned.
//
// The other atomics of the forward path need no deterministic twin: the embedding and node kernels' Σ(x, 1) adds into
// vsum[:, 0:4] are overwritten by the combine; the data_batch validation counter, the rollout step counters, the radius
// build (ordered-int bounding box, integer counts and scans) and the edge cutoff (integer histograms and scans,
// cutoff_csr.cu) are integer-only and deterministic already; the forward virtual-node update sums inside one block per
// graph; the peer-memory exchange adds the ranks in rank order.  The rollout's final centroid has a fixed-order kernel
// (distegnn_rollout_centroid_det).
#pragma once

#include "common.cuh"

namespace degnn {

constexpr int DET_EDGE_SLOT = 68;      // 64 (agg_m) + 3 (agg_x), padded to 16 bytes
constexpr int DET_MIN_CHUNK = 16;      // real<->virtual tiles per chunk, at least
constexpr int64_t DET_MAX_CHUNKS = 4096;   // bounds the in-order combine (and the slots) per graph
constexpr int DET_VTILE = 64;          // rows per real<->virtual tile (VW_TILE)

__host__ __device__ inline int det_nodes_per_tile(int C) { return DET_VTILE / C; }
inline int64_t det_tiles(int64_t N, int C) { return (N + det_nodes_per_tile(C) - 1) / det_nodes_per_tile(C); }
// log2 of the tiles per chunk: the smallest power of two >= DET_MIN_CHUNK that leaves at most DET_MAX_CHUNKS chunks
inline int det_chunk_shift(int64_t N, int C) {
    int s = 4;
    while (((det_tiles(N, C) + (1ll << s) - 1) >> s) > DET_MAX_CHUNKS) ++s;
    return s;
}
inline int64_t det_chunks(int64_t N, int C) {
    const int s = det_chunk_shift(N, C);
    return (det_tiles(N, C) + (1ll << s) - 1) >> s;
}
inline int det_K(int C) { return 4 + 3 * C + H * C; }
inline int64_t det_vsum_bytes(int64_t N, int C) { return (int64_t)align256(det_chunks(N, C) * det_K(C) * 4); }
inline int64_t det_edge_bytes(int64_t E) { return (int64_t)align256((E + 15) / 16 * DET_EDGE_SLOT * 4); }
inline float* det_vsum_slots(void* ws) { return reinterpret_cast<float*>(ws); }
inline float* det_edge_slots(void* ws, int64_t N, int C) {
    return reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + det_vsum_bytes(N, C));
}

// Null / misaligned / too small workspace -> DISTEGNN_EINVAL / DISTEGNN_EWORKSPACE (with the error string set).
// `n_edges` < 0: only the vsum part is needed.
int det_check_workspace(int64_t n_nodes, int64_t n_edges, int C, const void* ws, int64_t ws_bytes, const char* who);
// min(grid, max_ctas) (max_ctas 0: no cap); at least 1.  The public entry points pass 0; the testing library's capped
// twins (include/distegnn_b200_testing_det.h) pass a cap, so that tests can check that the bits do not depend on the grid.
inline int64_t det_grid(int64_t grid, int max_ctas) {
    if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
    return grid < 1 ? 1 : grid;
}

// the *_det entry points with a grid cap
int edge_layer_fwd_det(int64_t n_nodes, int64_t n_edges, int A, int C, int Na, unsigned flags, const int32_t* row,
                       const int32_t* col, const float* edge_attr_sorted, const float* x4, const float* P, const float* Q,
                       const float* layer_params, float* agg_m, float* agg_x, const int32_t* n_edges_dev,
                       void* workspace, int64_t workspace_bytes, void* stream, int max_ctas);
int edge_combine_det(int64_t n_nodes, int64_t n_edges, int C, const int32_t* row, const int32_t* n_edges_dev,
                     float* agg_m, float* agg_x, void* workspace, int64_t workspace_bytes, void* stream, int max_ctas);
int virtual_layer_fwd_det(int64_t n_nodes, int n_graphs, int A, int C, int Na, unsigned flags, const int32_t* batch32,
                          const float* x4, const float* Hn, const float* Xv, const float* G, const float* layer_params,
                          float* agg_v, float* trans_v, float* vsum, void* workspace, int64_t workspace_bytes,
                          void* stream, int max_ctas);
int vsum_combine_det(int64_t n_nodes, int n_graphs, int C, unsigned flags, const int32_t* batch32, const float* x4,
                     float* vsum, void* workspace, int64_t workspace_bytes, void* stream, int max_ctas);

}  // namespace degnn
