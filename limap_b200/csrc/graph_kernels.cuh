// Track-graph construction on the device (GlobalLineTriangulator::ComputeLineTracks up to the union-find):
// undirected edge set, zero-score filter, graph-node numbering in the reference's FindOrCreateNode order and the
// (score, node, node)-descending edge order of ComputeLineTrackLabelsGreedy. See graph_kernels.cu.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace lm {

// Radix key that sorts finite doubles in descending order (ascending order of the complemented, sign-folded bits).
__device__ __forceinline__ uint64_t descending_double_key(double w) {
  uint64_t b = (uint64_t)__double_as_longlong(w);
  b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
  return ~b;
}

void launch_undirected_keys(const int64_t *edges, int64_t ne, uint64_t *keys, cudaStream_t s);
void launch_keys_to_pairs(const uint64_t *keys, int64_t n, int64_t *pairs, cudaStream_t s);
void launch_nonzero_flags(const double *w, int64_t n, uint32_t *flag, cudaStream_t s);
void launch_compact_weighted_edges(const uint64_t *keys, const double *w, const uint32_t *flag, const uint32_t *pos, int64_t n,
                                   uint64_t *kc, double *wc, cudaStream_t s);
void launch_occurrence_keys(const uint64_t *kc, int64_t n2, uint64_t *occ, cudaStream_t s);
void launch_occurrence_heads(const uint64_t *occ_sorted, int64_t m, uint32_t *head, cudaStream_t s);
void launch_head_keys(const uint64_t *occ_sorted, const uint32_t *head, const uint32_t *pos, int64_t m, uint64_t *hk,
                      cudaStream_t s);
void launch_graph_index(const uint64_t *hk_sorted, int64_t ng, int32_t *gidx, int32_t *gnode, cudaStream_t s);
void launch_edge_order_keys(const uint64_t *kc, const double *wc, const int32_t *gidx, int64_t n2, uint64_t *by_nodes,
                            uint64_t *by_score, cudaStream_t s);

} // namespace lm
