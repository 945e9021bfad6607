// Track-graph construction on the device: everything of GlobalLineTriangulator::ComputeLineTracks
// (global_line_triangulator.cc:234-291) and ComputeLineTrackLabelsGreedy (merging/merging.cc:18-52) that is not the
// sequential union-find itself. The kernels are O(edges) gathers between CUB sorts / scans (plumbing):
//   directed valid connections -> undirected keys (min << 32 | max)          undirected_keys_kernel
//   radix sort + unique                                                      = the std::set order of :243-261
//   spatial-merging score per undirected edge                                edge_weights_kernel (tri_kernels.cu)
//   zero-score edges dropped, order kept (:284-285)                          nonzero_flags + scan + compact
//   Graph::FindOrCreateNode numbering (base/graph.cc:57-70): a node's index is the rank of its FIRST appearance in
//   the stream u0 v0 u1 v1 ...                                               occurrence keys (node << 32 | position),
//                                                                            sort, run heads, sort heads by position
//   edges in descending (score, idx0, idx1) order (merging.cc:27-29: std::sort of tuples, reversed)
//                                                                            two stable radix sorts, LSD
// The host then runs the union-find over an index array.
#include "graph_kernels.cuh"

namespace lm {

namespace {
constexpr int kT = 256;
inline int grid_for(int64_t n) { return (int)((n + kT - 1) / kT); }
} // namespace

__global__ void undirected_keys_kernel(const int64_t *__restrict__ edges, int64_t ne, uint64_t *__restrict__ keys) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint64_t a = (uint64_t)edges[2 * e], b = (uint64_t)edges[2 * e + 1];
  keys[e] = a < b ? (a << 32 | b) : (b << 32 | a);
}
__global__ void keys_to_pairs_kernel(const uint64_t *__restrict__ keys, int64_t n, int64_t *__restrict__ pairs) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  pairs[2 * e] = (int64_t)(keys[e] >> 32);
  pairs[2 * e + 1] = (int64_t)(keys[e] & 0xffffffffull);
}
__global__ void nonzero_flags_kernel(const double *__restrict__ w, int64_t n, uint32_t *__restrict__ flag) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e < n) flag[e] = (w[e] == 0.0) ? 0u : 1u; // `if (score == 0) continue;`
}
__global__ void compact_weighted_edges_kernel(const uint64_t *__restrict__ keys, const double *__restrict__ w,
                                              const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos, int64_t n,
                                              uint64_t *__restrict__ kc, double *__restrict__ wc) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n || !flag[e]) return;
  kc[pos[e]] = keys[e];
  wc[pos[e]] = w[e];
}
__global__ void occurrence_keys_kernel(const uint64_t *__restrict__ kc, int64_t n2, uint64_t *__restrict__ occ) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n2) return;
  occ[2 * e] = (kc[e] >> 32) << 32 | (uint64_t)(2 * e);
  occ[2 * e + 1] = (kc[e] & 0xffffffffull) << 32 | (uint64_t)(2 * e + 1);
}
__global__ void occurrence_heads_kernel(const uint64_t *__restrict__ occ, int64_t m, uint32_t *__restrict__ head) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < m) head[i] = (i == 0 || (occ[i] >> 32) != (occ[i - 1] >> 32)) ? 1u : 0u;
}
__global__ void head_keys_kernel(const uint64_t *__restrict__ occ, const uint32_t *__restrict__ head,
                                 const uint32_t *__restrict__ pos, int64_t m, uint64_t *__restrict__ hk) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m || !head[i]) return;
  hk[pos[i]] = (occ[i] & 0xffffffffull) << 32 | (occ[i] >> 32); // (first position, node)
}
__global__ void graph_index_kernel(const uint64_t *__restrict__ hk, int64_t ng, int32_t *__restrict__ gidx,
                                   int32_t *__restrict__ gnode) {
  const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (g >= ng) return;
  const int32_t node = (int32_t)(hk[g] & 0xffffffffull);
  gnode[g] = node;
  gidx[node] = (int32_t)g;
}
// descending order = ascending order of the complemented keys; scores are finite doubles (the usual sign fold keeps
// the order for negative values too)
__global__ void edge_order_keys_kernel(const uint64_t *__restrict__ kc, const double *__restrict__ wc,
                                       const int32_t *__restrict__ gidx, int64_t n2, uint64_t *__restrict__ by_nodes,
                                       uint64_t *__restrict__ by_score) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n2) return;
  const uint64_t i0 = (uint32_t)gidx[kc[e] >> 32], i1 = (uint32_t)gidx[kc[e] & 0xffffffffull];
  by_nodes[e] = ~(i0 << 32 | i1);
  by_score[e] = descending_double_key(wc[e]);
}

void launch_undirected_keys(const int64_t *edges, int64_t ne, uint64_t *keys, cudaStream_t s) {
  if (ne > 0) undirected_keys_kernel<<<grid_for(ne), kT, 0, s>>>(edges, ne, keys);
}
void launch_keys_to_pairs(const uint64_t *keys, int64_t n, int64_t *pairs, cudaStream_t s) {
  if (n > 0) keys_to_pairs_kernel<<<grid_for(n), kT, 0, s>>>(keys, n, pairs);
}
void launch_nonzero_flags(const double *w, int64_t n, uint32_t *flag, cudaStream_t s) {
  if (n > 0) nonzero_flags_kernel<<<grid_for(n), kT, 0, s>>>(w, n, flag);
}
void launch_compact_weighted_edges(const uint64_t *keys, const double *w, const uint32_t *flag, const uint32_t *pos, int64_t n,
                                   uint64_t *kc, double *wc, cudaStream_t s) {
  if (n > 0) compact_weighted_edges_kernel<<<grid_for(n), kT, 0, s>>>(keys, w, flag, pos, n, kc, wc);
}
void launch_occurrence_keys(const uint64_t *kc, int64_t n2, uint64_t *occ, cudaStream_t s) {
  if (n2 > 0) occurrence_keys_kernel<<<grid_for(n2), kT, 0, s>>>(kc, n2, occ);
}
void launch_occurrence_heads(const uint64_t *occ_sorted, int64_t m, uint32_t *head, cudaStream_t s) {
  if (m > 0) occurrence_heads_kernel<<<grid_for(m), kT, 0, s>>>(occ_sorted, m, head);
}
void launch_head_keys(const uint64_t *occ_sorted, const uint32_t *head, const uint32_t *pos, int64_t m, uint64_t *hk,
                      cudaStream_t s) {
  if (m > 0) head_keys_kernel<<<grid_for(m), kT, 0, s>>>(occ_sorted, head, pos, m, hk);
}
void launch_graph_index(const uint64_t *hk_sorted, int64_t ng, int32_t *gidx, int32_t *gnode, cudaStream_t s) {
  if (ng > 0) graph_index_kernel<<<grid_for(ng), kT, 0, s>>>(hk_sorted, ng, gidx, gnode);
}
void launch_edge_order_keys(const uint64_t *kc, const double *wc, const int32_t *gidx, int64_t n2, uint64_t *by_nodes,
                            uint64_t *by_score, cudaStream_t s) {
  if (n2 > 0) edge_order_keys_kernel<<<grid_for(n2), kT, 0, s>>>(kc, wc, gidx, n2, by_nodes, by_score);
}

} // namespace lm
