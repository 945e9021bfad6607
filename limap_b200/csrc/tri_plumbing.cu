// tri_plumbing.cu — the plumbing kernels of the line-triangulation path (DESIGN.md §3.3): block tables, match rows ->
// node-major rows and node offsets, valid-connection compaction and the host edge export, scene preparation, the
// multi-GPU pack / unpack and run_clustering's edge weights.
//   view_tables / row_count / row_place / node_row_off : turn the per-(image, neighbour) match tables into node-major
//       rows and every node's row range.
//   group_edges / edge_pairs / edge_weights : run_clustering's edge list and 3d scores
//       (global_line_triangulator.cc:234-291).
#include "tri_kernels.cuh"
#include <algorithm>

namespace lm {

// The per-run block tables (match tables ordered by (source view, neighbour), row offsets) are derived on the
// device from block descriptors that were uploaded together with the matches. Nothing has to cross PCIe when
// a run starts: any host->device transfer issued then (copy-engine copies, large kernel parameters, even
// zero-copy reads) was measured to wait ~3 ms behind a 160 MB match upload still in flight.
__global__ void block_keys_kernel(const RawBlock *__restrict__ raw, int n_all, int vb, int ve, int exhaustive,
                                  uint32_t *__restrict__ key, uint32_t *__restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_all) return;
  const RawBlock b = raw[i];
  const bool in = b.src_view >= vb && b.src_view < ve;
  key[i] = in ? (((uint32_t)b.src_view << 16) | (uint32_t)(exhaustive ? b.order : b.ng_view)) : 0xffffffffu;
  val[i] = (uint32_t)i;
}
__global__ void block_gather_kernel(const RawBlock *__restrict__ raw, const uint32_t *__restrict__ sorted_idx, int nb,
                                    int32_t *__restrict__ blk_src, int32_t *__restrict__ blk_ng,
                                    int64_t *__restrict__ blk_pair_off, int64_t *__restrict__ blk_rows,
                                    int32_t *__restrict__ blk_chunks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nb) return;
  if (i == nb) { blk_rows[i] = 0; blk_chunks[i] = 0; return; }
  const RawBlock b = raw[sorted_idx[i]];
  blk_src[i] = b.src_view;
  blk_ng[i] = b.ng_view;
  blk_pair_off[i] = b.pair_off;
  blk_rows[i] = b.n_rows;
  blk_chunks[i] = (int32_t)((b.n_rows + kRowChunk - 1) / kRowChunk);
}
void launch_block_keys(const RawBlock *raw, int n_all, int vb, int ve, int exhaustive, uint32_t *key, uint32_t *val,
                       cudaStream_t s) {
  if (n_all <= 0) return;
  block_keys_kernel<<<(n_all + 255) / 256, 256, 0, s>>>(raw, n_all, vb, ve, exhaustive, key, val);
}
void launch_block_gather(const RawBlock *raw, const uint32_t *sorted_idx, int nb, int32_t *blk_src, int32_t *blk_ng,
                         int64_t *blk_pair_off, int64_t *blk_rows, int32_t *blk_chunks, cudaStream_t s) {
  block_gather_kernel<<<(nb + 1 + 255) / 256, 256, 0, s>>>(raw, sorted_idx, nb, blk_src, blk_ng, blk_pair_off, blk_rows,
                                                           blk_chunks);
}
__global__ void zero_words_kernel(unsigned int *p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0u;
}
// cudaMemsetAsync may be routed to a copy engine and then waits behind a running match upload
void launch_zero_words(void *d_dst, int n_words, cudaStream_t s) {
  zero_words_kernel<<<(n_words + 127) / 128, 128, 0, s>>>(static_cast<unsigned int *>(d_dst), n_words);
}

// ------------------------------------------------------------------------------------------------
// Match tables -> node-major rows. Flat row order = (source view asc, neighbour view asc, row), the order in which
// TriangulateImage appends to tris_ (base_line_triangulator.cc:74-100). The rows of one source view already occupy the
// output range they end up in, so putting them in node order is a stable bucketing by line inside that range, and every
// node gets its candidates in (block, row) order, the reference's order.
//
// Every block is cut into chunks of at most kRowChunk rows (a chunk never spans blocks, so no kernel searches the block
// of a row). row_count counts the rows of every line of the source view per chunk into a table laid out per source view
// as [line][chunk of the view]. One exclusive scan over a pipeline group's slice of that table gives the first row of
// every (line, chunk) relative to the group's first row; the entry of a line's first chunk is its node's first row.
// row_place then writes each chunk's rows there, in order. Only one CTA advances a chunk's positions: no atomics, and
// the result is deterministic.

// lower_bound(blk_src[0, nb), v): the first block whose source view is v or later
LM_D int first_block_of(const int32_t *__restrict__ blk_src, int nb, int v) {
  int lo = 0, hi = nb;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (blk_src[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// The per-view tables of the shard's views [vb, ve]: first chunk, first flat row and count-table entries (lines x chunks).
__global__ void view_tables_kernel(const int32_t *__restrict__ blk_src, const int32_t *__restrict__ blk_chunk_off,
                                   const int64_t *__restrict__ blk_row_off, int nb, const int64_t *__restrict__ line_off,
                                   int vb, int ve, int32_t *__restrict__ view_chunk_off,
                                   int64_t *__restrict__ view_row_off, int32_t *__restrict__ view_ent) {
  const int v = vb + blockIdx.x * blockDim.x + threadIdx.x;
  if (v > ve) return;
  const int b = first_block_of(blk_src, nb, v);
  view_chunk_off[v] = blk_chunk_off[b];
  view_row_off[v] = blk_row_off[b];
  view_ent[v] = 0;
  if (v < ve)
    view_ent[v] = (int32_t)((line_off[v + 1] - line_off[v]) * (blk_chunk_off[first_block_of(blk_src, nb, v + 1)] - blk_chunk_off[b]));
}
void launch_view_tables(const RowTables &t, int vb, int ve, int32_t *view_ent, cudaStream_t s) {
  view_tables_kernel<<<(ve - vb + 1 + 255) / 256, 256, 0, s>>>(t.blk_src, t.blk_chunk_off, t.blk_row_off, t.nb, t.line_off,
                                                               vb, ve, const_cast<int32_t *>(t.view_chunk_off),
                                                               const_cast<int64_t *>(t.view_row_off), view_ent);
}

// Chunk k of the shard: its rows [r0, r1) and first match pair, its views and line counts, its column of the count table.
struct RowChunk {
  int64_t r0, r1, q0, tab; // tab: entry of line 0; line l at tab + l * nch
  int sv, nv, nl, nl_ng, nch;
};
LM_D RowChunk row_chunk(const RowTables &t, int k) {
  RowChunk c;
  const int b = last_le(t.blk_chunk_off, t.nb, k);
  const int64_t j = (int64_t)(k - t.blk_chunk_off[b]) * kRowChunk;
  c.r0 = t.blk_row_off[b] + j;
  c.r1 = min(c.r0 + kRowChunk, t.blk_row_off[b + 1]);
  c.q0 = t.blk_pair_off[b] + j;
  c.sv = t.blk_src[b];
  c.nv = t.blk_ng[b];
  c.nl = (int)(t.line_off[c.sv + 1] - t.line_off[c.sv]);
  c.nl_ng = (int)(t.line_off[c.nv + 1] - t.line_off[c.nv]);
  c.nch = t.view_chunk_off[c.sv + 1] - t.view_chunk_off[c.sv];
  c.tab = t.view_tab_off[c.sv] + (k - t.view_chunk_off[c.sv]);
  return c;
}

constexpr int kRowThreads = 256;

// Pass 1: rows per line of chunk k0 + blockIdx.x, and the IndexError flags (d_scalars word 1).
__global__ void __launch_bounds__(kRowThreads) row_count_kernel(const __grid_constant__ RowTables t,
                                                                const int32_t *__restrict__ pairs, int k0,
                                                                uint16_t *__restrict__ cnt, int *err) {
  extern __shared__ uint32_t lc[]; // two 16-bit line counters per word (a chunk has fewer than 2^16 rows)
  const RowChunk c = row_chunk(t, k0 + blockIdx.x);
  for (int i = threadIdx.x; i < (c.nl + 1) / 2; i += kRowThreads) lc[i] = 0u;
  __syncthreads();
  const int2 *pr = reinterpret_cast<const int2 *>(pairs) + c.q0;
  const int n = (int)(c.r1 - c.r0);
  for (int i = threadIdx.x; i < n; i += kRowThreads) {
    const int2 m = pr[i];
    int line = m.x;
    if (line < 0 || line >= c.nl) { *err = 1; line = 0; }
    if (m.y < 0 || m.y >= c.nl_ng) *err = 2;
    if (c.nl > 0) atomicAdd(&lc[line >> 1], 1u << ((line & 1) * 16));
  }
  __syncthreads();
  for (int l = threadIdx.x; l < c.nl; l += kRowThreads)
    cnt[c.tab + (int64_t)l * c.nch] = (uint16_t)(lc[l >> 1] >> ((l & 1) * 16));
}

// Pass 2: the rows of chunk k0 + blockIdx.x at their node-major positions (pos: the scanned count table, relative to
// row_base). A tile of kRowThreads rows at a time: a row's rank among the equal lines of its warp comes from
// __match_any_sync, and the warps take turns, in row order, to advance the chunk's running count of each line.
__global__ void __launch_bounds__(kRowThreads) row_place_kernel(const __grid_constant__ RowTables t,
                                                                const int32_t *__restrict__ pairs, int k0,
                                                                const uint32_t *__restrict__ pos, int64_t row_base,
                                                                uint32_t *__restrict__ row_ng) {
  extern __shared__ uint16_t run[]; // rows of every line this chunk has placed so far
  const RowChunk c = row_chunk(t, k0 + blockIdx.x);
  for (int l = threadIdx.x; l < c.nl; l += kRowThreads) run[l] = 0;
  __syncthreads();
  if (c.nl == 0) return; // (every row is out of range: row_count raised the IndexError)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 *pr = reinterpret_cast<const int2 *>(pairs) + c.q0;
  const int n = (int)(c.r1 - c.r0);
  int2 next = threadIdx.x < n ? pr[threadIdx.x] : make_int2(0, 0);
  for (int i0 = 0; i0 < n; i0 += kRowThreads) {
    const int i = i0 + threadIdx.x;
    const bool valid = i < n;
    const int2 m = next;
    if (i + kRowThreads < n) next = pr[i + kRowThreads];
    int line = m.x, ngl = m.y;
    if (line < 0 || line >= c.nl) line = 0;
    if (ngl < 0 || ngl >= c.nl_ng) ngl = 0;
    const unsigned same = __match_any_sync(0xffffffffu, valid ? line : -1);
    const unsigned before = same & ((1u << lane) - 1u);
    const bool head = valid && before == 0u; // the first row of its line in this warp
    uint32_t base = head ? __ldg(&pos[c.tab + (int64_t)line * c.nch]) : 0u;
    for (int w = 0; w < kRowThreads / 32; ++w) {
      if (w == warp && head) {
        const uint16_t k = run[line];
        run[line] = (uint16_t)(k + __popc(same));
        base += k;
      }
      __syncthreads();
    }
    base = __shfl_sync(0xffffffffu, base, __ffs(same) - 1);
    if (valid) row_ng[row_base + base + __popc(before)] = ((uint32_t)c.nv << 16) | (uint32_t)ngl;
  }
}

static cudaError_t set_smem(const void *f, size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                          : cudaSuccess;
}
cudaError_t launch_row_count(const RowTables &t, const int32_t *pairs, int k0, int n_chunks, int nl_max, uint16_t *cnt,
                             int *err, cudaStream_t s) {
  if (n_chunks <= 0) return cudaSuccess;
  const size_t smem = 4 * (size_t)((nl_max + 1) / 2);
  cudaError_t e = set_smem((const void *)row_count_kernel, smem);
  if (e != cudaSuccess) return e;
  row_count_kernel<<<n_chunks, kRowThreads, smem, s>>>(t, pairs, k0, cnt, err);
  return cudaGetLastError();
}
cudaError_t launch_row_place(const RowTables &t, const int32_t *pairs, int k0, int n_chunks, int nl_max,
                             const uint32_t *pos, int64_t row_base, uint32_t *row_ng, cudaStream_t s) {
  if (n_chunks <= 0) return cudaSuccess;
  const size_t smem = 4 * (size_t)((nl_max + 1) / 2);
  cudaError_t e = set_smem((const void *)row_place_kernel, smem);
  if (e != cudaSuccess) return e;
  row_place_kernel<<<n_chunks, kRowThreads, smem, s>>>(t, pairs, k0, pos, row_base, row_ng);
  return cudaGetLastError();
}

// TriangulateImageExhaustiveMatch (base_line_triangulator.cc:111-136): every line of the source view gets every line of
// every neighbour, so a row's position is closed-form: its node's first row plus the lines of the earlier neighbours.
__global__ void place_exhaustive_kernel(const __grid_constant__ RowTables t, int64_t n_rows, uint32_t *__restrict__ row_ng) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    const int b = last_le(t.blk_row_off, t.nb, r);
    const int sv = t.blk_src[b], nv = t.blk_ng[b];
    const int64_t nl = t.line_off[sv + 1] - t.line_off[sv], nl_ng = t.line_off[nv + 1] - t.line_off[nv];
    const int64_t q = r - t.blk_row_off[b], v0 = t.view_row_off[sv];
    const int64_t per_line = (t.view_row_off[sv + 1] - v0) / nl;
    row_ng[v0 + (q / nl_ng) * per_line + (t.blk_row_off[b] - v0) / nl + q % nl_ng] =
        ((uint32_t)nv << 16) | (uint32_t)(q % nl_ng);
  }
}
void launch_place_exhaustive(const RowTables &t, int64_t n_rows, uint32_t *row_ng, cudaStream_t s) {
  if (n_rows <= 0) return;
  int grid = (int)((n_rows + 255) / 256);
  grid = std::min(grid, current_device_sms() * 16);
  place_exhaustive_kernel<<<grid, 256, 0, s>>>(t, n_rows, row_ng);
}

// Row range of every node in [node_lo, node_hi] of one pipeline group, whose rows are [row_base, row_end) of the run;
// off[n] is a row index of the whole run and off[node_hi] = row_end. Matches: from the group's scanned count table,
// entries [.., t_end). Exhaustive matching: every line of a source view has the same number of rows. The largest node
// goes to max_rows.
__global__ void node_row_off_kernel(const __grid_constant__ RowTables t, const uint32_t *__restrict__ pos, int64_t t_end,
                                    int64_t row_base, int64_t row_end, int64_t node_lo, int64_t node_hi, int n_views,
                                    int exhaustive, uint32_t *__restrict__ off, unsigned int *max_rows) {
  const int64_t n = node_lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (n > node_hi) return;
  if (n == node_hi) { off[n] = (uint32_t)row_end; return; }
  const int sv = last_le(t.line_off, n_views, n);
  const int64_t l = n - t.line_off[sv];
  int64_t first, cnt;
  if (exhaustive) {
    cnt = (t.view_row_off[sv + 1] - t.view_row_off[sv]) / (t.line_off[sv + 1] - t.line_off[sv]);
    first = t.view_row_off[sv] + l * cnt;
  } else {
    const int64_t nch = t.view_chunk_off[sv + 1] - t.view_chunk_off[sv];
    const int64_t i = t.view_tab_off[sv] + l * nch, tot = row_end - row_base;
    const int64_t a = i < t_end ? (int64_t)pos[i] : tot, b = i + nch < t_end ? (int64_t)pos[i + nch] : tot;
    first = row_base + a;
    cnt = b - a;
  }
  off[n] = (uint32_t)first;
  if (cnt) atomicMax(max_rows, (unsigned int)cnt);
}
void launch_node_row_off(const RowTables &t, const uint32_t *pos, int64_t t_end, int64_t row_base, int64_t row_end,
                         int64_t node_lo, int64_t node_hi, int n_views, int exhaustive, uint32_t *off,
                         unsigned int *max_rows, cudaStream_t s) {
  const int grid = (int)((node_hi - node_lo + 1 + 255) / 256);
  node_row_off_kernel<<<grid, 256, 0, s>>>(t, pos, t_end, row_base, row_end, node_lo, node_hi, n_views, exhaustive, off,
                                           max_rows);
}

// valid_edges_ (global_line_triangulator.cc:130-142) in compact, node-major, candidate-ordered form.
__global__ void extract_nvalid_kernel(const NodeRecord *__restrict__ nodes, int64_t node_begin, int64_t n,
                                      uint32_t *__restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint32_t)nodes[node_begin + i].n_valid;
  if (i == n) out[i] = 0;
}
// Valid connections of one pipeline group, right after the group's node kernel: global offsets (the groups before it are
// done: their totals are on the device) and compact (neighbour view << 16 | line) entries in candidate order. One warp
// per node. (Writing the caller's page-locked result buffers from here over PCIe was measured: 0.25 ms SLOWER per step
// than one device-to-host copy after the run.)
__global__ void group_edges_kernel(const uint8_t *__restrict__ row_state, const uint32_t *__restrict__ row_ng,
                                   const uint32_t *__restrict__ node_row_off, const uint32_t *__restrict__ local_off,
                                   unsigned int *__restrict__ totals, int g, int64_t shard_node_begin, int64_t node_lo, int64_t n,
                                   int ns, uint32_t *__restrict__ edge_off, uint32_t *__restrict__ edge_ng) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
  if (i >= n) return;
  uint32_t before = 0;
  for (int k = 0; k < g; ++k) before += totals[k];
  const uint32_t lo = local_off[i], hi = local_off[i + 1];
  uint32_t base = before + lo;
  if (lane == 0) {
    edge_off[node_lo - shard_node_begin + i] = base;
    if (i == n - 1) {
      edge_off[node_lo - shard_node_begin + n] = before + local_off[n];
      totals[g] = local_off[n];
    }
  }
  if (hi == lo) return;
  const int64_t q0 = (int64_t)node_row_off[node_lo + i] * ns, q1 = (int64_t)node_row_off[node_lo + i + 1] * ns;
  for (int64_t qb = q0; qb < q1; qb += 32) { // q = row * ns + slot: candidate order
    const int64_t q = qb + lane;
    const bool v = (q < q1) && row_state[q] == 2;
    const unsigned m = __ballot_sync(0xffffffffu, v);
    if (v) edge_ng[base + __popc(m & ((1u << lane) - 1u))] = row_ng[q / ns];
    base += __popc(m);
  }
}
void launch_group_edges(const uint8_t *row_state, const uint32_t *row_ng, const uint32_t *node_row_off,
                        const uint32_t *local_off, unsigned int *totals, int g, int64_t shard_node_begin, int64_t node_lo,
                        int64_t n, int ns, uint32_t *edge_off, uint32_t *edge_ng, cudaStream_t s) {
  if (n <= 0) return;
  group_edges_kernel<<<(int)((n * 32 + 255) / 256), 256, 0, s>>>(row_state, row_ng, node_row_off, local_off, totals, g,
                                                                 shard_node_begin, node_lo, n, ns, edge_off, edge_ng);
}
// directed (src node, dst node) pairs of the compact edge list
__global__ void edge_pairs_kernel(const uint32_t *__restrict__ edge_off, const uint32_t *__restrict__ edge_ng,
                                  const int64_t *__restrict__ line_off, int64_t node_begin, int64_t n_nodes,
                                  int64_t n_edges, int64_t *__restrict__ out) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int64_t i = last_le(edge_off, n_nodes, (uint32_t)e);
  const uint32_t ng = edge_ng[e];
  out[2 * e] = node_begin + i;
  out[2 * e + 1] = line_off[ng >> 16] + (ng & 0xffffu);
}
void launch_edge_pairs(const uint32_t *edge_off, const uint32_t *edge_ng, const int64_t *line_off,
                       int64_t node_begin, int64_t n_nodes, int64_t n_edges, int64_t *out, cudaStream_t s) {
  if (n_edges <= 0) return;
  edge_pairs_kernel<<<(int)((n_edges + 255) / 256), 256, 0, s>>>(edge_off, edge_ng, line_off, node_begin, n_nodes,
                                                                 n_edges, out);
}
void launch_extract_nvalid(const NodeRecord *nodes, int64_t node_begin, int64_t n, uint32_t *out, cudaStream_t s) {
  extract_nvalid_kernel<<<(int)((n + 1 + 255) / 256), 256, 0, s>>>(nodes, node_begin, n, out);
}

// valid connections as (ng_img_id, ng_line_id) int32 pairs + int64 node offsets, ready for the caller's buffer
__global__ void edges_for_host_kernel(const uint32_t *__restrict__ edge_off, const uint32_t *__restrict__ edge_ng,
                                      const int32_t *__restrict__ img_ids, int64_t n_nodes_shard, int64_t n_edges,
                                      int64_t node_begin, int64_t n_nodes_total, int64_t *__restrict__ node_off,
                                      int32_t *__restrict__ pairs) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t < n_edges) {
    const uint32_t ng = edge_ng[t];
    pairs[2 * t] = img_ids[ng >> 16];
    pairs[2 * t + 1] = (int32_t)(ng & 0xffffu);
  }
  if (t <= n_nodes_total) {
    int64_t v = 0;
    if (t >= node_begin && t <= node_begin + n_nodes_shard) v = edge_off[t - node_begin];
    else if (t > node_begin + n_nodes_shard) v = n_edges;
    node_off[t] = v;
  }
}
void launch_edges_for_host(const uint32_t *edge_off, const uint32_t *edge_ng, const int32_t *img_ids,
                           int64_t n_nodes_shard, int64_t n_edges, int64_t node_begin, int64_t n_nodes_total,
                           int64_t *node_off, int32_t *pairs, cudaStream_t s) {
  const int64_t n = (n_edges > n_nodes_total + 1) ? n_edges : n_nodes_total + 1;
  edges_for_host_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(edge_off, edge_ng, img_ids, n_nodes_shard, n_edges,
                                                               node_begin, n_nodes_total, node_off, pairs);
}

// ---- scene preparation: the 2D segments as the kernels read them (add_halfpix, base_line_triangulator.cc:32-43) and the
// view of every node, derived on the device from what lm_scene_upload copied ------------------------------------------
__global__ void scene_prepare_kernel(const double *__restrict__ segs_raw, int64_t n_nodes, double add,
                                     const int64_t *__restrict__ line_off, int n_views, double *__restrict__ segs,
                                     uint16_t *__restrict__ node_view) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < 4 * n_nodes) segs[i] = segs_raw[i] + add;
  if (i < n_nodes && node_view) node_view[i] = (uint16_t)last_le(line_off, n_views, i);
}
void launch_scene_prepare(const double *segs_raw, int64_t n_nodes, double add, const int64_t *line_off, int n_views,
                          double *segs, uint16_t *node_view, cudaStream_t s) {
  if (n_nodes <= 0) return;
  scene_prepare_kernel<<<(int)((4 * n_nodes + 255) / 256), 256, 0, s>>>(segs_raw, n_nodes, add, line_off, n_views, segs, node_view);
}

// ---- multi-GPU exchange: one fixed-size message per rank (SURVEY.md 8e: "one all-gather of per-node results") ----
// message = [int64 n_edges, int64 n_nodes] | NodeRecord[max_nodes] | (uint32 src_node, uint32 dst_node)[cap_edges]
__global__ void gather_pack_kernel(const NodeRecord *__restrict__ nodes, int64_t node_begin, int64_t n_nodes,
                                   int64_t max_nodes, const uint32_t *__restrict__ edge_off,
                                   const uint32_t *__restrict__ edge_ng, const int64_t *__restrict__ line_off,
                                   int64_t cap_edges, char *__restrict__ msg) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  const int64_t ne = n_nodes > 0 ? (int64_t)edge_off[n_nodes] : 0;
  if (tid == 0) { reinterpret_cast<int64_t *>(msg)[0] = ne; reinterpret_cast<int64_t *>(msg)[1] = n_nodes; }
  const uint4 *src = reinterpret_cast<const uint4 *>(nodes + node_begin);
  uint4 *dst = reinterpret_cast<uint4 *>(msg + 16);
  const int64_t nv = n_nodes * (int64_t)(sizeof(NodeRecord) / 16);
  for (int64_t i = tid; i < nv; i += nth) dst[i] = src[i];
  uint2 *ed = reinterpret_cast<uint2 *>(msg + 16 + max_nodes * (int64_t)sizeof(NodeRecord));
  const int64_t nc = ne < cap_edges ? ne : cap_edges;
  for (int64_t e = tid; e < nc; e += nth) {
    const int64_t i = last_le(edge_off, n_nodes, (uint32_t)e);
    const uint32_t ng = edge_ng[e];
    ed[e] = make_uint2((uint32_t)(node_begin + i), (uint32_t)(line_off[ng >> 16] + (ng & 0xffffu)));
  }
}
// all ranks' messages -> node records in place, directed edges appended in rank order as int64 pairs;
// scal[0] = total edges, scal[1] = 1 when some rank had more edges than the message holds
__global__ void gather_unpack_kernel(const char *__restrict__ msgs, int world, const int64_t *__restrict__ rank_node_begin,
                                     int64_t max_nodes, int64_t cap_edges, int64_t msg_bytes,
                                     NodeRecord *__restrict__ nodes, int64_t *__restrict__ edges,
                                     int64_t *__restrict__ scal) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  int64_t ebase = 0;
  bool over = false;
  for (int r = 0; r < world; ++r) {
    const char *m = msgs + r * msg_bytes;
    int64_t ne = reinterpret_cast<const int64_t *>(m)[0];
    const int64_t nn = reinterpret_cast<const int64_t *>(m)[1];
    if (ne > cap_edges) { over = true; ne = cap_edges; }
    const uint4 *src = reinterpret_cast<const uint4 *>(m + 16);
    uint4 *dst = reinterpret_cast<uint4 *>(nodes + rank_node_begin[r]);
    const int64_t nv = nn * (int64_t)(sizeof(NodeRecord) / 16);
    for (int64_t i = tid; i < nv; i += nth) dst[i] = src[i];
    const uint2 *ed = reinterpret_cast<const uint2 *>(m + 16 + max_nodes * (int64_t)sizeof(NodeRecord));
    for (int64_t e = tid; e < ne; e += nth) {
      const uint2 v = ed[e];
      edges[2 * (ebase + e)] = (int64_t)v.x;
      edges[2 * (ebase + e) + 1] = (int64_t)v.y;
    }
    ebase += ne;
  }
  if (tid == 0) { scal[0] = ebase; scal[1] = over ? 1 : 0; }
}
void launch_gather_pack(const NodeRecord *nodes, int64_t node_begin, int64_t n_nodes, int64_t max_nodes,
                        const uint32_t *edge_off, const uint32_t *edge_ng, const int64_t *line_off, int64_t cap_edges,
                        char *msg, cudaStream_t s) {
  gather_pack_kernel<<<current_device_sms() * 4, 256, 0, s>>>(nodes, node_begin, n_nodes, max_nodes, edge_off, edge_ng, line_off, cap_edges, msg);
}
void launch_gather_unpack(const char *msgs, int world, const int64_t *rank_node_begin, int64_t max_nodes, int64_t cap_edges,
                          int64_t msg_bytes, NodeRecord *nodes, int64_t *edges, int64_t *scal, cudaStream_t s) {
  gather_unpack_kernel<<<current_device_sms() * 4, 256, 0, s>>>(msgs, world, rank_node_begin, max_nodes, cap_edges, msg_bytes, nodes, edges, scal);
}

// run_clustering edge weight (global_line_triangulator.cc:263-288): LineLinker3d::compute_score of the
// two best lines under set_to_spatial_merging().
__global__ void edge_weights_kernel(const __grid_constant__ EdgeParams p) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= p.n) return;
  const NodeRecord &a = p.nodes[p.edges[2 * e]];
  const NodeRecord &b = p.nodes[p.edges[2 * e + 1]];
  seg<vec3<double>> l1, l2;
  l1.s = mk3(a.line[0], a.line[1], a.line[2]); l1.e = mk3(a.line[3], a.line[4], a.line[5]);
  l2.s = mk3(b.line[0], b.line[1], b.line[2]); l2.e = mk3(b.line[3], b.line[4], b.line[5]);
  const double unc = smin(a.line[8], b.line[8]);
  p.weight[e] = linker_score<double, vec3<double>>(p.l3d, l1, l2, unc, true, a.line[6], a.line[7]);
}
void launch_edge_weights(const EdgeParams &p, cudaStream_t s) {
  if (p.n <= 0) return;
  const int grid = (int)((p.n + 127) / 128);
  edge_weights_kernel<<<grid, 128, 0, s>>>(p);
}

} // namespace lm
