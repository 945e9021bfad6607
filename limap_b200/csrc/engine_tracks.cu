// engine_tracks.cu — ComputeLineTracks: the track graph (graph_kernels.cu), the outer-edge peel, the greedy union-find
// and the aggregation of every track.
//
// Mirrors (file:line under /root/reference/src/limap/):
//   GlobalLineTriangulator::{run_clustering,build_tracks_from_clusters,ComputeLineTracks}
//       triangulation/global_line_triangulator.cc:168-359
//   merging::ComputeLineTrackLabelsGreedy      merging/merging.cc:18-103
//   merging::Aggregator::aggregate_line3d_list merging/aggregator.cc:53-101
#include "engine.cuh"
#include "graph_kernels.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <algorithm>
#include <cstdlib>
#include <iterator>
#include <queue>

// The total-least-squares direction of Aggregator::aggregate_line3d_list is the dominant eigenvector
// (merging/aggregator.cc:63-78; JacobiSVD V.col(0) up to sign).
void aggregate_items(const std::vector<AggItem> &it, int num_outliers, double out[7]) {
  const int n = (int)it.size();
  double min_unc = 1.7976931348623157e308;
  for (const AggItem &r : it) if (r.unc < min_unc) min_unc = r.unc;
  if (n < 4) { // aggregate_line3d_list_takebest (aggregator.cc:9-29); index 0 when no score > 0
    double best_score = 0.0;
    int best = -1;
    for (int i = 0; i < n; ++i) if (it[i].score > best_score) { best_score = it[i].score; best = i; }
    if (best < 0) best = 0;
    for (int k = 0; k < 6; ++k) out[k] = it[best].l[k];
    out[6] = min_unc;
    return;
  }
  double ctr[3] = {0, 0, 0};
  for (const AggItem &r : it) for (int k = 0; k < 3; ++k) { ctr[k] += r.l[k]; ctr[k] += r.l[3 + k]; }
  for (int k = 0; k < 3; ++k) ctr[k] = ctr[k] / (2 * n);
  double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (const AggItem &r : it)
    for (int e = 0; e < 2; ++e) {
      double p[3] = {r.l[3 * e] - ctr[0], r.l[3 * e + 1] - ctr[1], r.l[3 * e + 2] - ctr[2]};
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) S[a][b] += p[a] * p[b];
    }
  double V[3][3], ev[3], d[3];
  jacobi3(S, V, ev);
  int best = 0;
  if (ev[1] > ev[best]) best = 1;
  if (ev[2] > ev[best]) best = 2;
  for (int k = 0; k < 3; ++k) d[k] = V[k][best];
  double dn = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  for (int k = 0; k < 3; ++k) d[k] /= dn;
  std::vector<double> proj;
  for (const AggItem &r : it)
    for (int e = 0; e < 2; ++e)
      proj.push_back((r.l[3 * e] - ctr[0]) * d[0] + (r.l[3 * e + 1] - ctr[1]) * d[1] + (r.l[3 * e + 2] - ctr[2]) * d[2]);
  std::sort(proj.begin(), proj.end());
  const double a = proj[num_outliers], b = proj[2 * n - 1 - num_outliers];
  for (int k = 0; k < 3; ++k) { out[k] = ctr[k] + d[k] * a; out[3 + k] = ctr[k] + d[k] * b; }
  out[6] = min_unc;
}
static void aggregate(const std::vector<const lm::NodeRecord *> &recs, int num_outliers, double out[7]) {
  std::vector<AggItem> it(recs.size());
  for (size_t i = 0; i < recs.size(); ++i) it[i] = AggItem{recs[i]->line, recs[i]->line[8], recs[i]->score};
  aggregate_items(it, num_outliers, out);
}

size_t uf_root(size_t i, std::vector<int> &parent) { // base/graph.cc:157-166
  size_t r = i;
  while (parent[r] != -1) r = parent[r];
  while (parent[i] != -1) { size_t nx = parent[i]; parent[i] = (int)r; i = nx; } // full compression to the root
  return r;
}

// ComputeLineTrackLabelsGreedy (merging/merging.cc:18-103) after its sort: the union-find over the graph edges in the
// order given (each edge as idx1 << 32 | idx2) and the track numbering. image_of[i] in [0, n_images) is the image of
// node i. The reference's union_find_get_root compresses recursively (every node on the path points to the root
// afterwards); uf_root does the same iteratively. The union direction depends on the number of DISTINCT images of the
// two tracks (merging.cc:40-50): a bit set per root when there are few images (a union is an OR and a popcount), sorted
// id vectors otherwise. Returns the label of every node (-1: in no track of two or more nodes).
std::vector<int> greedy_track_labels(const std::vector<uint64_t> &order, const std::vector<int> &image_of, int n_images,
                                     int &n_tracks) {
  const size_t n_gn = image_of.size();
  std::vector<int> parent(n_gn, -1);
  const char *bs_env = getenv("LIMAP_B200_UF_BITSET_MAX_VIEWS"); // (tests force the vector path with 0)
  if (n_images <= (bs_env ? atoi(bs_env) : 1024)) {
    const size_t W = (size_t)(n_images + 63) / 64;
    std::vector<uint64_t> bits(n_gn * W, 0);
    std::vector<int> n_img(n_gn, 1);
    for (size_t i = 0; i < n_gn; ++i) bits[i * W + (size_t)image_of[i] / 64] = 1ull << (image_of[i] % 64);
    for (const uint64_t e : order) {
      size_t r1 = uf_root((size_t)(e >> 32), parent), r2 = uf_root((size_t)(e & 0xffffffffull), parent);
      if (r1 == r2) continue;
      size_t dst, srcn;
      if (n_img[r1] < n_img[r2]) { parent[r1] = (int)r2; dst = r2; srcn = r1; }
      else { parent[r2] = (int)r1; dst = r1; srcn = r2; }
      int cnt = 0;
      for (size_t w = 0; w < W; ++w) {
        bits[dst * W + w] |= bits[srcn * W + w];
        cnt += __builtin_popcountll(bits[dst * W + w]);
      }
      n_img[dst] = cnt;
    }
  } else {
    std::vector<std::vector<int>> images(n_gn); // sorted distinct image ids of each root's track
    for (size_t i = 0; i < n_gn; ++i) images[i].push_back(image_of[i]);
    for (const uint64_t e : order) {
      size_t r1 = uf_root((size_t)(e >> 32), parent), r2 = uf_root((size_t)(e & 0xffffffffull), parent);
      if (r1 == r2) continue;
      size_t dst, srcn;
      if (images[r1].size() < images[r2].size()) { parent[r1] = (int)r2; dst = r2; srcn = r1; }
      else { parent[r2] = (int)r1; dst = r1; srcn = r2; }
      std::vector<int> merged;
      std::set_union(images[dst].begin(), images[dst].end(), images[srcn].begin(), images[srcn].end(),
                     std::back_inserter(merged));
      images[dst].swap(merged);
      std::vector<int>().swap(images[srcn]);
    }
  }
  std::vector<int> label(n_gn, -1);
  n_tracks = 0;
  for (size_t i = 0; i < n_gn; ++i) {
    if (parent[i] == -1) continue;
    size_t pi = parent[i];
    if (parent[pi] == -1 && label[pi] == -1) label[pi] = n_tracks++;
  }
  for (size_t i = 0; i < n_gn; ++i) {
    if (parent[i] == -1) continue;
    label[i] = label[uf_root(i, parent)];
  }
  return label;
}

int sort_greedy_order(DevBuf &scratch, DevBuf &nodes, DevBuf &nodes_alt, DevBuf &score, DevBuf &score_alt, int n,
                      cudaStream_t s, const uint64_t *&out) {
  cub::DoubleBuffer<uint64_t> k(nodes.as<uint64_t>(), nodes_alt.as<uint64_t>());
  cub::DoubleBuffer<uint64_t> v(score.as<uint64_t>(), score_alt.as<uint64_t>());
  CU(cub_call(scratch, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, k, v, n, 0, 64, s); }));
  cub::DoubleBuffer<uint64_t> k2(v.Current(), v.Alternate());
  cub::DoubleBuffer<uint64_t> v2(k.Current(), k.Alternate());
  CU(cub_call(scratch, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, k2, v2, n, 0, 64, s); }));
  out = v2.Current();
  return LM_OK;
}

// The track graph on the device (graph_kernels.cu): from the nk undirected keys (min << 32 | max) of the valid
// connections in c->d_edge_keys (duplicates allowed) to the graph nodes in FindOrCreateNode order and the edges in the
// order ComputeLineTrackLabelsGreedy visits them, each edge as (idx0 << 32 | idx1). Two small read-backs; the
// union-find that follows is sequential by definition.
static int graph_on_device(lm_ctx *c, int64_t nk, std::vector<int64_t> &gnode, std::vector<uint64_t> &order) {
  cudaStream_t s = c->stream;
  gnode.clear();
  order.clear();
  if (nk <= 0) return LM_OK;
  if (nk >= (int64_t)1 << 30) return fail(LM_ERR_INVALID, "too many valid connections for the 32-bit positions of the graph build");
  auto sort_keys = [&](DevBuf &a, DevBuf &b, int64_t n, uint64_t *&out) -> int {
    cub::DoubleBuffer<uint64_t> dk(a.as<uint64_t>(), b.as<uint64_t>());
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &bytes) { return cub::DeviceRadixSort::SortKeys(t, bytes, dk, (int)n, 0, 64, s); }));
    out = dk.Current();
    return LM_OK;
  };
  auto scan_u32 = [&](const uint32_t *in, uint32_t *out, int64_t n) -> int {
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, in, out, (int)n, s); }));
    return LM_OK;
  };
  int rc;
  // undirected edge set in std::set order (:243-261)
  CU(c->d_edge_keys2.ensure(8 * nk + 8));
  uint64_t *sorted = nullptr;
  if ((rc = sort_keys(c->d_edge_keys, c->d_edge_keys2, nk, sorted))) return rc;
  uint64_t *ukeys = (sorted == c->d_edge_keys.as<uint64_t>()) ? c->d_edge_keys2.as<uint64_t>() : c->d_edge_keys.as<uint64_t>();
  CU(c->d_edge_cnt.ensure(16));
  CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) {
    return cub::DeviceSelect::Unique(t, b, sorted, ukeys, c->d_edge_cnt.as<int64_t>(), (int)nk, s);
  }));
  int64_t nu = 0;
  CU(cudaMemcpyAsync(&nu, c->d_edge_cnt.p, 8, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  // 3d score of every undirected edge (:263-288)
  CU(c->d_edges2.ensure(16 * nu));
  CU(c->d_edge_w.ensure(8 * nu));
  lm::launch_keys_to_pairs(ukeys, nu, c->d_edges2.as<int64_t>(), s);
  lm::EdgeParams ep;
  ep.nodes = c->d_nodes.as<lm::NodeRecord>();
  ep.edges = c->d_edges2.as<int64_t>();
  ep.weight = c->d_edge_w.as<double>();
  ep.n = nu;
  ep.l3d = to_dev<double>(spatial_merging(c->cfg.linker3d));
  lm::launch_edge_weights(ep, s);
  // zero-score edges dropped, order kept (:284-285)
  CU(c->d_g_flag.ensure(4 * (2 * nu + 2)));
  CU(c->d_g_pos.ensure(4 * (2 * nu + 2)));
  CU(c->d_g_kc.ensure(8 * nu + 8));
  CU(c->d_g_wc.ensure(8 * nu + 8));
  uint32_t *flag = c->d_g_flag.as<uint32_t>(), *pos = c->d_g_pos.as<uint32_t>();
  lm::launch_nonzero_flags(c->d_edge_w.as<double>(), nu, flag, s);
  CU(cudaMemsetAsync(flag + nu, 0, 4, s)); // the scan of n + 1 flags ends with the total
  if ((rc = scan_u32(flag, pos, nu + 1))) return rc;
  lm::launch_compact_weighted_edges(ukeys, c->d_edge_w.as<double>(), flag, pos, nu, c->d_g_kc.as<uint64_t>(),
                                    c->d_g_wc.as<double>(), s);
  uint32_t n2u = 0;
  CU(cudaMemcpyAsync(&n2u, pos + nu, 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  const int64_t n2 = n2u;
  c->stats.n_kernel_launches += 12;
  if (n2 == 0) return LM_OK;
  // Graph::FindOrCreateNode numbering: rank of a node's first appearance in u0 v0 u1 v1 ...
  const int64_t m = 2 * n2;
  CU(c->d_g_occ.ensure(8 * m));
  CU(c->d_g_occ2.ensure(8 * m));
  lm::launch_occurrence_keys(c->d_g_kc.as<uint64_t>(), n2, c->d_g_occ.as<uint64_t>(), s);
  uint64_t *occ = nullptr;
  if ((rc = sort_keys(c->d_g_occ, c->d_g_occ2, m, occ))) return rc;
  lm::launch_occurrence_heads(occ, m, flag, s);
  CU(cudaMemsetAsync(flag + m, 0, 4, s));
  if ((rc = scan_u32(flag, pos, m + 1))) return rc;
  uint32_t ngu = 0;
  CU(cudaMemcpyAsync(&ngu, pos + m, 4, cudaMemcpyDeviceToHost, s));
  CU(c->d_g_hk.ensure(8 * m));
  CU(c->d_g_hk2.ensure(8 * m));
  lm::launch_head_keys(occ, flag, pos, m, c->d_g_hk.as<uint64_t>(), s);
  CU(cudaStreamSynchronize(s));
  const int64_t ng = ngu;
  uint64_t *hk = nullptr;
  if ((rc = sort_keys(c->d_g_hk, c->d_g_hk2, ng, hk))) return rc;
  CU(c->d_g_gidx.ensure(4 * (size_t)std::max<int64_t>(c->n_nodes, 1)));
  CU(c->d_g_gnode.ensure(4 * ng));
  lm::launch_graph_index(hk, ng, c->d_g_gidx.as<int32_t>(), c->d_g_gnode.as<int32_t>(), s);
  // edges in descending (score, idx0, idx1) order: stable LSD, nodes first, score second
  CU(c->d_g_k1.ensure(8 * n2)); CU(c->d_g_k1b.ensure(8 * n2));
  CU(c->d_g_k2.ensure(8 * n2)); CU(c->d_g_k2b.ensure(8 * n2));
  lm::launch_edge_order_keys(c->d_g_kc.as<uint64_t>(), c->d_g_wc.as<double>(), c->d_g_gidx.as<int32_t>(), n2,
                             c->d_g_k1.as<uint64_t>(), c->d_g_k2.as<uint64_t>(), s);
  const uint64_t *final_nodes = nullptr;
  if ((rc = sort_greedy_order(c->d_sort_tmp, c->d_g_k1, c->d_g_k1b, c->d_g_k2, c->d_g_k2b, (int)n2, s, final_nodes)))
    return rc;
  std::vector<int32_t> gn32((size_t)ng);
  order.resize((size_t)n2);
  CU(cudaMemcpyAsync(gn32.data(), c->d_g_gnode.p, 4 * ng, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(order.data(), final_nodes, 8 * n2, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  c->stats.n_kernel_launches += 16;
  gnode.assign(gn32.begin(), gn32.end());
  for (uint64_t &o : order) o = ~o;
  return LM_OK;
}

extern "C" {

int64_t lm_tri_build_tracks(lm_ctx *c, int64_t *n_support_total) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int rc = ensure_ran(c);
  if (rc) return rc;
  CU(cudaSetDevice(c->device));
  if ((rc = collect_edges(c))) return rc;
  if ((rc = fetch_nodes(c))) return rc;
  cudaStream_t s = c->stream;
  const int64_t ne = c->n_edges_dev;
  c->tracks.clear();
  if (n_support_total) *n_support_total = 0;
  if (ne == 0) return 0;
  // The undirected keys (min << 32 | max) of the valid connections go to d_edge_keys; d_edges stays as collected, since
  // later calls and lm_tri_export_edges read it. filterNodeByNumOuterEdges keeps every node when min_num_outer_edges <= 0.
  int64_t nk = ne;
  const int min_outer = c->cfg.min_num_outer_edges;
  if (min_outer <= 0) {
    CU(c->d_edge_keys.ensure(8 * ne));
    lm::launch_undirected_keys(c->d_edges.as<int64_t>(), ne, c->d_edge_keys.as<uint64_t>(), s);
  } else {
    std::vector<int64_t> h_edges(2 * ne);
    CU(cudaMemcpyAsync(h_edges.data(), c->d_edges.p, 16 * ne, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    // filterNodeByNumOuterEdges (global_line_triangulator.cc:168-232)
    std::vector<char> flag(c->n_nodes, 1);
    std::vector<int> counter(c->n_nodes, 0);
    std::vector<int64_t> pstart(c->n_nodes + 1, 0);
    for (int64_t e = 0; e < ne; ++e) { counter[h_edges[2 * e]]++; pstart[h_edges[2 * e + 1] + 1]++; }
    for (int64_t n = 0; n < c->n_nodes; ++n) pstart[n + 1] += pstart[n];
    std::vector<int64_t> parents(ne), fill(pstart.begin(), pstart.end() - 1);
    for (int64_t e = 0; e < ne; ++e) parents[fill[h_edges[2 * e + 1]]++] = h_edges[2 * e];
    std::queue<int64_t> q;
    for (int64_t n = 0; n < c->n_nodes; ++n)
      if (counter[n] < min_outer) { flag[n] = 0; q.push(n); }
    while (!q.empty()) {
      int64_t n = q.front(); q.pop();
      for (int64_t k = pstart[n]; k < pstart[n + 1]; ++k) {
        int64_t pn = parents[k];
        if (!flag[pn]) continue;
        if (--counter[pn] < min_outer) { flag[pn] = 0; q.push(pn); }
      }
    }
    std::vector<uint64_t> keys;
    keys.reserve(ne);
    for (int64_t e = 0; e < ne; ++e) {
      int64_t a = h_edges[2 * e], b = h_edges[2 * e + 1];
      if (!flag[a] || !flag[b]) continue;
      if (a > b) std::swap(a, b);
      keys.push_back(((uint64_t)a << 32) | (uint64_t)b);
    }
    nk = (int64_t)keys.size();
    CU(c->d_edge_keys.ensure(8 * nk));
    CU(cudaMemcpyAsync(c->d_edge_keys.p, keys.data(), 8 * nk, cudaMemcpyHostToDevice, s)); // pageable: keys is read on return
  }
  std::vector<int64_t> gnode;
  std::vector<uint64_t> order; // (idx0 << 32 | idx1) of every graph edge, in the order the greedy labelling visits them
  if ((rc = graph_on_device(c, nk, gnode, order))) return rc;
  const size_t n_gn = gnode.size();
  if (n_gn == 0) return 0;
  // view index of a graph node: binary search in line_off
  std::vector<int> view_of(n_gn);
  for (size_t i = 0; i < n_gn; ++i)
    view_of[i] = (int)(std::upper_bound(c->line_off.begin(), c->line_off.end(), gnode[i]) - c->line_off.begin()) - 1;
  int n_tracks = 0;
  const std::vector<int> label = greedy_track_labels(order, view_of, c->V, n_tracks);
  // build_tracks_from_clusters (global_line_triangulator.cc:293-351)
  c->tracks.assign(n_tracks, Track());
  int64_t support = 0;
  for (size_t i = 0; i < n_gn; ++i) {
    if (label[i] < 0) continue;
    Track &t = c->tracks[label[i]];
    const int v = view_of[i];
    t.img.push_back(c->img_ids[v]);
    t.line.push_back((int)(gnode[i] - c->line_off[v]));
    t.node.push_back((int)i);
    t.gid.push_back(gnode[i]);
    ++support;
  }
  for (Track &t : c->tracks) {
    std::vector<const lm::NodeRecord *> recs;
    for (int64_t g : t.gid) recs.push_back(&c->h_nodes[g]);
    aggregate(recs, c->cfg.num_outliers_aggregator, t.agg);
  }
  if (n_support_total) *n_support_total = support;
  return n_tracks;
}

int lm_tri_get_tracks(lm_ctx *c, int64_t *track_off, int32_t *img_ids, int32_t *line_ids, int32_t *node_ids,
                      double *node_line3d, double *track_line) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int64_t n = 0;
  for (size_t t = 0; t < c->tracks.size(); ++t) {
    const Track &tr = c->tracks[t];
    track_off[t] = n;
    for (size_t k = 0; k < tr.img.size(); ++k, ++n) {
      img_ids[n] = tr.img[k];
      line_ids[n] = tr.line[k];
      node_ids[n] = tr.node[k];
      const lm::NodeRecord &r = c->h_nodes[tr.gid[k]];
      for (int q = 0; q < 9; ++q) node_line3d[10 * n + q] = r.line[q];
      node_line3d[10 * n + 9] = r.score;
    }
    for (int q = 0; q < 7; ++q) track_line[7 * t + q] = tr.agg[q];
  }
  track_off[c->tracks.size()] = n;
  return LM_OK;
}

int lm_aggregate_lines(int64_t T, const int64_t *off, const double *lines, const double *scores, int32_t num_outliers,
                       double *out_line) {
  if (T < 0 || !off || !out_line) return fail(LM_ERR_INVALID, "NULL argument");
  if (num_outliers < 0) return fail(LM_ERR_INVALID, "num_outliers must be >= 0");
  std::vector<AggItem> it;
  for (int64_t t = 0; t < T; ++t) {
    const int64_t n = off[t + 1] - off[t];
    double *o = out_line + 7 * t;
    if (n <= 0) { memset(o, 0, 7 * sizeof(double)); continue; }
    if (n >= 4 && 2 * n - 1 - num_outliers < num_outliers) return fail(LM_ERR_INVALID, "num_outliers too large for a group");
    it.resize(n);
    for (int64_t k = 0; k < n; ++k) it[k] = AggItem{lines + 7 * (off[t] + k), lines[7 * (off[t] + k) + 6], scores[off[t] + k]};
    aggregate_items(it, num_outliers, o);
  }
  return LM_OK;
}

} // extern "C"
