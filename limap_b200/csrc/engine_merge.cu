// engine_merge.cu — track filters, remerge and fit-and-merge (merge_kernels.cu).
#include "engine.cuh"
#include "merge_kernels.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <chrono>
#include <cstdlib>

// The fp32 gates of the remerge and the fit pair kernel (lm::RemergeParams, lm::FitPairParams): necessary conditions of
// the linker test under set_to_spatial_merging (DESIGN.md §3.5). And the origin of the ball gate's fp32 coordinates,
// which keeps them small: the mean of the finite midpoints of the n lines, line i starting at lines[stride * i].
template <typename Params>
static void merge_gates(const lm_linker_config &l3, const double *lines, int64_t n, int stride, Params &p, double origin[3]) {
  p.use_gate = (l3.th_angle > 0.0 && l3.th_angle < 89.0) ? 1 : 0;
  p.cos_gate = p.use_gate ? (float)(std::cos(l3.th_angle * 3.14159265358979323846 / 180.0) - 1e-5) : -1.0f;
  p.use_ball = (l3.use_innerseg && l3.th_innerseg >= 0.0 && l3.score_th > 0.0 && l3.score_th < 1.0) ? 1 : 0;
  origin[0] = origin[1] = origin[2] = 0;
  int64_t nfin = 0;
  for (int64_t t = 0; t < n; ++t) {
    const double *l = lines + stride * t;
    const double m[3] = {0.5 * (l[0] + l[3]), 0.5 * (l[1] + l[4]), 0.5 * (l[2] + l[5])};
    if (std::isfinite(m[0]) && std::isfinite(m[1]) && std::isfinite(m[2])) { origin[0] += m[0]; origin[1] += m[1]; origin[2] += m[2]; ++nfin; }
  }
  if (nfin) for (int k = 0; k < 3; ++k) origin[k] /= (double)nfin;
}

extern "C" {

// ---- track filters + remerge (merging/merging_utils.cc, merging/merging.cc:513-645) -------------------
int lm_tracks_support_flags(lm_ctx *c, int32_t n_views, const int32_t *model_ids, const double *kvec, const double *qvec,
                            const double *tvec, int64_t T, const int64_t *sup_off, const int32_t *sup_view,
                            const double *segs, const double *track_line, const lm_filter_config *cfg,
                            uint8_t *out_flags) {
  if (!c || !cfg || !sup_off || !kvec || !qvec || !tvec) return fail(LM_ERR_INVALID, "NULL argument");
  if (T < 0 || n_views <= 0) return fail(LM_ERR_INVALID, "bad sizes");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const int64_t n = sup_off[T];
  if (n == 0) return LM_OK;
  if (!sup_view || !segs || !track_line || !out_flags) return fail(LM_ERR_INVALID, "NULL argument");
  for (int64_t k = 0; k < n; ++k)
    if (sup_view[k] < 0 || sup_view[k] >= n_views) return fail(LM_ERR_INVALID, "support view index out of range");
  std::vector<lm::ViewD> views(n_views);
  for (int v = 0; v < n_views; ++v) {
    const int mid = model_ids ? model_ids[v] : 1;
    if (mid != 0 && mid != 1) return fail(LM_ERR_INVALID, "only SIMPLE_PINHOLE / PINHOLE are legal on this path");
    make_view(mid, kvec + 4 * v, qvec + 4 * v, tvec + 3 * v, views[v]);
  }
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t o_v = take(sizeof(lm::ViewD) * n_views), o_s = take(32 * n), o_so = take(8 * (T + 1)), o_sv = take(4 * n),
               o_tl = take(48 * T);
  CU(c->d_mg_in.ensure(off + 256));
  CU(c->d_mg_out.ensure(n + 256));
  char *in = c->d_mg_in.as<char>();
  CU(cudaEventRecord(c->ev0, s));
  CU(cudaMemcpyAsync(in + o_v, views.data(), sizeof(lm::ViewD) * n_views, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_s, segs, 32 * n, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_so, sup_off, 8 * (T + 1), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_sv, sup_view, 4 * n, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_tl, track_line, 48 * T, cudaMemcpyHostToDevice, s));
  lm::SupportParams p;
  p.views = reinterpret_cast<const lm::ViewD *>(in + o_v);
  p.sup_off = reinterpret_cast<const int64_t *>(in + o_so);
  p.sup_view = reinterpret_cast<const int32_t *>(in + o_sv);
  p.segs = reinterpret_cast<const double4 *>(in + o_s);
  p.track_line = reinterpret_cast<const double *>(in + o_tl);
  p.T = T; p.S = n;
  p.th_angular2d = cfg->th_angular_2d; p.th_perp2d = cfg->th_perp_2d;
  p.th_sv_angular3d = cfg->th_sv_angular_3d; p.th_overlap = cfg->th_overlap;
  p.flags = c->d_mg_out.as<uint8_t>();
  CU(cudaEventRecord(c->evk0, s));
  lm::launch_support_flags(p, s);
  CU(cudaEventRecord(c->evk1, s));
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out_flags, p.flags, n, cudaMemcpyDeviceToHost, s));
  CU(cudaEventRecord(c->ev1, s));
  CU(cudaStreamSynchronize(s));
  float ms = 0, msk = 0;
  CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  CU(cudaEventElapsedTime(&msk, c->evk0, c->evk1));
  c->mg_stats.n_supports = n;
  c->mg_stats.last_flags_ms = ms;
  c->mg_stats.last_flags_kernel_ms = msk;
  c->mg_stats.n_kernel_launches += 1;
  return LM_OK;
}

int64_t lm_remerge_labels(lm_ctx *c, int64_t T, const double *track_line, const uint8_t *active,
                          const lm_linker_config *linker3d, int32_t *out_labels, int64_t *out_n_edges) {
  if (!c || !linker3d) return fail(LM_ERR_INVALID, "NULL argument");
  if (T < 0 || T >= ((int64_t)1 << 31)) return fail(LM_ERR_INVALID, "bad track count");
  if (out_n_edges) *out_n_edges = 0;
  if (T == 0) return 0;
  if (!track_line || !active || !out_labels) return fail(LM_ERR_INVALID, "NULL argument");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const lm_linker_config l3 = spatial_merging(*linker3d);
  int64_t n_active = 0;
  for (int64_t t = 0; t < T; ++t) n_active += active[t] ? 1 : 0;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t o_l = take(56 * T), o_d = take(16 * T), o_b = take(16 * T), o_a = take(T), o_c = take(16);
  CU(c->d_mg_in.ensure(off + 256));
  char *in = c->d_mg_in.as<char>();
  CU(cudaEventRecord(c->ev0, s));
  CU(cudaMemcpyAsync(in + o_l, track_line, 56 * T, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_a, active, T, cudaMemcpyHostToDevice, s));
  lm::RemergeParams p;
  p.lines = reinterpret_cast<const double *>(in + o_l);
  p.dirf = reinterpret_cast<const float4 *>(in + o_d);
  p.ballf = reinterpret_cast<const float4 *>(in + o_b);
  p.active = reinterpret_cast<const uint8_t *>(in + o_a);
  p.T = T;
  p.all_active = (n_active == T) ? 1 : 0;
  p.lk = to_dev<double>(l3);
  p.counter = reinterpret_cast<unsigned long long *>(in + o_c);
  double origin[3];
  merge_gates(l3, track_line, T, 7, p, origin);
  lm::launch_remerge_dirs(p.lines, T, origin, l3.th_innerseg, reinterpret_cast<float4 *>(in + o_d),
                          reinterpret_cast<float4 *>(in + o_b), s);
  unsigned long long cap = (unsigned long long)std::max<int64_t>(4 * T, 1 << 16);
  unsigned long long cnt[2] = {0, 0};
  float msk = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
    CU(c->d_mg_edges.ensure(8 * cap));
    p.edges = c->d_mg_edges.as<uint32_t>();
    p.capacity = cap;
    lm::launch_zero_words(reinterpret_cast<unsigned int *>(in + o_c), 4, s);
    CU(cudaEventRecord(c->evk0, s));
    if (n_active > 0) lm::launch_remerge_pairs(p, s);
    CU(cudaEventRecord(c->evk1, s));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(cnt, p.counter, 16, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&msk, c->evk0, c->evk1));
    c->mg_stats.n_kernel_launches += 3;
    if (cnt[0] <= cap) break;
    cap = cnt[0]; // the list overflowed: run again with the exact size
  }
  const int64_t ne = (int64_t)cnt[0];
  std::vector<uint32_t> h_edges(2 * std::max<int64_t>(ne, 1));
  if (ne) CU(cudaMemcpyAsync(h_edges.data(), p.edges, 8 * ne, cudaMemcpyDeviceToHost, s));
  CU(cudaEventRecord(c->ev1, s));
  CU(cudaStreamSynchronize(s));
  float ms = 0;
  CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  // std::set<pair> iteration order = lexicographic (merging.cc:558-560)
  std::vector<uint64_t> keys(ne);
  for (int64_t e = 0; e < ne; ++e) keys[e] = ((uint64_t)h_edges[2 * e] << 32) | h_edges[2 * e + 1];
  std::sort(keys.begin(), keys.end());
  // union-find with the group-size heuristic (merging.cc:562-589)
  std::vector<int> parent(T, -1);
  std::vector<int64_t> gsize(T, 1);
  for (int64_t e = 0; e < ne; ++e) {
    const size_t r1 = uf_root((size_t)(keys[e] >> 32), parent), r2 = uf_root((size_t)(keys[e] & 0xffffffffu), parent);
    if (r1 == r2) continue;
    if (gsize[r1] < gsize[r2]) { parent[r1] = (int)r2; gsize[r2] += gsize[r1]; gsize[r1] = 0; }
    else { parent[r2] = (int)r1; gsize[r1] += gsize[r2]; gsize[r2] = 0; }
  }
  int64_t n_groups = 0;
  for (int64_t t = 0; t < T; ++t) out_labels[t] = (parent[t] == -1) ? (int32_t)(n_groups++) : -1;
  for (int64_t t = 0; t < T; ++t)
    if (out_labels[t] == -1) out_labels[t] = out_labels[uf_root((size_t)t, parent)];
  if (out_n_edges) *out_n_edges = ne;
  c->mg_stats.n_tracks = T;
  c->mg_stats.n_pairs_gated = (int64_t)cnt[1];
  c->mg_stats.n_edges = ne;
  c->mg_stats.last_remerge_ms = ms;
  c->mg_stats.last_remerge_kernel_ms = msk;
  return n_groups;
}

int lm_merge_get_stats(lm_ctx *c, lm_merge_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->mg_stats;
  return LM_OK;
}

// ---- MergeToLineTracks (merging/merging.cc:347-511) -------------------------------------------------------------------
// Device: per-line prep (uncertainty, bit-exact length, node flag, gate records), the pair kernel over 256 x 256 tiles of
// every (image, self) and (image, neighbour slot) block, a radix sort of the passing pairs by insertion key (the graph's
// edge list) and two stable radix sorts by (sim, node1, node2) descending (the greedy order). Host: the union-find, the
// tracks and their aggregation, as in lm_tri_build_tracks.
int64_t lm_merge_fits_build(lm_ctx *c, int32_t n_views, const int32_t *img_ids, const int32_t *model_ids,
                            const double *kvec, const double *qvec, const double *tvec, const int64_t *line_off,
                            const double *segs, const double *lines3d, const int64_t *ng_off, const int32_t *ng_ids,
                            double var2d, const lm_linker_config *linker2d, const lm_linker_config *linker3d,
                            int64_t *out_counts) {
  const auto t_begin = std::chrono::steady_clock::now();
  if (!c || !img_ids || !kvec || !qvec || !tvec || !line_off || !ng_off || !linker2d || !linker3d || !out_counts)
    return fail(LM_ERR_INVALID, "NULL argument");
  if (n_views <= 0 || n_views > 65535) return fail(LM_ERR_INVALID, "n_views must be in [1, 65535]");
  if (!std::isfinite(var2d)) return fail(LM_ERR_INVALID, "var2d must be finite");
  std::unordered_map<int, int> view_of;
  for (int v = 0; v < n_views; ++v) {
    if (v > 0 && img_ids[v] <= img_ids[v - 1]) return fail(LM_ERR_INVALID, "image ids must be strictly ascending");
    view_of[img_ids[v]] = v;
    const int mid = model_ids ? model_ids[v] : 1;
    if (mid != 0 && mid != 1) return fail(LM_ERR_INVALID, "only SIMPLE_PINHOLE / PINHOLE are legal on this path");
    if (line_off[v + 1] < line_off[v] || line_off[v + 1] - line_off[v] > 65535)
      return fail(LM_ERR_INVALID, "lines per image must be in [0, 65535]");
    if (ng_off[v + 1] < ng_off[v] || ng_off[v + 1] - ng_off[v] > 32767)
      return fail(LM_ERR_INVALID, "neighbours per image must be in [0, 32767]");
  }
  if (line_off[0] != 0 || ng_off[0] != 0) return fail(LM_ERR_INVALID, "line_off[0] and ng_off[0] must be 0");
  const int64_t n = line_off[n_views];
  if (n >= ((int64_t)1 << 31)) return fail(LM_ERR_INVALID, "too many lines");
  if (n > 0 && (!segs || !lines3d)) return fail(LM_ERR_INVALID, "NULL argument");
  for (int64_t k = 0; k < 6 * n; ++k)
    if (!std::isfinite(lines3d[k])) return fail(LM_ERR_INVALID, "3D fits must be finite");
  std::vector<int32_t> ng_view(ng_off[n_views]);
  for (int64_t k = 0; k < ng_off[n_views]; ++k) {
    auto it = view_of.find(ng_ids[k]);
    if (it == view_of.end()) return fail(LM_ERR_INVALID, "neighbour " + std::to_string(ng_ids[k]) + " is not an image");
    ng_view[k] = it->second;
  }
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  c->fm = lm_ctx::FitMerge();
  c->fm_stats = lm_fit_merge_stats();
  c->fm_stats.n_lines = n;
  const lm_linker_config l3 = spatial_merging(*linker3d);
  // views and tiles
  std::vector<lm::FitView> views(n_views);
  for (int v = 0; v < n_views; ++v) {
    const M3h R = quat_to_R(qvec + 4 * v);
    lm::FitView &w = views[v];
    for (int k = 0; k < 9; ++k) w.R[k] = R.m[k];
    for (int k = 0; k < 3; ++k) w.t[k] = tvec[3 * v + k];
    const double *kv = kvec + 4 * v;
    const bool simple = model_ids && model_ids[v] == 0;
    w.fx = kv[0]; w.fy = simple ? kv[0] : kv[1]; w.cx = kv[2]; w.cy = kv[3];
    w.f = simple ? kv[0] : (kv[0] + kv[1]) / 2.0; // Camera::uncertainty (camera.cc:228-242)
  }
  std::vector<lm::FitTile> tiles;
  auto n_tiles_of = [&](int v) { return (int)((line_off[v + 1] - line_off[v] + 255) / 256); };
  for (int v = 0; v < n_views; ++v) {
    const int na = n_tiles_of(v);
    for (int ta = 0; ta < na; ++ta)
      for (int tb = ta; tb < na; ++tb) tiles.push_back(lm::FitTile{v, v, -1, ta << 16 | tb});
    for (int64_t k = ng_off[v]; k < ng_off[v + 1]; ++k) {
      const int u = ng_view[k], nb = n_tiles_of(u);
      for (int ta = 0; ta < na; ++ta)
        for (int tb = 0; tb < nb; ++tb) tiles.push_back(lm::FitTile{v, u, (int)(k - ng_off[v]), ta << 16 | tb});
    }
  }
  if (tiles.size() >= ((size_t)1 << 31)) return fail(LM_ERR_INVALID, "too many tiles for one grid");
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t o_v = take(sizeof(lm::FitView) * n_views), o_lo = take(8 * (n_views + 1)), o_id = take(4 * n_views),
               o_s = take(32 * n), o_l = take(48 * n), o_t = take(sizeof(lm::FitTile) * tiles.size());
  CU(c->d_fm_in.ensure(off + 256));
  char *in = c->d_fm_in.as<char>();
  off = 0;
  const size_t o_r = take(56 * n), o_len = take(8 * n), o_nz = take(n), o_d = take(16 * n), o_b = take(16 * n), o_c = take(32);
  CU(c->d_fm_work.ensure(off + 256));
  char *wk = c->d_fm_work.as<char>();
  CU(cudaMemcpyAsync(in + o_v, views.data(), sizeof(lm::FitView) * n_views, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_lo, line_off, 8 * (n_views + 1), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_id, img_ids, 4 * n_views, cudaMemcpyHostToDevice, s));
  if (n) {
    CU(cudaMemcpyAsync(in + o_s, segs, 32 * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(in + o_l, lines3d, 48 * n, cudaMemcpyHostToDevice, s));
  }
  if (!tiles.empty())
    CU(cudaMemcpyAsync(in + o_t, tiles.data(), sizeof(lm::FitTile) * tiles.size(), cudaMemcpyHostToDevice, s));
  lm::FitPairParams p;
  double origin[3];
  merge_gates(l3, lines3d, n, 6, p, origin); // (every fit is finite: see above)
  lm::FitPrepParams pp;
  pp.views = reinterpret_cast<const lm::FitView *>(in + o_v);
  pp.line_off = reinterpret_cast<const int64_t *>(in + o_lo);
  pp.lines3d = reinterpret_cast<const double *>(in + o_l);
  pp.V = n_views; pp.n = n; pp.var2d = var2d;
  pp.ox = origin[0]; pp.oy = origin[1]; pp.oz = origin[2]; pp.th_innerseg = l3.th_innerseg;
  pp.rec = reinterpret_cast<double *>(wk + o_r);
  pp.len = reinterpret_cast<double *>(wk + o_len);
  pp.nonzero = reinterpret_cast<uint8_t *>(wk + o_nz);
  pp.dirf = reinterpret_cast<float4 *>(wk + o_d);
  pp.ballf = reinterpret_cast<float4 *>(wk + o_b);
  lm::launch_fit_prep(pp, s);
  p.views = pp.views; p.line_off = pp.line_off;
  p.img_ids = reinterpret_cast<const int32_t *>(in + o_id);
  p.segs = reinterpret_cast<const double4 *>(in + o_s);
  p.rec = pp.rec; p.nonzero = pp.nonzero; p.dirf = pp.dirf; p.ballf = pp.ballf;
  p.tiles = reinterpret_cast<const lm::FitTile *>(in + o_t);
  p.lk3 = to_dev<double>(l3);
  p.lk2 = to_dev<double>(*linker2d);
  p.counter = reinterpret_cast<unsigned long long *>(wk + o_c);
  const char *cap_env = getenv("LIMAP_B200_FIT_EDGE_CAPACITY"); // (tests force the overflow retry with a small value)
  unsigned long long cap = cap_env ? (unsigned long long)std::max(1, atoi(cap_env))
                                   : (unsigned long long)std::max<int64_t>(16 * n, 1 << 20);
  unsigned long long cnt[3] = {0, 0, 0};
  float msk = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
    CU(c->d_fm_keys.ensure(8 * cap));
    CU(c->d_fm_pairs.ensure(8 * cap));
    p.keys = c->d_fm_keys.as<unsigned long long>();
    p.pairs = c->d_fm_pairs.as<unsigned long long>();
    p.capacity = cap;
    lm::launch_zero_words(p.counter, 6, s);
    CU(cudaEventRecord(c->evk0, s));
    lm::launch_fit_pairs(p, (int64_t)tiles.size(), s);
    CU(cudaEventRecord(c->evk1, s));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(cnt, p.counter, 24, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&msk, c->evk0, c->evk1));
    c->mg_stats.n_kernel_launches += attempt == 0 ? 3 : 2;
    if (cnt[0] <= cap) break;
    cap = cnt[0]; // the list overflowed: run again with the exact size
    ++c->fm_stats.n_retries;
  }
  const int64_t ne = (int64_t)cnt[0];
  if (ne >= ((int64_t)1 << 31)) return fail(LM_ERR_INVALID, "too many graph edges for the 32-bit sort sizes");
  std::vector<double> len(n), rec(7 * n);
  std::vector<uint64_t> ins_pairs(ne), order(ne);
  c->fm.sim.resize(ne);
  if (ne > 0) {
    CU(c->d_fm_keys2.ensure(8 * ne)); CU(c->d_fm_pairs2.ensure(8 * ne));
    CU(c->d_fm_bn.ensure(8 * ne)); CU(c->d_fm_bn2.ensure(8 * ne));
    CU(c->d_fm_bs.ensure(8 * ne)); CU(c->d_fm_bs2.ensure(8 * ne));
    CU(c->d_fm_sim.ensure(8 * ne));
    // insertion order: the keys are unique (merging.cc:466-477)
    cub::DoubleBuffer<unsigned long long> k1(c->d_fm_keys.as<unsigned long long>(), c->d_fm_keys2.as<unsigned long long>());
    cub::DoubleBuffer<unsigned long long> v1(c->d_fm_pairs.as<unsigned long long>(), c->d_fm_pairs2.as<unsigned long long>());
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, k1, v1, (int)ne, 0, 64, s); }));
    const unsigned long long *ins = v1.Current();
    lm::launch_fit_order_keys(ins, pp.len, ne, c->d_fm_bn.as<unsigned long long>(), c->d_fm_bs.as<unsigned long long>(),
                              c->d_fm_sim.as<double>(), s);
    CU(cudaMemcpyAsync(ins_pairs.data(), ins, 8 * ne, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(c->fm.sim.data(), c->d_fm_sim.p, 8 * ne, cudaMemcpyDeviceToHost, s));
    const uint64_t *greedy = nullptr;
    const int rc = sort_greedy_order(c->d_sort_tmp, c->d_fm_bn, c->d_fm_bn2, c->d_fm_bs, c->d_fm_bs2, (int)ne, s, greedy);
    if (rc) return rc;
    CU(cudaMemcpyAsync(order.data(), greedy, 8 * ne, cudaMemcpyDeviceToHost, s));
    c->mg_stats.n_kernel_launches += 7;
  }
  if (n) {
    CU(cudaMemcpyAsync(len.data(), pp.len, 8 * n, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(rec.data(), pp.rec, 56 * n, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  c->fm.length = len;
  // graph nodes: lines of non-zero length in (image, line) order (merging.cc:370-382)
  std::vector<int32_t> node_of(n, -1);
  std::vector<int> image_of;
  c->fm.unc.resize(n);
  for (int v = 0; v < n_views; ++v)
    for (int64_t g = line_off[v]; g < line_off[v + 1]; ++g) {
      c->fm.unc[g] = rec[7 * g + 6];
      if (len[g] == 0) continue;
      node_of[g] = (int32_t)c->fm.node_line.size();
      c->fm.node_line.push_back(g);
      image_of.push_back(v);
    }
  c->fm.edges.resize(2 * ne);
  for (int64_t e = 0; e < ne; ++e) {
    c->fm.edges[2 * e] = node_of[ins_pairs[e] >> 32];
    c->fm.edges[2 * e + 1] = node_of[ins_pairs[e] & 0xffffffffull];
  }
  for (uint64_t &o : order) {
    o = ~o;
    o = (uint64_t)(uint32_t)node_of[o >> 32] << 32 | (uint64_t)(uint32_t)node_of[o & 0xffffffffull];
  }
  int n_tracks = 0;
  const std::vector<int> label = greedy_track_labels(order, image_of, n_views, n_tracks);
  std::vector<std::vector<int32_t>> members(n_tracks);
  for (size_t i = 0; i < label.size(); ++i)
    if (label[i] >= 0) members[label[i]].push_back((int32_t)i);
  c->fm.track_off.assign(1, 0);
  c->fm.track_line.resize(7 * (size_t)n_tracks);
  std::vector<AggItem> items;
  for (int t = 0; t < n_tracks; ++t) {
    items.clear();
    for (int32_t k : members[t]) {
      c->fm.track_nodes.push_back(k);
      const int64_t g = c->fm.node_line[k];
      items.push_back(AggItem{&rec[7 * g], rec[7 * g + 6], len[g]}); // score = length (merging.cc:493)
    }
    c->fm.track_off.push_back((int64_t)c->fm.track_nodes.size());
    aggregate_items(items, 0, &c->fm.track_line[7 * (size_t)t]); // aggregate_line3d_list(lines, scores, 0)
  }
  out_counts[0] = (int64_t)c->fm.node_line.size();
  out_counts[1] = ne;
  out_counts[2] = (int64_t)c->fm.track_nodes.size();
  lm_fit_merge_stats &st = c->fm_stats;
  st.n_nodes = out_counts[0];
  st.n_pairs_tested = (int64_t)cnt[2];
  st.n_pairs_gated = (int64_t)cnt[1];
  st.n_edges = ne;
  st.n_tracks = n_tracks;
  st.pair_kernel_ms = msk;
  st.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
  return n_tracks;
}

int lm_merge_fits_get(lm_ctx *c, double *unc, double *length, int64_t *node_line, int32_t *edges, double *sim, int64_t *track_off,
                      int32_t *track_nodes, double *track_line) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  const lm_ctx::FitMerge &r = c->fm;
  auto put = [](const auto &v, auto *out) { if (out) std::copy(v.begin(), v.end(), out); };
  put(r.unc, unc);
  put(r.length, length);
  put(r.node_line, node_line);
  put(r.edges, edges);
  put(r.sim, sim);
  put(r.track_off, track_off);
  put(r.track_nodes, track_nodes);
  put(r.track_line, track_line);
  return LM_OK;
}

int lm_merge_fits_get_stats(lm_ctx *c, lm_fit_merge_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->fm_stats;
  return LM_OK;
}

} // extern "C"
