// engine_locmatch.cu — line matching of query images against a line map (locmatch_kernels.cu): the epipolar sweep,
// the filter of given pairs, the grouping per query line and the reprojection filter behind lm_locmatch_*.
#include "engine.cuh"
#include "locmatch_kernels.cuh"
#include <chrono>
#include <cub/cub.cuh>

namespace {

using Clock = std::chrono::steady_clock;

int upload(DevBuf &b, const void *src, size_t bytes, cudaStream_t s) {
  CU(b.ensure(bytes + 16));
  if (bytes) CU(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
  return LM_OK;
}

// Exclusive scan of n + 1 int64 values (the last one 0): out[n] is the total.
int scan(lm_ctx *c, const int64_t *in, int64_t *out, int64_t n) {
  CU(cub_call(c->lmm.tmp, [&](void *t, size_t &b) {
    return cub::DeviceScan::ExclusiveSum(t, b, in, out, n + 1, c->stream);
  }));
  return LM_OK;
}

int64_t read_i64(lm_ctx *c, const int64_t *d) {
  int64_t v = 0;
  if (cudaMemcpyAsync(&v, d, 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess) return -1;
  if (cudaStreamSynchronize(c->stream) != cudaSuccess) return -1;
  return v;
}

lm::LocScene scene(lm_ctx *c) {
  auto &m = c->lmm;
  return lm::LocScene{m.views.as<lm::LocView>(), m.line_off.as<int64_t>(), m.lines.as<double4>(),
                      m.has_map ? m.track.as<int32_t>() : nullptr, m.tracks.as<double>()};
}

// Items: checked, uploaded with the row offsets (one row per (item, query line)).
int set_items(lm_ctx *c, int64_t n_items, const int32_t *items, lm::LocItems &it) {
  auto &m = c->lmm;
  if (n_items < 0 || (n_items > 0 && !items)) return fail(LM_ERR_INVALID, "bad items");
  std::vector<int64_t> row_off(n_items + 1, 0);
  for (int64_t k = 0; k < n_items; ++k) {
    const int32_t q = items[2 * k], t = items[2 * k + 1];
    if (q < 0 || q >= m.n_images || t < 0 || t >= m.n_images) return fail(LM_ERR_INVALID, "item image out of range");
    row_off[k + 1] = row_off[k] + (m.h_line_off[q + 1] - m.h_line_off[q]);
  }
  m.h_items.assign(items, items + 2 * n_items);
  m.n_items = n_items;
  if (int rc = upload(m.items, items, 8 * n_items, c->stream)) return rc;
  if (int rc = upload(m.row_off, row_off.data(), 8 * (n_items + 1), c->stream)) return rc;
  it = lm::LocItems{m.items.as<int2>(), m.row_off.as<int64_t>(), n_items};
  return LM_OK;
}

lm::LocItems items_of(lm_ctx *c) {
  return lm::LocItems{c->lmm.items.as<int2>(), c->lmm.row_off.as<int64_t>(), c->lmm.n_items};
}

// No result and no 2D-3D list: what a new scene, or a sweep or filter that has not finished, leaves behind.
void invalidate(lm_ctx *c) {
  auto &m = c->lmm;
  m.n_items = m.n_e = m.n_out = 0;
  m.e_tracks = false;
  m.h_items.clear();
  m.h_item_off.assign(1, 0);
  m.h_out_off.assign(1, 0);
  m.d_out = nullptr;
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

// The item offsets of E to the host; E becomes the result.
int finish_e(lm_ctx *c, int to_tracks, int64_t n_e) {
  auto &m = c->lmm;
  m.h_item_off.resize(m.n_items + 1);
  CU(cudaMemcpyAsync(m.h_item_off.data(), m.item_off.p, 8 * (m.n_items + 1), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  m.n_e = n_e;
  m.e_tracks = to_tracks != 0;
  m.h_out_off = m.h_item_off;
  m.d_out = m.E.as<int2>();
  m.n_out = n_e;
  return LM_OK;
}

// kernel_ms / test_ms: device time of the call's kernels (host waits between them excluded) / of its test kernel
void stats_end(lm_ctx *c, Clock::time_point t0, int64_t tests, int64_t pairs, double kernel_ms, double test_ms) {
  auto &st = c->lmm_stats;
  st.n_items = c->lmm.n_items;
  st.n_tests = tests;
  st.n_pairs_2to2 = pairs;
  st.n_out = c->lmm.n_out;
  st.kernel_ms = kernel_ms;
  st.test_ms = test_ms;
  st.total_ms = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
}

} // namespace

extern "C" {

int lm_locmatch_set_scene(lm_ctx *c, int32_t n_images, const double *kvec, const double *qvec, const double *tvec,
                          const int64_t *line_off, const double *lines, const int32_t *line_track, int64_t n_tracks,
                          const double *track_lines) {
  if (!c || !line_off) return fail(LM_ERR_INVALID, "NULL argument");
  if (n_images < 0 || n_tracks < 0) return fail(LM_ERR_INVALID, "negative size");
  if (n_images > 0 && (!kvec || !qvec || !tvec)) return fail(LM_ERR_INVALID, "NULL camera array");
  if (line_off[0] != 0) return fail(LM_ERR_INVALID, "line_off must start at 0");
  for (int32_t i = 0; i < n_images; ++i)
    if (line_off[i + 1] < line_off[i] || line_off[i + 1] - line_off[i] > INT32_MAX)
      return fail(LM_ERR_INVALID, "bad line_off");
  const int64_t N = line_off[n_images];
  if (N > 0 && !lines) return fail(LM_ERR_INVALID, "NULL lines");
  if (n_tracks > 0 && !track_lines) return fail(LM_ERR_INVALID, "NULL track_lines");
  if (line_track)
    for (int64_t i = 0; i < N; ++i)
      if (line_track[i] < -1 || line_track[i] >= n_tracks) return fail(LM_ERR_INVALID, "line_track out of range");
  CU(cudaSetDevice(c->device));
  auto &m = c->lmm;
  std::vector<lm::LocView> v(std::max<int32_t>(n_images, 1));
  for (int32_t i = 0; i < n_images; ++i) {
    lm::ViewD d;
    make_view(1, kvec + 4 * i, qvec + 4 * i, tvec + 3 * i, d);
    const M3h R = quat_to_R(qvec + 4 * i);
    memcpy(v[i].M, d.M, sizeof(d.M));
    memcpy(v[i].C, d.C, sizeof(d.C));
    memcpy(v[i].R, R.m, sizeof(R.m));
    memcpy(v[i].t, tvec + 3 * i, 24);
    memcpy(v[i].k, kvec + 4 * i, 32);
  }
  if (int rc = upload(m.views, v.data(), sizeof(lm::LocView) * n_images, c->stream)) return rc;
  if (int rc = upload(m.line_off, line_off, 8 * (n_images + 1), c->stream)) return rc;
  if (int rc = upload(m.lines, lines, 32 * N, c->stream)) return rc;
  if (line_track)
    if (int rc = upload(m.track, line_track, 4 * N, c->stream)) return rc;
  if (int rc = upload(m.tracks, track_lines, 48 * n_tracks, c->stream)) return rc;
  CU(cudaStreamSynchronize(c->stream)); // the host staging (v) goes out of scope
  m.n_images = n_images;
  m.n_lines = N;
  m.n_tracks = n_tracks;
  m.has_map = line_track != nullptr;
  m.h_line_off.assign(line_off, line_off + n_images + 1);
  invalidate(c);
  return LM_OK;
}

int64_t lm_locmatch_sweep(lm_ctx *c, int64_t n_items, const int32_t *items, double th, int32_t to_tracks) {
  const auto t0 = Clock::now();
  if (!c) return fail(LM_ERR_INVALID, "NULL argument");
  auto &m = c->lmm;
  if (to_tracks && !m.has_map) return fail(LM_ERR_INVALID, "to_tracks needs the scene's line_track");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  invalidate(c);
  lm::LocItems it;
  if (int rc = set_items(c, n_items, items, it)) return rc;
  // mask words: a row of item k has ceil(n_target_lines / 32) words
  std::vector<int64_t> word_off(n_items + 1, 0);
  int64_t n_rows = 0, tests = 0;
  for (int64_t k = 0; k < n_items; ++k) {
    const int64_t nq = m.h_line_off[items[2 * k] + 1] - m.h_line_off[items[2 * k]];
    const int64_t nt = m.h_line_off[items[2 * k + 1] + 1] - m.h_line_off[items[2 * k + 1]];
    word_off[k + 1] = word_off[k] + nq * ((nt + 31) / 32);
    n_rows += nq;
    tests += nq * nt;
  }
  if (int rc = upload(m.word_off, word_off.data(), 8 * (n_items + 1), s)) return rc;
  CU(m.mask.ensure(4 * word_off[n_items] + 16));
  CU(m.cnt.ensure(8 * (n_rows + 1)));
  CU(m.scan.ensure(8 * (n_rows + 1)));
  CU(m.item_off.ensure(8 * (n_items + 1)));
  CU(m.small.ensure(16));
  CU(cudaMemsetAsync(m.small.p, 0, 16, s));
  CU(cudaMemsetAsync(m.cnt.as<int64_t>() + n_rows, 0, 8, s));
  const lm::LocScene sc = scene(c);
  CU(cudaEventRecord(c->evk0, s));
  if (n_rows > 0)
    lm::launch_locmatch_sweep_count(sc, it, m.word_off.as<int64_t>(), th, to_tracks, m.mask.as<uint32_t>(),
                                    m.cnt.as<int64_t>(), m.small.as<unsigned long long>(), s);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->ev0, s));
  if (int rc = scan(c, m.cnt.as<int64_t>(), m.scan.as<int64_t>(), n_rows)) return rc;
  CU(cudaEventRecord(c->ev1, s));
  const int64_t n_e = read_i64(c, m.scan.as<int64_t>() + n_rows); // (synchronises: the events above are complete)
  if (n_e < 0) return fail(LM_ERR_CUDA, cudaGetErrorString(cudaGetLastError()));
  const double test_ms = elapsed(c->evk0, c->ev0), first_ms = elapsed(c->evk0, c->ev1);
  CU(m.E.ensure(8 * n_e + 16));
  CU(cudaEventRecord(c->evk0, s));
  if (n_e > 0)
    lm::launch_locmatch_sweep_place(sc, it, m.word_off.as<int64_t>(), m.mask.as<uint32_t>(), m.scan.as<int64_t>(),
                                    to_tracks, m.E.as<int2>(), s);
  lm::launch_gather_offsets(m.scan.as<int64_t>(), m.row_off.as<int64_t>(), n_items, m.item_off.as<int64_t>(), s);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->evk1, s));
  int64_t n_pairs = read_i64(c, reinterpret_cast<const int64_t *>(m.small.p));
  if (int rc = finish_e(c, to_tracks, n_e)) return rc;
  c->stats.n_kernel_launches += 4;
  stats_end(c, t0, tests, n_pairs, first_ms + elapsed(c->evk0, c->evk1), test_ms);
  return n_e;
}

int64_t lm_locmatch_filter(lm_ctx *c, int64_t n_items, const int32_t *items, const int64_t *pair_off,
                           const int32_t *pairs, int32_t use_iou, double th, int32_t to_tracks) {
  const auto t0 = Clock::now();
  if (!c || !pair_off) return fail(LM_ERR_INVALID, "NULL argument");
  auto &m = c->lmm;
  if (to_tracks && !m.has_map) return fail(LM_ERR_INVALID, "to_tracks needs the scene's line_track");
  if (n_items < 0 || pair_off[0] != 0) return fail(LM_ERR_INVALID, "pair_off must start at 0");
  for (int64_t k = 0; k < n_items; ++k)
    if (pair_off[k + 1] < pair_off[k]) return fail(LM_ERR_INVALID, "bad pair_off");
  const int64_t P = pair_off[n_items];
  if (P > 0 && !pairs) return fail(LM_ERR_INVALID, "NULL pairs");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  invalidate(c);
  lm::LocItems it;
  if (int rc = set_items(c, n_items, items, it)) return rc;
  if (int rc = upload(m.pair_off, pair_off, 8 * (n_items + 1), s)) return rc;
  if (int rc = upload(m.pairs, pairs, 8 * P, s)) return rc;
  CU(m.flag.ensure(8 * (P + 1)));
  CU(m.scan.ensure(8 * (P + 1)));
  CU(m.item_off.ensure(8 * (n_items + 1)));
  CU(m.err.ensure(16));
  CU(cudaMemsetAsync(m.err.p, 0, 16, s));
  CU(m.small.ensure(16));
  CU(cudaMemsetAsync(m.small.p, 0, 16, s));
  const lm::LocScene sc = scene(c);
  CU(cudaEventRecord(c->evk0, s));
  lm::launch_locmatch_filter_flags(sc, it, m.pair_off.as<int64_t>(), m.pairs.as<int2>(), P, use_iou, th, to_tracks,
                                   m.flag.as<int64_t>(), m.err.as<int>(), m.small.as<unsigned long long>(), s);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->ev0, s));
  if (int rc = scan(c, m.flag.as<int64_t>(), m.scan.as<int64_t>(), P)) return rc;
  CU(cudaEventRecord(c->ev1, s));
  int err = 0;
  CU(cudaMemcpyAsync(&err, m.err.p, 4, cudaMemcpyDeviceToHost, s));
  const int64_t n_e = read_i64(c, m.scan.as<int64_t>() + P); // (synchronises: the events above are complete)
  if (n_e < 0) return fail(LM_ERR_CUDA, cudaGetErrorString(cudaGetLastError()));
  if (err) return fail(LM_ERR_INVALID, "a pair's line id is out of range");
  const double test_ms = elapsed(c->evk0, c->ev0), first_ms = elapsed(c->evk0, c->ev1);
  CU(m.E.ensure(8 * n_e + 16));
  CU(cudaEventRecord(c->evk0, s));
  lm::launch_locmatch_filter_place(sc, it, m.pair_off.as<int64_t>(), m.pairs.as<int2>(), P, m.scan.as<int64_t>(),
                                   to_tracks, m.E.as<int2>(), s);
  lm::launch_gather_offsets(m.scan.as<int64_t>(), m.pair_off.as<int64_t>(), n_items, m.item_off.as<int64_t>(), s);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->evk1, s));
  const int64_t n_pairs = read_i64(c, reinterpret_cast<const int64_t *>(m.small.p));
  if (int rc = finish_e(c, to_tracks, n_e)) return rc;
  c->stats.n_kernel_launches += 3;
  stats_end(c, t0, use_iou ? P : 0, n_pairs, first_ms + elapsed(c->evk0, c->evk1), test_ms);
  return n_e;
}

int64_t lm_locmatch_group(lm_ctx *c, int32_t dist_func, double dist_thres, double sine_thres, double angle_scale) {
  const auto t0 = Clock::now();
  if (!c) return fail(LM_ERR_INVALID, "NULL argument");
  auto &m = c->lmm;
  if (!m.e_tracks) return fail(LM_ERR_INVALID, "lm_locmatch_group needs a to_tracks sweep or filter first");
  if (dist_func < -1 || dist_func > 2) return fail(LM_ERR_INVALID, "unknown dist function");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const lm::LocItems it = items_of(c);
  // queries: runs of items with the same query image
  std::vector<int64_t> q_item_off{0}, qrow_off{0}, q_first;
  for (int64_t k = 0; k < m.n_items; ++k) {
    if (k > 0 && m.h_items[2 * k] == m.h_items[2 * (k - 1)]) continue;
    if (k > 0) q_item_off.push_back(k);
    const int32_t q = m.h_items[2 * k];
    qrow_off.push_back(qrow_off.back() + m.h_line_off[q + 1] - m.h_line_off[q]);
  }
  if (m.n_items > 0) q_item_off.push_back(m.n_items);
  const int64_t nq = (int64_t)q_item_off.size() - 1, n_qrows = qrow_off.back();
  for (int64_t q = 0; q <= nq; ++q) q_first.push_back(m.h_item_off[q_item_off[q]]);
  const int64_t n_rows = m.n_items ? read_i64(c, m.row_off.as<int64_t>() + m.n_items) : 0;
  const int64_t n_e = m.n_e;
  CU(m.g_qoff.ensure(8 * 2 * (nq + 1) + 16));
  CU(cudaMemcpyAsync(m.g_qoff.p, q_item_off.data(), 8 * (nq + 1), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(m.g_qoff.as<int64_t>() + nq + 1, q_first.data(), 8 * (nq + 1), cudaMemcpyHostToDevice, s));
  if (int rc = upload(m.g_qrow, qrow_off.data(), 8 * (nq + 1), s)) return rc;
  CU(m.g_cnt.ensure(4 * n_rows + 16));
  CU(m.g_run.ensure(4 * n_rows + 16));
  CU(m.g_first.ensure(8 * n_rows + 16));
  CU(m.g_key.ensure(8 * n_rows + 16));
  CU(m.g_head.ensure(8 * (n_e + 1)));
  CU(m.g_qhead.ensure(8 * n_qrows + 16));
  CU(m.g_qtot.ensure(8 * n_qrows + 16));
  CU(m.G.ensure(8 * n_e + 16));
  CU(cudaMemsetAsync(m.g_cnt.p, 0, 4 * n_rows, s));
  CU(cudaMemsetAsync(m.g_run.p, 0, 4 * n_rows, s));
  CU(cudaMemsetAsync(m.g_first.p, 0xff, 8 * n_rows, s));
  CU(cudaMemsetAsync(m.g_head.p, 0, 8 * (n_e + 1), s));
  lm::LocGroup g;
  g.E = m.E.as<int2>();
  g.item_off = m.item_off.as<int64_t>();
  g.q_item_off = m.g_qoff.as<int64_t>();
  g.qrow_off = m.g_qrow.as<int64_t>();
  g.n_e = n_e;
  g.n_queries = nq;
  g.cnt = m.g_cnt.as<unsigned int>();
  g.first = m.g_first.as<unsigned long long>();
  g.key = m.g_key.as<int64_t>();
  g.run = m.g_run.as<unsigned int>();
  g.head = m.g_head.as<int64_t>();
  g.qhead = m.g_qhead.as<int64_t>();
  g.qtot = m.g_qtot.as<int64_t>();
  CU(cudaEventRecord(c->evk0, s));
  lm::launch_group_count(it, g, s);
  lm::launch_group_heads(it, g, n_qrows, s);
  CU(cudaGetLastError());
  CU(m.scan.ensure(8 * (n_e + 1)));
  if (int rc = scan(c, m.g_head.as<int64_t>(), m.scan.as<int64_t>(), n_e)) return rc;
  g.head = m.scan.as<int64_t>();
  lm::launch_group_keys(it, g, n_qrows, s);
  lm::launch_group_place(it, g, m.G.as<int2>(), s);
  CU(cudaGetLastError());
  const int64_t *qfirst = m.g_qoff.as<int64_t>() + nq + 1;
  int64_t n_out = n_e;
  if (dist_func < 0) {
    m.d_out = m.G.as<int2>();
    CU(cudaEventRecord(c->evk1, s));
    m.h_out_off = q_first;
  } else {
    CU(m.flag.ensure(8 * (n_e + 1)));
    CU(m.pos.ensure(8 * (n_e + 1)));
    CU(m.sel.ensure(4 * n_e + 16));
    CU(m.out.ensure(8 * n_e + 16));
    CU(cudaMemsetAsync(m.flag.p, 0, 8 * (n_e + 1), s));
    const lm::ReprojParams rp{dist_func, dist_thres, sine_thres, angle_scale};
    if (n_qrows > 0)
      lm::launch_reproj_filter(scene(c), it, g, m.G.as<int2>(), rp, m.flag.as<int64_t>(), m.sel.as<int32_t>(), s);
    CU(cudaGetLastError());
    if (int rc = scan(c, m.flag.as<int64_t>(), m.pos.as<int64_t>(), n_e)) return rc;
    lm::launch_reproj_place(g, m.G.as<int2>(), m.pos.as<int64_t>(), m.sel.as<int32_t>(), m.out.as<int2>(), s);
    // per-query offsets of the filtered list
    CU(m.g_qout.ensure(8 * (nq + 1)));
    lm::launch_gather_offsets(m.pos.as<int64_t>(), qfirst, nq, m.g_qout.as<int64_t>(), s);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->evk1, s));
    m.h_out_off.resize(nq + 1);
    CU(cudaMemcpyAsync(m.h_out_off.data(), m.g_qout.p, 8 * (nq + 1), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    n_out = m.h_out_off[nq];
    m.d_out = m.out.as<int2>();
  }
  CU(cudaStreamSynchronize(s));
  m.n_out = n_out;
  c->stats.n_kernel_launches += dist_func < 0 ? 4 : 7;
  stats_end(c, t0, 0, 0, elapsed(c->evk0, c->evk1), 0.0);
  return n_out;
}

int lm_locmatch_get(lm_ctx *c, int64_t *off, int32_t *pairs, int64_t cap) {
  if (!c) return fail(LM_ERR_INVALID, "NULL argument");
  auto &m = c->lmm;
  if (pairs && cap < m.n_out) return fail(LM_ERR_INVALID, "pairs buffer too small");
  if (off) memcpy(off, m.h_out_off.data(), 8 * m.h_out_off.size());
  if (pairs && m.n_out > 0) {
    CU(cudaMemcpyAsync(pairs, m.d_out, 8 * m.n_out, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  return LM_OK;
}

int lm_locmatch_get_stats(lm_ctx *c, lm_locmatch_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->lmm_stats;
  return LM_OK;
}

} // extern "C"
