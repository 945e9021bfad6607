// engine.cu — host side of the C ABI declared in include/limap_b200.h: context, scene upload, batched
// TriangulateImage, result getters and the multi-GPU exchange. The later stages live in engine_*.cu (engine.cuh).
//
// Mirrors (file:line under /root/reference/src/limap/):
//   BaseLineTriangulator::{Init,TriangulateImage,TriangulateImageExhaustiveMatch}
//       triangulation/base_line_triangulator.cc:45-136
//   GlobalLineTriangulator::ScoringCallback    triangulation/global_line_triangulator.cc:59-69
// There is no CPU fallback: without a CUDA device lm_ctx_create fails with LM_ERR_NOGPU.
#include "engine.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cstdlib>
#include <memory>
#include <set>

M3h quat_to_R(const double q_in[4]) { // base/pose.cc:12-18 (Eigen toRotationMatrix)
  double n = std::sqrt(q_in[0] * q_in[0] + q_in[1] * q_in[1] + q_in[2] * q_in[2] + q_in[3] * q_in[3]);
  double q[4];
  if (n == 0) { q[0] = 1; q[1] = q_in[1]; q[2] = q_in[2]; q[3] = q_in[3]; }
  else for (int i = 0; i < 4; ++i) q[i] = q_in[i] / n;
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  M3h R;
  R.m[0] = 1 - (tyy + tzz); R.m[1] = txy - twz; R.m[2] = txz + twy;
  R.m[3] = txy + twz; R.m[4] = 1 - (txx + tzz); R.m[5] = tyz - twx;
  R.m[6] = txz - twy; R.m[7] = tyz + twx; R.m[8] = 1 - (txx + tyy);
  return R;
}

// Per-view constants (tri_kernels.cuh ViewT) from the reference's camera arrays.
void make_view(int model_id, const double *kv, const double *qv, const double *t, lm::ViewD &d) {
  const double fx = kv[0], fy = kv[1], cx = kv[2], cy = kv[3];
  // CameraPose(qvec, tvec) normalises qvec (base/camera.h:92-93)
  M3h R = quat_to_R(qv);
  // K^-1 (closed form of Eigen's cofactor inverse for the pinhole K)
  const double ki[9] = {1.0 / fx, 0, -cx / fx, 0, 1.0 / fy, -cy / fy, 0, 0, 1};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) // M = R^T * Kinv
      d.M[3 * i + j] = R.m[0 * 3 + i] * ki[0 * 3 + j] + R.m[1 * 3 + i] * ki[1 * 3 + j] + R.m[2 * 3 + i] * ki[2 * 3 + j];
  for (int i = 0; i < 3; ++i) d.C[i] = -(R.m[0 * 3 + i] * t[0] + R.m[1 * 3 + i] * t[1] + R.m[2 * 3 + i] * t[2]);
  const double K[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      d.P[4 * i + j] = K[3 * i] * R.m[j] + K[3 * i + 1] * R.m[3 + j] + K[3 * i + 2] * R.m[6 + j];
    d.P[4 * i + 3] = K[3 * i] * t[0] + K[3 * i + 1] * t[1] + K[3 * i + 2] * t[2];
  }
  d.fbar = (model_id == 0) ? fx : (fx + fy) / 2.0;
  d.pad = 0;
}

int fetch_nodes(lm_ctx *c) {
  if (c->h_nodes_valid) return LM_OK;
  c->h_nodes.resize(c->n_nodes);
  CU(cudaMemcpyAsync(c->h_nodes.data(), c->d_nodes.p, sizeof(lm::NodeRecord) * c->n_nodes, cudaMemcpyDeviceToHost,
                     c->stream));
  CU(cudaStreamSynchronize(c->stream));
  c->h_nodes_valid = true;
  return LM_OK;
}
static int fetch_rows(lm_ctx *c) {
  if (c->h_rows_valid) return LM_OK;
  c->h_node_row_off.resize(c->n_nodes + 1);
  c->h_row_ng.resize(c->n_rows);
  c->h_row_state.resize(c->n_rows * c->ns);
  CU(cudaMemcpyAsync(c->h_node_row_off.data(), c->d_node_row_off.p, 4 * (c->n_nodes + 1), cudaMemcpyDeviceToHost,
                     c->stream));
  if (c->n_rows) {
    CU(cudaMemcpyAsync(c->h_row_ng.data(), c->d_row_ng.p, 4 * c->n_rows, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(c->h_row_state.data(), c->d_row_state.p, c->n_rows * c->ns, cudaMemcpyDeviceToHost, c->stream));
    if (c->cfg.debug_mode) {
      c->h_row_cand.resize(c->n_rows * c->ns * 10);
      CU(cudaMemcpyAsync(c->h_row_cand.data(), c->d_row_cand.p, 80 * c->n_rows * c->ns, cudaMemcpyDeviceToHost, c->stream));
    }
  }
  CU(cudaStreamSynchronize(c->stream));
  c->h_rows_valid = true;
  return LM_OK;
}

static int fetch_edges(lm_ctx *c) {
  if (c->h_edges_valid) return LM_OK;
  const int64_t n = c->node_end - c->node_begin;
  c->h_edge_off.assign(n + 1, 0);
  c->h_edge_ng.resize(c->stats.n_valid_edges);
  if (n > 0) {
    CU(cudaMemcpyAsync(c->h_edge_off.data(), c->d_edge_off.p, 4 * (n + 1), cudaMemcpyDeviceToHost, c->stream));
    if (c->stats.n_valid_edges)
      CU(cudaMemcpyAsync(c->h_edge_ng.data(), c->d_edge_ng.p, 4 * c->stats.n_valid_edges, cudaMemcpyDeviceToHost,
                         c->stream));
  }
  CU(cudaStreamSynchronize(c->stream));
  c->h_edges_valid = true;
  return LM_OK;
}

int ensure_ran(lm_ctx *c) {
  if (c->ran) return LM_OK;
  return lm_tri_run(c);
}

int collect_edges(lm_ctx *c) {
  if (c->edges_collected) {
    // (the overflow stays set after lm_tri_gather_status read it: the truncated edges are never used)
    const int64_t over = lm_tri_gather_status(c, nullptr);
    if (over < 0) return (int)over;
    if (over) return fail(LM_ERR_STATE, "the last multi-GPU exchange overflowed its edge capacity: repeat it with a larger message");
    return LM_OK;
  }
  const int64_t ne = c->stats.n_valid_edges;
  CU(c->d_edges.ensure(16 * std::max<int64_t>(ne, 1)));
  lm::launch_edge_pairs(c->d_edge_off.as<uint32_t>(), c->d_edge_ng.as<uint32_t>(), c->d_line_off.as<int64_t>(),
                        c->node_begin, c->node_end - c->node_begin, ne, c->d_edges.as<int64_t>(), c->stream);
  c->stats.n_kernel_launches += 1;
  c->n_edges_dev = ne;
  c->edges_collected = true;
  return LM_OK;
}

extern "C" {

const char *lm_last_error(void) { return g_err.c_str(); }
const char *lm_version(void) { return "limap_b200 0.1 (sm_90a)"; }

int lm_ctx_create(int device, lm_ctx **out) {
  if (!out) return fail(LM_ERR_INVALID, "out is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(LM_ERR_NOGPU, std::string("no CUDA device (") + cudaGetErrorString(e) +
                                  "); limap_b200 has no CPU fallback");
  if (device < 0 || device >= n) return fail(LM_ERR_INVALID, "device index out of range");
  CU(cudaSetDevice(device));
  std::unique_ptr<lm_ctx> c(new lm_ctx()); // (released to the caller only once every resource exists)
  c->device = device;
  CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  c->own_stream = true;
  CU(cudaEventCreate(&c->ev0));
  CU(cudaEventCreate(&c->ev1));
  CU(cudaEventCreate(&c->evk0));
  CU(cudaEventCreate(&c->evk1));
  CU(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  {
    int lo_p = 0, hi_p = 0; // (numerically lowest = greatest priority: the small preparation kernels take the next free SM slots)
    CU(cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p));
    CU(cudaStreamCreateWithPriority(&c->prep_stream, cudaStreamNonBlocking, hi_p));
    CU(cudaStreamCreateWithPriority(&c->out_stream, cudaStreamNonBlocking, hi_p));
    CU(cudaEventCreateWithFlags(&c->ev_run_begin, cudaEventDisableTiming));
  }
  CU(cudaHostAlloc(reinterpret_cast<void **>(&c->h_pin), 2048, cudaHostAllocDefault));
  CU(cudaEventCreateWithFlags(&c->ev_scene, cudaEventDisableTiming));
  cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
  cudaDeviceGetAttribute(&c->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  memset(&c->stats, 0, sizeof(c->stats));
  memset(&c->ba_stats, 0, sizeof(c->ba_stats));
  memset(&c->vp_stats, 0, sizeof(c->vp_stats));
  memset(&c->mg_stats, 0, sizeof(c->mg_stats));
  *out = c.release();
  return LM_OK;
}

// Runs on the context's device (lm_ctx_destroy, or lm_ctx_create on failure). The device buffers free themselves after
// the body, once no stream can still use them.
lm_ctx::~lm_ctx() {
  cudaStreamSynchronize(stream);
  for (cudaStream_t s : {copy_stream, prep_stream, out_stream})
    if (s) cudaStreamSynchronize(s);
  for (cudaEvent_t e : {ev0, ev1, evk0, evk1, ev_raw, ev_scene, ev_run_begin})
    if (e) cudaEventDestroy(e);
  for (auto e : evk) cudaEventDestroy(e);
  for (auto e : evp) cudaEventDestroy(e);
  for (auto &ch : chunks) cudaEventDestroy(ch.ev);
  for (auto e : event_pool) cudaEventDestroy(e);
  for (cudaStream_t s : {copy_stream, prep_stream, out_stream})
    if (s) cudaStreamDestroy(s);
  if (own_stream && stream) cudaStreamDestroy(stream); // (a stream set through lm_ctx_set_stream is the caller's)
  if (h_pin) cudaFreeHost(h_pin);
  if (h_ba_pin) cudaFreeHost(h_ba_pin);
}

void lm_ctx_destroy(lm_ctx *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  delete c;
}

int lm_ctx_set_stream(lm_ctx *c, void *s) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  c->stream = (cudaStream_t)s;
  c->own_stream = false;
  return LM_OK;
}
int lm_ctx_synchronize(lm_ctx *c) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->copy_stream));
  CU(cudaStreamSynchronize(c->stream));
  return LM_OK;
}

static int tri_clear_impl(lm_ctx *c, bool sync_copies);
static int upload_segs(lm_ctx *c, bool with_node_view) {
  // add_halfpix (base_line_triangulator.cc:32-43) is applied when both scene and config are known: on the device, from
  // the raw copy of the caller's segments, in stream order behind that copy.
  if (c->n_nodes)
    lm::launch_scene_prepare(c->d_segs_raw.as<double>(), c->n_nodes, (c->have_cfg && c->cfg.add_halfpix) ? 0.5 : 0.0,
                             c->d_line_off.as<int64_t>(), c->V, c->d_segs.as<double>(),
                             with_node_view ? c->d_node_view.as<uint16_t>() : nullptr, c->copy_stream);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->ev_scene, c->copy_stream));
  return LM_OK;
}

int lm_scene_upload(lm_ctx *c, int32_t n_views, const int32_t *img_ids, const int32_t *model_ids, const double *kvec,
                    const double *qvec, const double *tvec, const int64_t *line_off, const double *segs) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (n_views <= 0 || n_views > 65535) return fail(LM_ERR_INVALID, "n_views must be in [1, 65535]");
  CU(cudaSetDevice(c->device));
  for (int v = 1; v < n_views; ++v)
    if (img_ids[v] <= img_ids[v - 1]) return fail(LM_ERR_INVALID, "img_ids must be strictly ascending");
  CU(cudaStreamSynchronize(c->copy_stream)); // the host staging tables below may still feed a previous upload
  CU(cudaStreamSynchronize(c->stream));      // ... and a previous run may still read buffers that get re-allocated
  c->V = n_views;
  c->img_ids.assign(img_ids, img_ids + n_views);
  c->id2view.clear();
  for (int v = 0; v < n_views; ++v) c->id2view[img_ids[v]] = v;
  c->line_off.assign(line_off, line_off + n_views + 1);
  c->n_nodes = line_off[n_views];
  if (c->n_nodes >= ((int64_t)1 << 31) - 64) return fail(LM_ERR_INVALID, "more than 2^31 2D lines in one scene");
  std::vector<lm::ViewD> &views = c->h_views;
  views.resize(n_views);
  for (int v = 0; v < n_views; ++v) {
    if (model_ids[v] != 0 && model_ids[v] != 1)
      return fail(LM_ERR_INVALID, "only SIMPLE_PINHOLE / PINHOLE are legal on this path (IsUndistorted check)");
    if (line_off[v + 1] - line_off[v] > 65535) return fail(LM_ERR_INVALID, "more than 65535 lines in one image");
    make_view(model_ids[v], kvec + 4 * v, qvec + 4 * v, tvec + 3 * v, views[v]);
  }
  CU(c->d_views.ensure(sizeof(lm::ViewD) * n_views));
  CU(c->d_node_view.ensure(std::max<size_t>(2, 2 * c->n_nodes)));
  CU(c->d_line_off.ensure(8 * (n_views + 1)));
  CU(c->d_segs_raw.ensure(std::max<size_t>(32, 32 * (size_t)c->n_nodes)));
  CU(c->d_segs.ensure(std::max<size_t>(32, 32 * (size_t)c->n_nodes)));
  CU(cudaMemcpyAsync(c->d_views.p, views.data(), sizeof(lm::ViewD) * n_views, cudaMemcpyHostToDevice, c->copy_stream));
  CU(cudaMemcpyAsync(c->d_line_off.p, c->line_off.data(), 8 * (n_views + 1), cudaMemcpyHostToDevice, c->copy_stream));
  CU(c->d_img_ids.ensure(4 * n_views));
  CU(cudaMemcpyAsync(c->d_img_ids.p, c->img_ids.data(), 4 * n_views, cudaMemcpyHostToDevice, c->copy_stream));
  // the 2D segments go up straight from the caller's buffer (a pinned buffer is not staged: it must stay unchanged until
  // the next call that synchronises, e.g. lm_tri_run; pageable memory is staged by the driver before this returns)
  if (c->n_nodes)
    CU(cudaMemcpyAsync(c->d_segs_raw.p, segs, 32 * (size_t)c->n_nodes, cudaMemcpyHostToDevice, c->copy_stream));
  c->have_scene = true;
  c->outside_shard_clean = false;
  int rc = upload_segs(c, true);
  if (rc) return rc;
  c->image_added.assign(n_views, 0);
  c->stats.n_nodes = c->n_nodes;
  return tri_clear_impl(c, false); // (both streams were drained on entry: no match chunk is in flight)
}

int lm_tri_configure(lm_ctx *c, const lm_tri_config *cfg) {
  if (!c || !cfg) return fail(LM_ERR_INVALID, "NULL argument");
  if (cfg->merging_strategy != 0)
    return fail(LM_ERR_INVALID, "Error!The given merging strategy is not implemented"); // global_line_triangulator.cc:318
  const bool halfpix_changed = !c->have_cfg || (c->cfg.add_halfpix != cfg->add_halfpix);
  c->cfg = *cfg;
  c->have_cfg = true;
  c->ran = false;
  if (c->have_scene && halfpix_changed) return upload_segs(c, false);
  return LM_OK;
}
int lm_tri_set_ranges(lm_ctx *c, const double lo[3], const double hi[3]) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  c->ranges_flag = true;
  for (int i = 0; i < 3; ++i) { c->rlo[i] = lo[i]; c->rhi[i] = hi[i]; }
  c->ran = false;
  return LM_OK;
}
int lm_tri_unset_ranges(lm_ctx *c) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  c->ranges_flag = false;
  c->ran = false;
  return LM_OK;
}
int lm_tri_set_vps(lm_ctx *c, int32_t n_images, const int32_t *img_ids, const int64_t *label_off, const int32_t *labels,
                   const int64_t *vp_off, const double *vps) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_scene) return fail(LM_ERR_STATE, "lm_scene_upload must precede InitVPResults");
  CU(cudaSetDevice(c->device));
  std::vector<int32_t> lab(std::max<int64_t>(c->n_nodes, 1), -1);
  std::vector<int64_t> voff(c->V + 1, 0);
  std::vector<int64_t> cnt(c->V, 0);
  std::vector<int> src(c->V, -1);
  for (int i = 0; i < n_images; ++i) {
    auto it = c->id2view.find(img_ids[i]);
    if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id in InitVPResults");
    const int v = it->second;
    const int64_t nl = label_off[i + 1] - label_off[i];
    if (nl != c->line_off[v + 1] - c->line_off[v]) return fail(LM_ERR_INVALID, "VPResult.labels size != number of lines");
    cnt[v] = vp_off[i + 1] - vp_off[i];
    src[v] = i;
    for (int64_t l = 0; l < nl; ++l) {
      const int32_t x = labels[label_off[i] + l];
      if (x >= cnt[v]) return fail(LM_ERR_INVALID, "VP label out of range");
      lab[c->line_off[v] + l] = x;
    }
  }
  for (int v = 0; v < c->V; ++v) voff[v + 1] = voff[v] + cnt[v];
  std::vector<double> vv(3 * std::max<int64_t>(voff[c->V], 1), 0.0);
  for (int v = 0; v < c->V; ++v)
    if (src[v] >= 0)
      memcpy(&vv[3 * voff[v]], vps + 3 * vp_off[src[v]], 24 * cnt[v]);
  CU(cudaStreamSynchronize(c->stream)); // a previous run may still read the tables that are re-allocated
  CU(c->d_vp_label.ensure(4 * lab.size()));
  CU(c->d_vp_voff.ensure(8 * voff.size()));
  CU(c->d_vp_vps.ensure(8 * vv.size()));
  CU(cudaMemcpyAsync(c->d_vp_label.p, lab.data(), 4 * lab.size(), cudaMemcpyHostToDevice, c->copy_stream));
  CU(cudaMemcpyAsync(c->d_vp_voff.p, voff.data(), 8 * voff.size(), cudaMemcpyHostToDevice, c->copy_stream));
  CU(cudaMemcpyAsync(c->d_vp_vps.p, vv.data(), 8 * vv.size(), cudaMemcpyHostToDevice, c->copy_stream));
  CU(cudaEventRecord(c->ev_scene, c->copy_stream));
  CU(cudaStreamSynchronize(c->copy_stream)); // the staging vectors die here
  c->have_vps = true;
  c->ran = false;
  return LM_OK;
}

int lm_tri_clear(lm_ctx *c) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  return tri_clear_impl(c, true);
}
static int tri_clear_impl(lm_ctx *c, bool sync_copies) {
  c->blocks.clear();
  c->raw_uploaded = 0;
  std::fill(c->image_added.begin(), c->image_added.end(), 0);
  if (c->copy_stream && sync_copies) cudaStreamSynchronize(c->copy_stream); // (the chunk events go back to the pool)
  for (auto &ch : c->chunks) c->event_pool.push_back(ch.ev);
  c->chunks.clear();
  c->pairs_rows = 0;
  c->any_exhaustive = c->any_matches = false;
  c->ran = false;
  c->h_nodes_valid = c->h_rows_valid = c->h_edges_valid = false;
  c->edges_collected = false;
  c->tracks.clear();
  return LM_OK;
}
int lm_tri_set_node_sink(lm_ctx *c, void *host_nodes) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  c->node_sink = static_cast<char *>(host_nodes);
  return LM_OK;
}
int lm_tri_set_pipeline_groups(lm_ctx *c, int32_t n) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (n < 1 || n > 64) return fail(LM_ERR_INVALID, "pipeline groups must be in [1, 64]");
  c->pipeline_groups = n;
  return LM_OK;
}

int lm_tri_set_shard(lm_ctx *c, int32_t b, int32_t e) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (b != c->shard_begin || e != c->shard_end) c->outside_shard_clean = false;
  c->shard_begin = b;
  c->shard_end = e;
  c->ran = false;
  return LM_OK;
}

// Mirror the block descriptors added since the last call on the device (copy stream, ahead of their matches).
static int upload_raw_blocks(lm_ctx *c) {
  const int64_t n = (int64_t)c->blocks.size();
  if (n <= c->raw_uploaded) return LM_OK;
  if ((size_t)n * sizeof(lm::RawBlock) > c->d_raw_blocks.cap) {
    CU(cudaStreamSynchronize(c->copy_stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(c->d_raw_blocks.grow_keep(std::max<size_t>((size_t)n * sizeof(lm::RawBlock) * 2, 1 << 16),
                                 c->raw_uploaded * sizeof(lm::RawBlock), c->stream));
  }
  // pageable source: the runtime stages it before returning, so `blocks` may grow (and move) afterwards
  CU(cudaMemcpyAsync(c->d_raw_blocks.as<lm::RawBlock>() + c->raw_uploaded, c->blocks.data() + c->raw_uploaded,
                     (n - c->raw_uploaded) * sizeof(lm::RawBlock), cudaMemcpyHostToDevice, c->copy_stream));
  if (!c->ev_raw) CU(cudaEventCreateWithFlags(&c->ev_raw, cudaEventDisableTiming));
  CU(cudaEventRecord(c->ev_raw, c->copy_stream));
  c->raw_uploaded = n;
  return LM_OK;
}

// Upload `total` match rows into the device store in chunks, one event per chunk, on the copy stream.
static int upload_pairs(lm_ctx *c, const int32_t *pairs, int64_t total, bool on_device) {
  if ((size_t)(c->pairs_rows + total) * 8 > c->d_pairs.cap) {
    CU(cudaStreamSynchronize(c->copy_stream));
    CU(c->d_pairs.grow_keep(std::max<size_t>((size_t)(c->pairs_rows + total) * 8 * 2, 1 << 20), c->pairs_rows * 8,
                            c->stream));
  }
  // one event per copy; the copies start at 2 MB and double up to 16 MB, so that the first pipeline group of a run (a few
  // per cent of the rows) does not wait for a full-size chunk
  const int64_t kChunk = 2 << 20;
  int64_t step = 256 << 10;
  for (int64_t o = 0, n = 0; o < total; o += n, step = std::min(kChunk, step * 2)) {
    n = std::min(step, total - o);
    CU(cudaMemcpyAsync(c->d_pairs.as<char>() + (c->pairs_rows + o) * 8, pairs + 2 * o, n * 8,
                       on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->copy_stream));
    cudaEvent_t ev;
    if (!c->event_pool.empty()) { ev = c->event_pool.back(); c->event_pool.pop_back(); }
    else CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CU(cudaEventRecord(ev, c->copy_stream));
    c->chunks.push_back({c->pairs_rows + o + n, ev});
  }
  return LM_OK;
}

// The shared tail of the match-based entry points, once their arguments are validated: append the blocks (pair_off
// already counts from the start of the device store), upload their descriptors and then `total` rows of `pairs`, and
// mark the blocks' source images as triangulated.
static int append_matches(lm_ctx *c, const std::vector<lm::RawBlock> &nb, const int32_t *pairs, int64_t total,
                          bool on_device) {
  c->blocks.insert(c->blocks.end(), nb.begin(), nb.end());
  int rc = upload_raw_blocks(c);
  if (!rc) rc = upload_pairs(c, pairs, total, on_device);
  if (rc) return rc;
  c->pairs_rows += total;
  for (const lm::RawBlock &b : nb) c->image_added[b.src_view] = 1;
  c->any_matches = true;
  c->ran = false;
  return LM_OK;
}

static int add_matches_impl(lm_ctx *c, int32_t img_id, int32_t n_ng, const int32_t *ng_ids, const int64_t *row_off,
                            const int32_t *pairs, bool on_device) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_scene) return fail(LM_ERR_STATE, "lm_scene_upload must precede TriangulateImage");
  CU(cudaSetDevice(c->device));
  auto it = c->id2view.find(img_id);
  if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id " + std::to_string(img_id));
  const int sv = it->second;
  if (c->image_added[sv]) return fail(LM_ERR_STATE, "image " + std::to_string(img_id) + " was already triangulated");
  if (c->any_exhaustive) return fail(LM_ERR_STATE, "cannot mix exhaustive and match-based triangulation in one run");
  const int64_t total = n_ng > 0 ? row_off[n_ng] : 0;
  std::set<int> seen;
  std::vector<lm::RawBlock> nb;
  for (int g = 0; g < n_ng; ++g) {
    auto f = c->id2view.find(ng_ids[g]);
    if (f == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown neighbor image id " + std::to_string(ng_ids[g]));
    if (!seen.insert(ng_ids[g]).second) return fail(LM_ERR_INVALID, "duplicate neighbor id in one TriangulateImage call");
    if (row_off[g + 1] < row_off[g]) return fail(LM_ERR_INVALID, "row_off must be non-decreasing");
    // order 0: the run visits neighbours in ascending id = std::map order (base_line_triangulator.cc:74)
    nb.push_back({sv, f->second, row_off[g + 1] - row_off[g], c->pairs_rows + row_off[g], 0, 0});
  }
  const int rc = append_matches(c, nb, pairs, total, on_device);
  if (!rc) c->image_added[sv] = 1; // (an image without neighbours, too)
  return rc;
}
int lm_tri_add_image_matches(lm_ctx *c, int32_t img_id, int32_t n_ng, const int32_t *ng_ids, const int64_t *row_off,
                             const int32_t *pairs) {
  return add_matches_impl(c, img_id, n_ng, ng_ids, row_off, pairs, false);
}
int lm_tri_add_image_matches_device(lm_ctx *c, int32_t img_id, int32_t n_ng, const int32_t *ng_ids,
                                    const int64_t *row_off, const int32_t *d_pairs) {
  return add_matches_impl(c, img_id, n_ng, ng_ids, row_off, d_pairs, true);
}
int lm_tri_add_matches_bulk(lm_ctx *c, int32_t n_blocks, const int32_t *src_img_ids, const int32_t *ng_img_ids,
                            const int64_t *row_off, const int32_t *pairs) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_scene) return fail(LM_ERR_STATE, "lm_scene_upload must precede TriangulateImage");
  if (c->any_exhaustive) return fail(LM_ERR_STATE, "cannot mix exhaustive and match-based triangulation in one run");
  CU(cudaSetDevice(c->device));
  const int64_t total = n_blocks > 0 ? row_off[n_blocks] : 0;
  std::vector<lm::RawBlock> nb;
  nb.reserve(n_blocks);
  for (int b = 0; b < n_blocks; ++b) {
    auto is = c->id2view.find(src_img_ids[b]), in_ = c->id2view.find(ng_img_ids[b]);
    if (is == c->id2view.end() || in_ == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id in matches");
    if (c->image_added[is->second]) return fail(LM_ERR_STATE, "image " + std::to_string(src_img_ids[b]) + " was already triangulated");
    if (row_off[b + 1] < row_off[b]) return fail(LM_ERR_INVALID, "row_off must be non-decreasing");
    nb.push_back({is->second, in_->second, row_off[b + 1] - row_off[b], c->pairs_rows + row_off[b], 0, 0});
  }
  return append_matches(c, nb, pairs, total, false);
}

int lm_tri_get_nodes(lm_ctx *c, lm_node_record *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  int rc = ensure_ran(c);
  if (rc) return rc;
  CU(cudaMemcpyAsync(out, c->d_nodes.p, sizeof(lm::NodeRecord) * c->n_nodes, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return LM_OK;
}

int64_t lm_tri_get_all_valid_edges(lm_ctx *c, int64_t *node_off, int32_t *edges) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int rc = ensure_ran(c);
  if (rc) return rc;
  const int64_t ne = c->stats.n_valid_edges;
  if (!node_off && !edges) return ne;
  // converted on the device and copied straight into the caller's buffers (pinned buffers avoid staging)
  const int64_t nsh = c->node_end - c->node_begin;
  if (nsh <= 0) { // empty shard: nothing on the device to convert
    if (node_off) memset(node_off, 0, 8 * (size_t)(c->n_nodes + 1));
    return 0;
  }
  const size_t off_bytes = 8 * (size_t)(c->n_nodes + 1), pair_bytes = 8 * (size_t)std::max<int64_t>(ne, 1);
  CU(c->d_host_edges.ensure(off_bytes + pair_bytes + 256));
  int64_t *d_off = c->d_host_edges.as<int64_t>();
  int32_t *d_pairs = reinterpret_cast<int32_t *>(c->d_host_edges.as<char>() + ((off_bytes + 255) / 256) * 256);
  lm::launch_edges_for_host(c->d_edge_off.as<uint32_t>(), c->d_edge_ng.as<uint32_t>(), c->d_img_ids.as<int32_t>(), nsh,
                            ne, c->node_begin, c->n_nodes, d_off, d_pairs, c->stream);
  c->stats.n_kernel_launches += 1;
  if (node_off) CU(cudaMemcpyAsync(node_off, d_off, off_bytes, cudaMemcpyDeviceToHost, c->stream));
  if (edges && ne) CU(cudaMemcpyAsync(edges, d_pairs, 8 * (size_t)ne, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return ne;
}

int lm_tri_add_image_exhaustive(lm_ctx *c, int32_t img_id, int32_t n_ng, const int32_t *ng_ids) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_scene) return fail(LM_ERR_STATE, "lm_scene_upload must precede TriangulateImageExhaustiveMatch");
  auto it = c->id2view.find(img_id);
  if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id " + std::to_string(img_id));
  const int sv = it->second;
  if (c->image_added[sv]) return fail(LM_ERR_STATE, "image " + std::to_string(img_id) + " was already triangulated");
  if (c->any_matches) return fail(LM_ERR_STATE, "cannot mix exhaustive and match-based triangulation in one run");
  const int64_t nl = c->line_off[sv + 1] - c->line_off[sv];
  std::vector<lm::RawBlock> nb;
  for (int g = 0; g < n_ng; ++g) {
    auto f = c->id2view.find(ng_ids[g]);
    if (f == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown neighbor image id " + std::to_string(ng_ids[g]));
    // no stored pairs; order g: neighbours are visited in the given order (base_line_triangulator.cc:116-117)
    nb.push_back({sv, f->second, nl * (c->line_off[f->second + 1] - c->line_off[f->second]), -1, g, 0});
  }
  c->blocks.insert(c->blocks.end(), nb.begin(), nb.end());
  c->image_added[sv] = 1;
  c->any_exhaustive = true;
  c->ran = false;
  return upload_raw_blocks(c);
}

// ---- lm_tri_run, one function per stage ---------------------------------------------------------------------------
// What a run covers: the blocks of the shard's source views [vb, ve) in flat order (source view, neighbour order).
struct RunPlan {
  int vb = 0, ve = 0, ns = 1;    // ns: proposal slots per match row (3 with VP proposals)
  bool exhaustive = false;
  std::vector<lm::RawBlock> blk; // the blocks in flat order
  std::vector<int64_t> row_off;  // first flat row of every block; row_off[nb] = n_rows
  int nb = 0, n_groups = 1;      // blocks, pipeline groups
  int64_t n_rows = 0;
  std::vector<int64_t> chunk_off; // first row chunk (lm::kRowChunk rows) of every block; chunk_off[nb] = chunks
  std::vector<int64_t> tab_off;   // [V+1] first count-table entry of every view of the shard (lines x chunks)
};

// What one attempt of the run queued (a staging overflow repeats the run once): whether tri_node_kernel's fast
// instantiation runs, its staging capacity (candidate slots per node), the launches, the groups that ran the kernel.
struct Attempt {
  bool fast = false;
  int cap = 0, launches = 0;
  std::vector<char> group_has_kernel;
};

static int plan_run(const lm_ctx &c, RunPlan &r) {
  r.vb = std::max(0, c.shard_begin);
  r.ve = (c.shard_end < 0) ? c.V : std::min(c.V, c.shard_end);
  // (lm_tri_set_shard may precede the scene upload: the shard is checked against the scene here)
  if (r.vb > r.ve) return fail(LM_ERR_INVALID, "shard begins after its end or after the last view");
  r.exhaustive = c.any_exhaustive;
  r.ns = (c.cfg.use_vp && !c.cfg.disable_vp_triangulation && c.have_vps) ? 3 : 1;
  for (const lm::RawBlock &b : c.blocks)
    if (b.src_view >= r.vb && b.src_view < r.ve) r.blk.push_back(b);
  std::stable_sort(r.blk.begin(), r.blk.end(), [&r](const lm::RawBlock &a, const lm::RawBlock &b) {
    if (a.src_view != b.src_view) return a.src_view < b.src_view;
    if (r.exhaustive) return a.order < b.order;
    return a.ng_view < b.ng_view;
  });
  r.nb = (int)r.blk.size();
  r.row_off.assign(r.nb + 1, 0);
  for (int i = 0; i < r.nb; ++i) r.row_off[i + 1] = r.row_off[i] + r.blk[i].n_rows;
  r.n_rows = r.row_off[r.nb];
  // the sort and scan item counts are 32-bit signed
  if (r.n_rows >= ((int64_t)1 << 31) - 64) return fail(LM_ERR_INVALID, "more than 2^31 match rows in one run (shard the scene by source image)");
  r.n_groups = r.exhaustive ? 1 : (int)std::max<int64_t>(1, std::min<int64_t>(c.pipeline_groups, r.n_rows >> 16));
  // the sizes of the chunk and count tables that queue_block_tables derives on the device
  r.chunk_off.assign(r.nb + 1, 0);
  for (int i = 0; i < r.nb; ++i) r.chunk_off[i + 1] = r.chunk_off[i] + (r.blk[i].n_rows + lm::kRowChunk - 1) / lm::kRowChunk;
  r.tab_off.assign(c.V + 1, 0);
  for (int v = r.vb, i = 0; v < r.ve; ++v) {
    const int64_t k = r.chunk_off[i];
    while (i < r.nb && r.blk[i].src_view == v) ++i;
    r.tab_off[v + 1] = r.tab_off[v] + (c.line_off[v + 1] - c.line_off[v]) * (r.chunk_off[i] - k);
  }
  if (r.tab_off[r.ve] >= ((int64_t)1 << 31) - 64)
    return fail(LM_ERR_INVALID, "more than 2^31 (line, row chunk) counts in one run (shard the scene by source image)");
  return LM_OK;
}

// Every device buffer and event of the run but the slab, whose size depends on the staging capacity.
static int ensure_run_buffers(lm_ctx *c, const RunPlan &r) {
  const int nb = r.nb, n_all = (int)c->blocks.size();
  const int64_t rows = std::max<int64_t>(r.n_rows, 1), slots = std::max<int64_t>(r.n_rows * r.ns, 1);
  const int64_t n_shard_nodes = c->node_end - c->node_begin;
  CU(c->d_blk_row_off.ensure(8 * (nb + 1)));
  CU(c->d_blk_src.ensure(4 * std::max(nb + 1, 2)));
  CU(c->d_blk_ng.ensure(4 * std::max(nb + 1, 2)));
  CU(c->d_blk_pair_off.ensure(8 * std::max(nb, 1)));
  CU(c->d_row_ng.ensure(4 * rows));
  CU(c->d_blk_chunks.ensure(4 * (nb + 2))); CU(c->d_blk_chunk_off.ensure(4 * (nb + 2)));
  CU(c->d_view_chunk_off.ensure(4 * (c->V + 1))); CU(c->d_view_ent.ensure(4 * (c->V + 1)));
  CU(c->d_view_tab_off.ensure(4 * (c->V + 1))); CU(c->d_view_row_off.ensure(8 * (c->V + 1)));
  if (!r.exhaustive) {
    const int64_t ent = std::max<int64_t>(r.tab_off[r.ve], 1);
    CU(c->d_row_cnt.ensure(2 * ent)); CU(c->d_row_pos.ensure(4 * ent));
  }
  CU(c->d_node_row_off.ensure(4 * (c->n_nodes + 2)));
  CU(c->d_scalars.ensure(1024));
  CU(c->d_nodes.ensure(sizeof(lm::NodeRecord) * std::max<int64_t>(c->n_nodes, 1)));
  CU(c->d_row_state.ensure(slots));
  if (c->cfg.debug_mode) CU(c->d_row_cand.ensure(80 * slots));
  CU(c->d_blk_rows.ensure(8 * (nb + 2)));
  if (n_all) {
    CU(c->d_bkey.ensure(4 * n_all)); CU(c->d_bkey2.ensure(4 * n_all));
    CU(c->d_bval.ensure(4 * n_all)); CU(c->d_bval2.ensure(4 * n_all));
  }
  for (cudaEvent_t e; (int)c->evk.size() < 2 * r.n_groups; c->evk.push_back(e)) CU(cudaEventCreate(&e));
  for (cudaEvent_t e; (int)c->evp.size() < r.n_groups; c->evp.push_back(e))
    CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  const size_t shard_bytes = 4 * (n_shard_nodes + 2);
  CU(c->d_nvalid.ensure(shard_bytes)); CU(c->d_local_off.ensure(shard_bytes)); CU(c->d_edge_off.ensure(shard_bytes));
  CU(c->d_edge_ng.ensure(4 * slots));
  return LM_OK;
}

// The shard's block tables, derived on the prepare stream from the descriptors uploaded with the matches (no transfer
// now): keys by (source view, neighbour order), CUB sort, gather, the exclusive scans of the rows and row chunks, and
// the per-view chunk, row and count-table offsets.
static lm::RowTables row_tables(const lm_ctx &c, const RunPlan &r) {
  lm::RowTables t;
  t.blk_row_off = c.d_blk_row_off.as<int64_t>();
  t.blk_src = c.d_blk_src.as<int32_t>();
  t.blk_ng = c.d_blk_ng.as<int32_t>();
  t.blk_pair_off = c.d_blk_pair_off.as<int64_t>();
  t.blk_chunk_off = c.d_blk_chunk_off.as<int32_t>();
  t.nb = r.nb;
  t.line_off = c.d_line_off.as<int64_t>();
  t.view_chunk_off = c.d_view_chunk_off.as<int32_t>();
  t.view_tab_off = c.d_view_tab_off.as<int32_t>();
  t.view_row_off = c.d_view_row_off.as<int64_t>();
  return t;
}

static int queue_block_tables(lm_ctx *c, const RunPlan &r) {
  cudaStream_t sp = c->prep_stream;
  const int nb = r.nb, n_all = (int)c->blocks.size();
  if (n_all) {
    // the descriptors travel on the copy stream ahead of their matches (bulk add: ahead of all matches)
    if (c->ev_raw) CU(cudaStreamWaitEvent(sp, c->ev_raw, 0));
    lm::launch_block_keys(c->d_raw_blocks.as<lm::RawBlock>(), n_all, r.vb, r.ve, r.exhaustive ? 1 : 0,
                          c->d_bkey.as<uint32_t>(), c->d_bval.as<uint32_t>(), sp);
    cub::DoubleBuffer<uint32_t> bk(c->d_bkey.as<uint32_t>(), c->d_bkey2.as<uint32_t>());
    cub::DoubleBuffer<uint32_t> bv(c->d_bval.as<uint32_t>(), c->d_bval2.as<uint32_t>());
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, bk, bv, n_all, 0, 32, sp); }));
    lm::launch_block_gather(c->d_raw_blocks.as<lm::RawBlock>(), bv.Current(), nb, c->d_blk_src.as<int32_t>(),
                            c->d_blk_ng.as<int32_t>(), c->d_blk_pair_off.as<int64_t>(), c->d_blk_rows.as<int64_t>(),
                            c->d_blk_chunks.as<int32_t>(), sp);
  } else {
    lm::launch_zero_words(c->d_blk_rows.p, 4, sp);
    lm::launch_zero_words(c->d_blk_chunks.p, 2, sp);
  }
  CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) {
    return cub::DeviceScan::ExclusiveSum(t, b, c->d_blk_rows.as<int64_t>(), c->d_blk_row_off.as<int64_t>(), nb + 1, sp);
  }));
  CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) {
    return cub::DeviceScan::ExclusiveSum(t, b, c->d_blk_chunks.as<int32_t>(), c->d_blk_chunk_off.as<int32_t>(), nb + 1, sp);
  }));
  const lm::RowTables t = row_tables(*c, r);
  int32_t *ent = c->d_view_ent.as<int32_t>();
  lm::launch_view_tables(t, r.vb, r.ve, ent, sp);
  CU(cub_call(c->d_sort_tmp, [&](void *tmp, size_t &b) {
    return cub::DeviceScan::ExclusiveSum(tmp, b, ent + r.vb, c->d_view_tab_off.as<int32_t>() + r.vb, r.ve - r.vb + 1, sp);
  }));
  return LM_OK;
}

// The node kernel's parameters that come from the context and the configuration, including the constants derived from
// the configuration. queue_group sets the per-group ones (node range, staging capacity, slab).
static lm::TriParams make_tri_params(const lm_ctx &c, int ns) {
  lm::TriParams p;
  memset(&p, 0, sizeof(p));
  p.views = c.d_views.as<lm::ViewD>();
  p.segs = c.d_segs.as<double4>();
  p.node_view = c.d_node_view.as<uint16_t>();
  p.line_off = c.d_line_off.as<int64_t>();
  p.node_row_off = c.d_node_row_off.as<uint32_t>();
  p.nodes = c.d_nodes.as<lm::NodeRecord>();
  p.row_state = c.d_row_state.as<uint8_t>();
  p.row_cand = c.cfg.debug_mode ? c.d_row_cand.as<double>() : nullptr;
  p.row_ng = c.d_row_ng.as<uint32_t>();
  // d_scalars words: [1] index error, [2] staging overflow, bytes 16..47 counters, words [16 + g] largest node of group g
  p.counters = reinterpret_cast<unsigned long long *>(c.d_scalars.as<char>() + 16);
  p.overflow = c.d_scalars.as<int>() + 2;
  p.node_begin = c.node_begin;
  p.node_end = c.node_end;
  const lm_tri_config &g = c.cfg;
  p.min_length_2d = g.min_length_2d; p.line_tri_angle_threshold = g.line_tri_angle_threshold;
  p.IoU_threshold = g.IoU_threshold; p.sensitivity_threshold = g.sensitivity_threshold; p.var2d = g.var2d;
  p.fullscore_th = g.fullscore_th; p.max_valid_conns = g.max_valid_conns;
  p.use_endpoints_triangulation = g.use_endpoints_triangulation; p.disable_algebraic = g.disable_algebraic_triangulation;
  p.use_vp = (ns == 3); p.disable_vp = g.disable_vp_triangulation;
  p.vp_label = c.d_vp_label.as<int32_t>(); p.vp_off = c.d_vp_voff.as<int64_t>(); p.vps = c.d_vp_vps.as<double>();
  p.ranges_flag = c.ranges_flag;
  for (int i = 0; i < 3; ++i) { p.rlo[i] = c.rlo[i]; p.rhi[i] = c.rhi[i]; }
  p.l2d = to_dev<double>(g.linker2d);
  lm_linker_config l3 = g.linker3d; // set_to_shared_parent_scoring (line_linker.h:115-121)
  l3.use_angle = 1; l3.use_overlap = 0; l3.use_perp = 0; l3.use_innerseg = 0; l3.use_scaleinv = 1;
  p.l3d = to_dev<double>(l3);
  const double kPi = 3.14159265358979323846;
  const double t3 = p.l3d.th_angle, t2 = p.l2d.th_angle;
  p.cos_th3d_f = (t3 >= 90.0) ? -1.0f : (float)(std::cos(t3 * kPi / 180.0) - 4e-6);
  const double c2 = (t2 >= 90.0) ? 0.0 : std::cos(t2 * kPi / 180.0);
  p.cos2_th2d = c2 * c2;
  p.th_perp2_2d = p.l2d.th_perp * p.l2d.th_perp;
  const double ta = p.line_tri_angle_threshold, tsn = p.sensitivity_threshold;
  p.tri_poly_ok = (ta > 0.0 && ta < 90.0);
  p.sens_poly_ok = (tsn > 0.0 && tsn < 90.0);
  p.sin2_tri = std::sin(ta * kPi / 180.0) * std::sin(ta * kPi / 180.0);
  p.sin2_sens = std::sin(tsn * kPi / 180.0) * std::sin(tsn * kPi / 180.0);
  p.fast_forms = (p.l2d.use_innerseg || getenv("LIMAP_B200_REFERENCE_FORMS")) ? 0 : 1;
  p.inv_sig_a3 = 1.0 / (p.l3d.th_angle * p.l3d.mult);
  p.inv_sig_s3 = 1.0 / (p.l3d.th_scaleinv * p.l3d.mult);
  p.inv_sig_a2 = 1.0 / (p.l2d.th_angle * p.l2d.mult);
  p.inv_sig_p2 = 1.0 / (p.l2d.th_perp * p.l2d.mult);
  p.q_cut3 = -2.0 * std::log(p.l3d.score_th) * (1.0 + 1e-9);
  p.q_cut3_lo = -2.0 * std::log(p.l3d.score_th) * (1.0 - 1e-9);
  p.q_cut2 = -2.0 * std::log(p.l2d.score_th) * (1.0 + 1e-9);
  p.q_cut2_lo = -2.0 * std::log(p.l2d.score_th) * (1.0 - 1e-9);
  p.inv_smart_den2 = 1.0 / (p.l2d.th_smartoverlap - p.l2d.th_overlap);
  return p;
}

// Results outside the shard (filled by lm_tri_import_nodes in a multi-GPU run) start from the empty record, so a
// getter never sees uninitialised memory; done once per scene/shard, imports survive later runs.
static int clear_outside_shard(lm_ctx *c) {
  if (c->outside_shard_clean || (c->node_begin <= 0 && c->node_end >= c->n_nodes)) return LM_OK;
  cudaStream_t s = c->stream;
  if (c->node_begin > 0) {
    CU(cudaMemsetAsync(c->d_nodes.p, 0, sizeof(lm::NodeRecord) * c->node_begin, s));
    CU(cudaMemsetAsync(c->d_node_row_off.p, 0, 4 * c->node_begin, s));
  }
  if (c->node_end < c->n_nodes) {
    CU(cudaMemsetAsync(c->d_nodes.as<lm::NodeRecord>() + c->node_end, 0, sizeof(lm::NodeRecord) * (c->n_nodes - c->node_end), s));
    CU(cudaMemsetAsync(c->d_node_row_off.as<uint32_t>() + c->node_end + 1, 0, 4 * (c->n_nodes - c->node_end), s));
  }
  c->outside_shard_clean = true;
  return LM_OK;
}

static int round_cap(int64_t n, int step) { return (int)std::max<int64_t>(step, (n + step - 1) / step * step); }

// The staging capacity of the node kernel (candidates per node held in shared memory) comes from the previous run
// (default: 224). A first exhaustive run knows it on the host: every node sees all lines of every neighbour.
static int initial_cap(const lm_ctx &c, const RunPlan &r, bool fast, int &cap) {
  const int step = lm::tri_cap_step(fast);
  cap = c.cap_hint > 0 ? round_cap(c.cap_hint, step) : 224;
  if (!r.exhaustive || c.cap_hint != 0) return LM_OK;
  int64_t mr = 0, cur = 0;
  int cur_src = -1;
  for (const lm::RawBlock &b : r.blk) {
    if (b.src_view != cur_src) { cur_src = b.src_view; cur = 0; }
    cur += c.line_off[b.ng_view + 1] - c.line_off[b.ng_view];
    mr = std::max(mr, cur);
  }
  if (mr * r.ns > 65535) return fail(LM_ERR_INVALID, "more than 65535 candidates possible for one 2D line");
  cap = round_cap(mr * r.ns, step);
  return LM_OK;
}

// First block after pipeline group g, which starts at block b0. Small groups at both ends (smoothstep): the first one is
// the only one whose matches nothing else can hide, the last one is the only one whose results nothing else can hide.
// A group finishes its last source image.
static int group_end(const RunPlan &r, int g, int b0) {
  if (g + 1 >= r.n_groups) return r.nb;
  const double tg = (g + 1.0) / r.n_groups;
  const int64_t target = (int64_t)((double)r.n_rows * (tg * tg * (3.0 - 2.0 * tg)));
  int b1 = b0;
  while (b1 < r.nb && r.row_off[b1] < target) ++b1;
  while (b1 < r.nb && b1 > 0 && r.blk[b1].src_view == r.blk[b1 - 1].src_view) ++b1;
  return b1;
}

// Pipeline group g: blocks [b0, b1), source views [v0, v1). The prepare stream waits for the group's matches, puts its
// rows in node order and finds every node's rows; the engine's stream runs the node kernel between two timing events;
// the output stream compacts the group's valid connections and copies its records into the node sink.
static int queue_group(lm_ctx *c, const RunPlan &r, lm::TriParams p, int g, int b0, int b1, int v0, int v1, Attempt &a) {
  cudaStream_t s = c->stream, sp = c->prep_stream;
  const int64_t rb = r.row_off[b0], re = r.row_off[b1];
  const int64_t node_lo = c->line_off[v0], node_hi = c->line_off[v1];
  if (!r.exhaustive && re > rb) {
    int64_t need = 0;
    for (int b = b0; b < b1; ++b) need = std::max(need, r.blk[b].pair_off + r.blk[b].n_rows);
    for (const auto &ch : c->chunks) // chunks complete in order: wait for the first one that covers `need`
      if (ch.row_end >= need) { CU(cudaStreamWaitEvent(sp, ch.ev, 0)); break; }
  }
  // rows in node order (tri_plumbing.cu): matches count the rows of every (line, row chunk), scan the group's slice of
  // the count table and place every chunk's rows; exhaustive matching places every row in closed form
  const lm::RowTables t = row_tables(*c, r);
  uint32_t *row_ng = c->d_row_ng.as<uint32_t>();
  const uint32_t *pos = c->d_row_pos.as<uint32_t>();
  const int k0 = (int)r.chunk_off[b0], n_chunks = (int)(r.chunk_off[b1] - r.chunk_off[b0]);
  const int64_t t0 = r.tab_off[v0], t1 = r.tab_off[v1];
  int nl_max = 0;
  for (int v = v0; v < v1; ++v) nl_max = std::max(nl_max, (int)(c->line_off[v + 1] - c->line_off[v]));
  if (re > rb && !r.exhaustive) {
    CU(lm::launch_row_count(t, c->d_pairs.as<int32_t>(), k0, n_chunks, nl_max, c->d_row_cnt.as<uint16_t>(),
                            c->d_scalars.as<int>() + 1, sp));
    CU(cub_call(c->d_sort_tmp, [&](void *tmp, size_t &b) {
      return cub::DeviceScan::ExclusiveScan(tmp, b, c->d_row_cnt.as<uint16_t>() + t0, c->d_row_pos.as<uint32_t>() + t0,
                                            ::cuda::std::plus<uint32_t>(), (uint32_t)0, (int)(t1 - t0), sp);
    }));
    a.launches += 3; // count, the scan's two kernels
  }
  lm::launch_node_row_off(t, pos, t1, rb, re, node_lo, node_hi, c->V, r.exhaustive ? 1 : 0,
                          c->d_node_row_off.as<uint32_t>(), c->d_scalars.as<unsigned int>() + 16 + g, sp);
  ++a.launches;
  if (re > rb) {
    if (r.exhaustive)
      lm::launch_place_exhaustive(t, r.n_rows, row_ng, sp);
    else
      CU(lm::launch_row_place(t, c->d_pairs.as<int32_t>(), k0, n_chunks, nl_max, pos, rb, row_ng, sp));
    ++a.launches;
  }
  CU(cudaEventRecord(c->evp[g], sp));
  CU(cudaStreamWaitEvent(s, c->evp[g], 0));
  p.node_begin = node_lo; p.node_end = node_hi; p.cap = a.cap;
  const int64_t n_group_nodes = node_hi - node_lo;
  size_t smem = lm::tri_smem_bytes(a.cap, a.fast);
  int grid;
  if (smem <= (size_t)std::max(0, c->max_smem_optin - 1024)) {
    p.use_slab = 0;
    grid = (int)std::min<int64_t>(n_group_nodes, (int64_t)1 << 30);
  } else {
    // nodes larger than shared memory (exhaustive matching): persistent CTAs with a global staging slab
    p.use_slab = 1;
    grid = (int)std::min<int64_t>(n_group_nodes, (int64_t)c->sm_count * 4);
    p.slab_stride = (int64_t)((smem + 255) / 256 * 256);
    CU(c->d_slab.ensure((size_t)p.slab_stride * std::max(grid, 1)));
    p.slab = c->d_slab.as<char>();
    smem = 0;
  }
  if (n_group_nodes <= 0) return LM_OK;
  CU(cudaEventRecord(c->evk[2 * g], s));
  CU(lm::launch_tri_node_kernel(p, grid, smem, s));
  CU(cudaEventRecord(c->evk[2 * g + 1], s));
  a.group_has_kernel[g] = 1;
  ++a.launches;
  // valid_edges_ of the group in compact form, under the node kernels of the later groups: per-node counts -> exclusive
  // scan -> ordered scatter at the global offsets
  cudaStream_t so = c->out_stream;
  CU(cudaStreamWaitEvent(so, c->evk[2 * g + 1], 0));
  uint32_t *nv = c->d_nvalid.as<uint32_t>() + (node_lo - c->node_begin);
  lm::launch_extract_nvalid(p.nodes, node_lo, n_group_nodes, nv, so);
  // (d_scan_tmp, not d_sort_tmp: the preparation stream scans the next group's counts meanwhile)
  CU(cub_call(c->d_scan_tmp, [&](void *t, size_t &b) {
    return cub::DeviceScan::ExclusiveSum(t, b, nv, c->d_local_off.as<uint32_t>(), (int)(n_group_nodes + 1), so);
  }));
  lm::launch_group_edges(p.row_state, p.row_ng, p.node_row_off, c->d_local_off.as<uint32_t>(),
                         c->d_scalars.as<unsigned int>() + 80, g, c->node_begin, node_lo, n_group_nodes, r.ns,
                         c->d_edge_off.as<uint32_t>(), c->d_edge_ng.as<uint32_t>(), so);
  a.launches += 4;
  if (c->node_sink) // the group's records go to the caller's buffer under the kernels of the later groups
    CU(cudaMemcpyAsync(c->node_sink + sizeof(lm::NodeRecord) * node_lo, c->d_nodes.as<lm::NodeRecord>() + node_lo,
                       sizeof(lm::NodeRecord) * n_group_nodes, cudaMemcpyDeviceToHost, c->out_stream));
  return LM_OK;
}

// The end of an attempt: the engine's stream waits for the output stream, then the one read-back of the run (error and
// overflow flags, counters, largest node per group) and its one host synchronisation. Sets `overflow` when some node did
// not fit the staging capacity: the hint is then exact, and the stats are left to the repeated attempt.
static int finish_run(lm_ctx *c, const RunPlan &r, const Attempt &a, bool &overflow) {
  cudaStream_t s = c->stream;
  CU(cudaGetLastError());
  // the engine's stream ends the run: whatever follows on it (getters, exchange) sees the compact connections
  CU(cudaEventRecord(c->ev_run_begin, c->out_stream));
  CU(cudaStreamWaitEvent(s, c->ev_run_begin, 0));
  CU(cudaEventRecord(c->ev1, s));
  const unsigned int *hs = c->h_pin;
  CU(cudaMemcpyAsync(c->h_pin, c->d_scalars.p, 512, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  CU(cudaStreamSynchronize(c->copy_stream)); // uploads of images outside this shard may still be in flight
  CU(cudaStreamSynchronize(c->out_stream));
  c->stats.n_kernel_launches += a.launches;
  if (hs[1] == 1)
    return fail(LM_ERR_INVALID, "IndexError! Out-of-index matches exist (line_id >= number of lines of the image). "
                                "Please make sure you are reusing the correct descriptors and matches.");
  if (hs[1] == 2) return fail(LM_ERR_INVALID, "IndexError! Out-of-index neighbor line id in matches.");
  int max_rows_all = 0;
  for (int g = 0; g < r.n_groups; ++g) max_rows_all = std::max(max_rows_all, (int)hs[16 + g]);
  if ((int64_t)max_rows_all * r.ns > 65535) return fail(LM_ERR_INVALID, "more than 65535 candidates possible for one 2D line");
  c->cap_hint = round_cap((int64_t)max_rows_all * r.ns, lm::tri_cap_step(a.fast));
  overflow = hs[2] != 0;
  if (overflow) return LM_OK;
  float ms = 0;
  CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  double node_kernel_ms = 0;
  for (int g = 0; g < r.n_groups; ++g)
    if (a.group_has_kernel[g]) {
      float msk = 0;
      CU(cudaEventElapsedTime(&msk, c->evk[2 * g], c->evk[2 * g + 1]));
      node_kernel_ms += msk;
    }
  c->stats.max_rows_per_node = max_rows_all;
  c->stats.last_node_kernel_ms = node_kernel_ms;
  const unsigned long long *cnt = reinterpret_cast<const unsigned long long *>(hs + 4);
  c->stats.n_rows = r.n_rows;
  c->stats.n_candidates = (int64_t)cnt[0];
  c->stats.n_valid_edges = (int64_t)cnt[1];
  c->stats.n_pairs_gated = (int64_t)cnt[2];
  c->stats.n_pairs_exact = (int64_t)cnt[3];
  c->stats.last_run_ms = ms;
  c->ran = true;
  return LM_OK;
}

int lm_tri_run(lm_ctx *c) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_scene) return fail(LM_ERR_STATE, "no scene uploaded");
  if (!c->have_cfg) return fail(LM_ERR_STATE, "lm_tri_configure must precede lm_tri_run");
  CU(cudaSetDevice(c->device));
  RunPlan plan;
  int rc = plan_run(*c, plan);
  if (rc) return rc;
  c->n_rows = plan.n_rows;
  c->ns = plan.ns;
  c->node_begin = c->line_off[plan.vb];
  c->node_end = c->line_off[plan.ve];
  c->h_nodes_valid = c->h_rows_valid = c->h_edges_valid = false;
  c->edges_collected = c->edges_count_on_device = c->edges_overflowed = false;
  c->tracks.clear();
  if ((rc = ensure_run_buffers(c, plan))) return rc;
  const lm::TriParams p = make_tri_params(*c, plan.ns);
  // Two compute streams: `sp` prepares the rows of a pipeline group (node order, node offsets), `s` runs the node
  // kernels. The preparation of group g+1 is queued right behind that of group g, so it executes under the node kernel of
  // group g; everything `sp` touches is per-group slices, its own scratch, or is read by `s` only after the group's event.
  cudaStream_t s = c->stream, sp = c->prep_stream;
  // The kernel flags the nodes that do not fit the staging capacity, and the run is then repeated once at the exact
  // size. No read-back, no host synchronisation until everything of an attempt is queued.
  for (int attempt = 0;; ++attempt) {
    CU(cudaEventRecord(c->ev0, s));
    CU(cudaEventRecord(c->ev_run_begin, s)); // whatever the caller queued on the engine's stream comes first
    CU(cudaStreamWaitEvent(sp, c->ev_run_begin, 0));
    // scene tables / VP tables travel on the copy stream (see lm_ctx::ev_scene)
    CU(cudaStreamWaitEvent(sp, c->ev_scene, 0));
    CU(cudaStreamWaitEvent(s, c->ev_scene, 0));
    lm::launch_zero_words(c->d_scalars.p, 256, sp);
    if ((rc = queue_block_tables(c, plan))) return rc;
    if ((rc = clear_outside_shard(c))) return rc;
    Attempt a;
    a.fast = lm::tri_fast(p);
    if ((rc = initial_cap(*c, plan, a.fast, a.cap))) return rc;
    a.group_has_kernel.assign(plan.n_groups, 0);
    // groups of whole source images: row placement + node kernel of group g overlap the upload of group g+1
    for (int g = 0, b0 = 0, v0 = plan.vb; g < plan.n_groups; ++g) {
      const int b1 = group_end(plan, g, b0), v1 = (b1 < plan.nb) ? plan.blk[b1].src_view : plan.ve;
      if ((rc = queue_group(c, plan, p, g, b0, b1, v0, v1, a))) return rc;
      b0 = b1;
      v0 = v1;
    }
    bool overflow = false;
    if ((rc = finish_run(c, plan, a, overflow))) return rc;
    if (!overflow) return LM_OK;
    if (attempt > 0) return fail(LM_ERR_STATE, "node staging overflow after resizing");
  }
}

int lm_tri_get_stats(lm_ctx *c, lm_tri_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->stats;
  return LM_OK;
}

int lm_tri_get_best(lm_ctx *c, int32_t img_id, double *out_line, int32_t *out_ng, int32_t *out_ncand) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int rc = ensure_ran(c);
  if (rc) return rc;
  if ((rc = fetch_nodes(c))) return rc;
  auto it = c->id2view.find(img_id);
  if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id");
  const int v = it->second;
  for (int64_t n = c->line_off[v]; n < c->line_off[v + 1]; ++n) {
    const lm::NodeRecord &r = c->h_nodes[n];
    const int64_t l = n - c->line_off[v];
    for (int k = 0; k < 9; ++k) out_line[10 * l + k] = r.line[k];
    out_line[10 * l + 9] = r.score;
    out_ng[2 * l] = r.n_cand ? c->img_ids[r.ng_view] : 0;
    out_ng[2 * l + 1] = r.ng_line;
    if (out_ncand) out_ncand[l] = r.n_cand;
  }
  return LM_OK;
}

int64_t lm_tri_get_valid_edges(lm_ctx *c, int32_t img_id, int64_t *off, int32_t *edges) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int rc = ensure_ran(c);
  if (rc) return rc;
  if ((rc = fetch_edges(c))) return rc;
  auto it = c->id2view.find(img_id);
  if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id");
  const int v = it->second;
  const int64_t L = c->line_off[v + 1] - c->line_off[v];
  const bool in_shard = c->line_off[v] >= c->node_begin && c->line_off[v + 1] <= c->node_end;
  int64_t n_out = 0;
  for (int64_t l = 0; l < L; ++l) {
    if (off) off[l] = n_out;
    if (!in_shard) continue;
    const int64_t i = c->line_off[v] + l - c->node_begin;
    for (uint32_t e = c->h_edge_off[i]; e < c->h_edge_off[i + 1]; ++e) {
      if (edges) {
        edges[2 * n_out] = c->img_ids[c->h_edge_ng[e] >> 16];
        edges[2 * n_out + 1] = (int32_t)(c->h_edge_ng[e] & 0xffffu);
      }
      ++n_out;
    }
  }
  if (off) off[L] = n_out;
  return n_out;
}

int lm_tri_get_cands_node(lm_ctx *c, int32_t img_id, int32_t line_id, int32_t cap, double *out_line, int32_t *out_ng) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (!c->have_cfg || !c->cfg.debug_mode) return fail(LM_ERR_STATE, "GetScoredTrisNode needs debug_mode");
  int rc = ensure_ran(c);
  if (rc) return rc;
  if ((rc = fetch_rows(c))) return rc;
  auto it = c->id2view.find(img_id);
  if (it == c->id2view.end()) return fail(LM_ERR_INVALID, "unknown image id");
  const int64_t n = c->line_off[it->second] + line_id;
  if (line_id < 0 || n >= c->line_off[it->second + 1]) return fail(LM_ERR_INVALID, "line id out of range");
  int k = 0;
  for (int64_t q = (int64_t)c->h_node_row_off[n] * c->ns; q < (int64_t)c->h_node_row_off[n + 1] * c->ns; ++q) {
    if (c->h_row_state[q] == 0) continue;
    const uint32_t r = (uint32_t)(q / c->ns);
    if (k < cap) {
      for (int t = 0; t < 10; ++t) out_line[10 * k + t] = c->h_row_cand[(size_t)q * 10 + t];
      out_ng[2 * k] = c->img_ids[c->h_row_ng[r] >> 16];
      out_ng[2 * k + 1] = (int32_t)(c->h_row_ng[r] & 0xffffu);
    }
    ++k;
  }
  return k;
}

int64_t lm_tri_num_nodes(lm_ctx *c) { return c ? c->n_nodes : 0; }
int64_t lm_scene_node_offset(lm_ctx *c, int32_t v) {
  if (!c || v < 0 || v > c->V) return -1;
  return c->line_off[v];
}
int lm_tri_export_nodes(lm_ctx *c, int64_t b, int64_t e, void *d_out) {
  if (!c || !d_out || b < 0 || e > c->n_nodes || b > e) return fail(LM_ERR_INVALID, "bad node range");
  int rc = ensure_ran(c);
  if (rc) return rc;
  CU(cudaMemcpyAsync(d_out, c->d_nodes.as<lm::NodeRecord>() + b, sizeof(lm::NodeRecord) * (e - b),
                     cudaMemcpyDeviceToDevice, c->stream));
  return LM_OK;
}
int lm_tri_import_nodes(lm_ctx *c, int64_t b, int64_t e, const void *d_in) {
  if (!c || !d_in || b < 0 || e > c->n_nodes || b > e) return fail(LM_ERR_INVALID, "bad node range");
  CU(c->d_nodes.ensure(sizeof(lm::NodeRecord) * std::max<int64_t>(c->n_nodes, 1)));
  CU(cudaMemcpyAsync(c->d_nodes.as<lm::NodeRecord>() + b, d_in, sizeof(lm::NodeRecord) * (e - b),
                     cudaMemcpyDeviceToDevice, c->stream));
  c->h_nodes_valid = false;
  return LM_OK;
}

int64_t lm_tri_num_valid_edges(lm_ctx *c) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  int rc = ensure_ran(c);
  if (rc) return rc;
  if ((rc = collect_edges(c))) return rc;
  return c->n_edges_dev;
}
int lm_tri_export_edges(lm_ctx *c, void *d_out) {
  if (!c || !d_out) return fail(LM_ERR_INVALID, "NULL argument");
  int rc = ensure_ran(c);
  if (rc) return rc;
  if ((rc = collect_edges(c))) return rc;
  if (c->n_edges_dev)
    CU(cudaMemcpyAsync(d_out, c->d_edges.p, 16 * c->n_edges_dev, cudaMemcpyDeviceToDevice, c->stream));
  return LM_OK;
}
int lm_tri_import_edges(lm_ctx *c, int64_t n, const void *d_in, int32_t append) {
  if (!c || (n && !d_in)) return fail(LM_ERR_INVALID, "NULL argument");
  if (append) { // after this run's own valid connections (collected now if no getter did)
    int rc = ensure_ran(c);
    if (!rc) rc = collect_edges(c);
    if (rc) return rc;
  }
  const int64_t base = append ? c->n_edges_dev : 0;
  CU(c->d_edges.grow_keep((size_t)(base + n) * 16, 16 * base, c->stream));
  if (n) CU(cudaMemcpyAsync(c->d_edges.as<char>() + 16 * base, d_in, 16 * n, cudaMemcpyDeviceToDevice, c->stream));
  c->n_edges_dev = base + n;
  c->edges_collected = true;
  return LM_OK;
}

int64_t lm_tri_gather_message_bytes(int64_t max_nodes, int64_t cap_edges) {
  if (max_nodes < 0 || cap_edges < 0) return fail(LM_ERR_INVALID, "bad sizes");
  return (16 + max_nodes * (int64_t)sizeof(lm::NodeRecord) + cap_edges * 8 + 15) / 16 * 16;
}
int lm_tri_pack_message(lm_ctx *c, int64_t max_nodes, int64_t cap_edges, void *d_msg) {
  if (!c || !d_msg) return fail(LM_ERR_INVALID, "NULL argument");
  int rc = ensure_ran(c);
  if (rc) return rc;
  const int64_t n = c->node_end - c->node_begin;
  if (n > max_nodes) return fail(LM_ERR_INVALID, "shard has more nodes than the message holds");
  lm::launch_gather_pack(c->d_nodes.as<lm::NodeRecord>(), c->node_begin, n, max_nodes, c->d_edge_off.as<uint32_t>(),
                         c->d_edge_ng.as<uint32_t>(), c->d_line_off.as<int64_t>(), cap_edges, static_cast<char *>(d_msg),
                         c->stream);
  CU(cudaGetLastError());
  c->stats.n_kernel_launches += 1;
  return LM_OK;
}
int lm_tri_unpack_messages(lm_ctx *c, int32_t world, const int64_t *rank_node_begin, int64_t max_nodes, int64_t cap_edges,
                           const void *d_msgs) {
  if (!c || !d_msgs || !rank_node_begin || world <= 0 || world > 64) return fail(LM_ERR_INVALID, "bad argument");
  CU(cudaSetDevice(c->device));
  for (int r = 0; r < world; ++r)
    if (rank_node_begin[r] < 0 || rank_node_begin[r] > c->n_nodes) return fail(LM_ERR_INVALID, "bad node range");
  CU(c->d_nodes.ensure(sizeof(lm::NodeRecord) * std::max<int64_t>(c->n_nodes, 1)));
  if ((size_t)world * cap_edges * 16 + 16 > c->d_edges.cap) {
    CU(cudaStreamSynchronize(c->stream));
    CU(c->d_edges.ensure((size_t)world * cap_edges * 16 + 16));
  }
  CU(c->d_gather.ensure(8 * 64 + 64));
  // rank table as kernel-readable memory: tiny, written through pinned memory on the compute stream's own order
  int64_t *h = reinterpret_cast<int64_t *>(c->h_pin + 128); // bytes 512.. of the pinned pad
  for (int r = 0; r < world; ++r) h[r] = rank_node_begin[r];
  if (memcmp(c->gather_tab, h, 8 * world) != 0 || c->gather_world != world) {
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpyAsync(c->d_gather.as<char>() + 64, h, 8 * world, cudaMemcpyHostToDevice, c->copy_stream));
    CU(cudaStreamSynchronize(c->copy_stream));
    memcpy(c->gather_tab, h, 8 * world);
    c->gather_world = world;
  }
  lm::launch_gather_unpack(static_cast<const char *>(d_msgs), world, reinterpret_cast<const int64_t *>(c->d_gather.as<char>() + 64),
                           max_nodes, cap_edges, lm_tri_gather_message_bytes(max_nodes, cap_edges),
                           c->d_nodes.as<lm::NodeRecord>(), c->d_edges.as<int64_t>(), c->d_gather.as<int64_t>(), c->stream);
  CU(cudaGetLastError());
  c->stats.n_kernel_launches += 1;
  c->h_nodes_valid = false;
  c->edges_collected = true;
  c->edges_count_on_device = true;
  return LM_OK;
}
int64_t lm_tri_gather_status(lm_ctx *c, int64_t *n_edges_total) {
  if (!c) return fail(LM_ERR_INVALID, "ctx is NULL");
  if (c->edges_count_on_device) {
    int64_t *h = reinterpret_cast<int64_t *>(c->h_pin + 256);
    CU(cudaMemcpyAsync(h, c->d_gather.p, 16, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    c->n_edges_dev = h[0];
    c->edges_overflowed = h[1] != 0;
    c->edges_count_on_device = false;
  }
  if (n_edges_total) *n_edges_total = c->n_edges_dev;
  // 1: some rank had more valid connections than cap_edges -- repeat the exchange with a larger message
  return c->edges_overflowed ? 1 : 0;
}

} // extern "C"
