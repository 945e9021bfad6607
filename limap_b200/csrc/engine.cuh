// engine.cuh — what the host side of the C ABI (engine.cu and one engine_<stage>.cu per later stage) shares: error
// reporting, device buffers, the context and the host helpers more than one stage uses.
#pragma once
#include "../../include/limap_b200.h"
#include "tri_kernels.cuh"
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

static_assert(sizeof(lm_node_record) == sizeof(lm::NodeRecord), "record layout");

inline thread_local std::string g_err;
inline int fail(int code, const std::string &msg) {
  g_err = msg;
  return code;
}
#define CU(call)                                                                                                    \
  do {                                                                                                              \
    cudaError_t e_ = (call);                                                                                        \
    if (e_ != cudaSuccess)                                                                                          \
      return fail(LM_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                                 \
  } while (0)

// A device allocation with one owner: freed on destruction, moved but never copied.
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; } // (o frees ours)
  ~DevBuf() { release(); }
  // contents are not kept
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // Grow to at least `bytes` keeping the first `keep` bytes: they are copied on `s`, which is then synchronised.
  cudaError_t grow_keep(size_t bytes, size_t keep, cudaStream_t s) {
    if (bytes <= cap) return cudaSuccess;
    DevBuf nb;
    cudaError_t e = nb.ensure(bytes);
    if (e == cudaSuccess && keep) e = cudaMemcpyAsync(nb.p, p, keep, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) *this = std::move(nb);
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// CUB's two-call protocol: f(nullptr, bytes) asks for the scratch size, f(scratch, bytes) runs. Work queued on two
// streams at once needs two scratch buffers.
template <typename F> cudaError_t cub_call(DevBuf &scratch, F f) {
  size_t tmp_bytes = 0;
  cudaError_t e = f(nullptr, tmp_bytes);
  if (e == cudaSuccess) e = scratch.ensure(tmp_bytes);
  if (e == cudaSuccess) e = f(scratch.p, tmp_bytes);
  return e;
}

struct M3h {
  double m[9];
};
M3h quat_to_R(const double q_in[4]);
// Per-view constants (tri_kernels.cuh ViewT) from the reference's camera arrays.
void make_view(int model_id, const double *kv, const double *qv, const double *t, lm::ViewD &d);

template <typename T> lm::LinkerDev<T> to_dev(const lm_linker_config &c) {
  lm::LinkerDev<T> d;
  d.score_th = (T)c.score_th; d.th_angle = (T)c.th_angle; d.th_overlap = (T)c.th_overlap;
  d.th_smartoverlap = (T)c.th_smartoverlap; d.th_smartangle = (T)c.th_smartangle; d.th_perp = (T)c.th_perp;
  d.th_innerseg = (T)c.th_innerseg; d.th_scaleinv = (T)c.th_scaleinv;
  d.mult = (T)(1.0 / std::sqrt(-std::log(c.score_th) * 2.0)); // line_linker.cc:9-13
  d.use_angle = c.use_angle; d.use_overlap = c.use_overlap; d.use_smartangle = c.use_smartangle;
  d.use_perp = c.use_perp; d.use_innerseg = c.use_innerseg; d.use_scaleinv = c.use_scaleinv;
  return d;
}

// LineLinker3d::set_to_spatial_merging (line_linker.h:123-129)
inline lm_linker_config spatial_merging(lm_linker_config l) {
  l.use_angle = 1; l.use_overlap = 1; l.use_perp = 0; l.use_innerseg = 1; l.use_scaleinv = 0;
  return l;
}

struct Track {
  std::vector<int> img, line, node;
  std::vector<int64_t> gid;
  double agg[7];
};

struct AggItem { // one Line3d of a line3d_list: endpoints, uncertainty, score
  const double *l;
  double unc, score;
};

struct lm_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
  // match uploads run on their own stream so that a run can start on the first source images while the rest
  // of the tables is still crossing PCIe
  cudaStream_t copy_stream = nullptr;
  cudaStream_t prep_stream = nullptr; // row expansion + sort of pipeline group g+1 run under the node kernel of group g
  std::vector<cudaEvent_t> evp;       // per pipeline group: rows of the group sorted, node offsets known
  cudaEvent_t ev_run_begin = nullptr;
  cudaStream_t out_stream = nullptr;  // device -> host copies of finished groups (lm_tri_set_node_sink)
  char *node_sink = nullptr;
  DevBuf d_scan_tmp, d_local_off;
  struct CopyChunk { int64_t row_end; cudaEvent_t ev; };
  std::vector<CopyChunk> chunks;
  std::vector<cudaEvent_t> event_pool;
  DevBuf d_raw_blocks, d_bkey, d_bkey2, d_bval, d_bval2, d_blk_rows; // device mirror of `blocks` + sort scratch
  int64_t raw_uploaded = 0;
  cudaEvent_t ev_raw = nullptr; // recorded on the copy stream after the latest descriptor upload
  // Every host->device transfer (scene, VPs, matches) travels on the copy stream; the compute stream only waits
  // for events. A compute stream whose latest operation is itself a host->device copy has its next operations
  // (event records, kernel launches) ordered behind whatever the H2D copy engine is working on -- i.e. behind a
  // bulk match upload issued in between (measured in round 1: ~3 ms per hypersim100 step).
  cudaEvent_t ev_scene = nullptr;
  std::vector<lm::ViewD> h_views;    // staging of the scene tables (kept alive: the copies are asynchronous)
  std::vector<cudaEvent_t> evk;      // per pipeline group: node-kernel begin/end (read after the run's only sync)
  DevBuf d_gather;                   // [0] total edges, [1] overflow flag of the last unpack; +64: rank node table
  int64_t gather_tab[64] = {0};
  int gather_world = 0;
  bool edges_count_on_device = false; // n_edges_dev is still on the device (lm_tri_unpack_messages)
  int cap_hint = 0;                  // staging capacity of the node kernel, from the previous run (0: default)
  bool outside_shard_clean = false;  // node records / row offsets outside the shard were zero-filled
  int sm_count = 132;
  int max_smem_optin = 0;
  // scene
  bool have_scene = false;
  int V = 0;
  std::vector<int> img_ids;
  std::unordered_map<int, int> id2view;
  std::vector<int64_t> line_off;
  int64_t n_nodes = 0;
  DevBuf d_views, d_segs, d_segs_raw, d_node_view, d_line_off, d_img_ids, d_host_edges;
  // config
  bool have_cfg = false;
  lm_tri_config cfg;
  bool ranges_flag = false;
  double rlo[3] = {0, 0, 0}, rhi[3] = {0, 0, 0};
  // InitVPResults
  bool have_vps = false;
  DevBuf d_vp_label, d_vp_voff, d_vp_vps;
  int ns = 1; // proposal slots per match row of the last run (3 with VP proposals)
  // staged matches
  std::vector<lm::RawBlock> blocks; // one per (source image, neighbour) table, in the order they were added
  std::vector<char> image_added;
  DevBuf d_pairs;
  int64_t pairs_rows = 0;
  bool any_exhaustive = false, any_matches = false;
  int shard_begin = 0, shard_end = -1;
  int pipeline_groups = 1; // lm_tri_set_pipeline_groups
  // pinned landing pad of the small device->host reads inside a run (no staging through pageable memory)
  unsigned int *h_pin = nullptr;
  // run buffers
  DevBuf d_blk_row_off, d_blk_src, d_blk_ng, d_blk_pair_off;
  DevBuf d_key, d_key2, d_val, d_val2, d_sort_tmp;
  DevBuf d_node_row_off, d_scalars; // scalars: [0] max_rows(uint) [1] err(int) ; counters at +16
  DevBuf d_nodes, d_row_state, d_row_cand, d_slab;
  DevBuf d_edges, d_edges2, d_edge_keys, d_edge_keys2, d_edge_w, d_edge_cnt;
  DevBuf d_g_flag, d_g_pos, d_g_kc, d_g_wc, d_g_occ, d_g_occ2, d_g_hk, d_g_hk2, d_g_gidx, d_g_gnode, d_g_k1, d_g_k1b, d_g_k2, d_g_k2b;
  DevBuf d_nvalid, d_edge_off, d_edge_ng; // compact valid_edges_ of the shard (node-major, candidate order)
  uint32_t *sorted_val = nullptr;
  uint32_t *sorted_key = nullptr;
  int64_t n_rows = 0;
  int64_t node_begin = 0, node_end = 0;
  bool ran = false;
  lm_tri_stats stats;
  // host caches (filled lazily after a run)
  bool h_nodes_valid = false;
  std::vector<lm::NodeRecord> h_nodes;
  bool h_rows_valid = false;
  std::vector<uint32_t> h_node_row_off, h_row_ng;
  std::vector<uint8_t> h_row_state;
  std::vector<double> h_row_cand;
  bool h_edges_valid = false;
  std::vector<uint32_t> h_edge_off, h_edge_ng;
  int64_t n_edges_dev = 0; // directed valid edges collected on device
  bool edges_collected = false;
  // line BA
  DevBuf d_ba_in, d_ba_blocks, d_ba_out;
  DevBuf d_vp_pts, d_vp_off, d_vp_labels, d_vp_nc, d_vp_ps, d_vp_mat;
  lm_ba_stats ba_stats;
  void *h_ba_pin = nullptr; // pinned landing pad of lm_ba_solve's results
  size_t h_ba_pin_cap = 0;
  lm_vp_stats vp_stats;
  DevBuf d_vp_idx;
  // track filters / remerge
  DevBuf d_mg_in, d_mg_out, d_mg_edges;
  // fit-and-merge (lm_merge_fits_build)
  DevBuf d_fm_in, d_fm_work, d_fm_keys, d_fm_keys2, d_fm_pairs, d_fm_pairs2, d_fm_bn, d_fm_bn2, d_fm_bs, d_fm_bs2, d_fm_sim;
  struct FitMerge {
    std::vector<double> unc, length, sim, track_line;
    std::vector<int64_t> node_line, track_off;
    std::vector<int32_t> edges, track_nodes;
  } fm;
  lm_fit_merge_stats fm_stats = {};
  DevBuf d_sfm_in, d_sfm_keys, d_sfm_keys2, d_sfm_a, d_sfm_b, d_sfm_c, d_sfm_d; // neighbour ranking scratch
  lm_merge_stats mg_stats;
  // tracks
  std::vector<Track> tracks;
  ~lm_ctx();
};

// engine.cu
int ensure_ran(lm_ctx *c);
int fetch_nodes(lm_ctx *c);
int collect_edges(lm_ctx *c);

// engine_tracks.cu
size_t uf_root(size_t i, std::vector<int> &parent);
std::vector<int> greedy_track_labels(const std::vector<uint64_t> &order, const std::vector<int> &image_of, int n_images,
                                     int &n_tracks);
void aggregate_items(const std::vector<AggItem> &it, int num_outliers, double out[7]);
// The greedy edge order (merging.cc:32-34), descending (score, idx0, idx1): two stable LSD radix sorts of n complemented
// keys, by the node keys first, then by the score keys with the node keys carried along. `out` points at the sorted
// node keys (still complemented), in one of the two node buffers.
int sort_greedy_order(DevBuf &scratch, DevBuf &nodes, DevBuf &nodes_alt, DevBuf &score, DevBuf &score_alt, int n,
                      cudaStream_t s, const uint64_t *&out);

// Cyclic Jacobi sweeps of a symmetric 3x3 matrix: the eigenvalues land in ev, the eigenvectors in the columns of V.
inline void jacobi3(const double Ain[3][3], double V[3][3], double ev[3]) {
  double A[3][3];
  memcpy(A, Ain, sizeof(A));
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    double diag = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (off == 0 || off <= 1e-32 * diag) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (A[p][q] == 0) continue;
        double theta = (A[q][q] - A[p][p]) / (2 * A[p][q]);
        double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        double cs = 1 / std::sqrt(t * t + 1), sn = t * cs;
        for (int k = 0; k < 3; ++k) { double a = A[k][p], b = A[k][q]; A[k][p] = cs * a - sn * b; A[k][q] = sn * a + cs * b; }
        for (int k = 0; k < 3; ++k) { double a = A[p][k], b = A[q][k]; A[p][k] = cs * a - sn * b; A[q][k] = sn * a + cs * b; }
        for (int k = 0; k < 3; ++k) { double a = V[k][p], b = V[k][q]; V[k][p] = cs * a - sn * b; V[k][q] = sn * a + cs * b; }
      }
  }
  for (int k = 0; k < 3; ++k) ev[k] = A[k][k];
}
