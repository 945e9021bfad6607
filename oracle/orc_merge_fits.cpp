// orc_merge_fits.cpp — CPU restatement of merging.merging (merging.py:6-21): SetUncertaintySegs3d
// (merging/merging_utils.cc:15-25) and MergeToLineTracks (merging/merging.cc:347-511).
//
// TEST INFRASTRUCTURE (oracle). PARITY PINNED to the reference's compiled MergeToLineTracks through its stored outputs
// (oracle/ref_merge_fits.cpp, tests/golden/ref/merge_to_linetracks_*.npz, tests/test_merge_to_linetracks_oracle.py).
// Built by oracle/merge_fits.py into oracle/_build/liblimap_orc_merge.so; only tests/ and scripts/ load it.
#include "orc_geom.h"
#include "orc_triangulation.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

namespace {

// LineLinker3d::check_connection (base/line_linker.cc:284-304)
bool check_connection3d(const LineLinker3d &lk, const Line3d &l1, const Line3d &l2) {
  const LinkerConfig &c = lk.config;
  if (c.use_angle)
    if (!(compute_angle(l1, l2) <= c.th_angle)) return false;
  if (c.use_overlap)
    if (!(lk.score_overlap(l1, l2) == 1.0)) return false;
  if (c.use_angle && c.use_overlap && c.use_smartangle)
    if (!(lk.score_smartangle(l1, l2) >= c.score_th)) return false;
  if (c.use_perp)
    if (!(lk.score_perp(l1, l2) >= c.score_th)) return false;
  if (c.use_innerseg)
    if (!(lk.score_innerseg(l1, l2) >= c.score_th)) return false;
  if (c.use_scaleinv)
    if (!(lk.score_scaleinv(l1, l2) >= c.score_th)) return false;
  return true;
}

// LineLinker2d::check_connection (base/line_linker.cc:120-137)
bool check_connection2d(const LineLinker2d &lk, const Line2d &l1, const Line2d &l2) {
  const LinkerConfig &c = lk.config;
  if (c.use_angle)
    if (!(compute_angle(l1, l2) <= c.th_angle)) return false;
  if (c.use_overlap)
    if (!(lk.score_overlap(l1, l2) == 1.0)) return false;
  if (c.use_angle && c.use_overlap && c.use_smartangle)
    if (!(lk.score_smartangle(l1, l2) >= c.score_th)) return false;
  if (c.use_perp)
    if (!(lk.score_perp(l1, l2) >= c.score_th)) return false;
  if (c.use_innerseg)
    if (!(lk.score_innerseg(l1, l2) >= c.score_th)) return false;
  return true;
}

std::vector<CameraView> make_views(int n_views, const int32_t *model_ids, const double *kvec, const double *qvec,
                                   const double *tvec) {
  std::vector<CameraView> views(n_views);
  for (int v = 0; v < n_views; ++v) {
    views[v].cam.model_id = model_ids ? model_ids[v] : 1;
    for (int k = 0; k < 4; ++k) views[v].cam.kvec[k] = kvec[4 * v + k];
    views[v].pose.set(qvec + 4 * v, tvec + 3 * v);
  }
  return views;
}

} // namespace

extern "C" void orc_merge_set_num_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}

namespace {
// Line3d::length() as the compiled reference evaluates it: the squared norm is accumulated coefficient by coefficient
// and the compiler contracts the last two steps into fused multiply-adds, sqrt(fma(z, z, fma(y, y, x * x))) (checked
// bit for bit against the stored reference outputs). The lengths become graph edge weights whose ties decide the
// greedy order, so the product reproduces them exactly.
double fit_length(const Line3d &l) {
  const double dx = l.start.x - l.end.x, dy = l.start.y - l.end.y, dz = l.start.z - l.end.z;
  return std::sqrt(std::fma(dz, dz, std::fma(dy, dy, dx * dx)));
}
struct MergeResult {
  std::vector<double> unc;                 // per input line
  std::vector<int64_t> node_line;          // graph node -> global line index
  std::vector<int32_t> edges;              // [n_edges][2] in insertion order
  std::vector<double> sim;
  std::vector<int64_t> track_off;
  std::vector<int32_t> track_nodes;
  std::vector<double> track_line;          // [T][7]
};
thread_local MergeResult g_merge;
} // namespace

extern "C" {

// Inputs: views in ascending image id order (img_ids, model_ids, kvec, qvec, tvec), line_off[V+1], segs[n][4],
// lines3d[n][6] (start, end), neighbours of view v: ng_ids[ng_off[v] .. ng_off[v+1]) as image ids (each must be an image:
// the caller checks), var2d, the 2D linker and the 3D linker (set_to_spatial_merging() is applied here).
// Returns the number of tracks; the outputs are read with orc_merge_fetch. counts[4] = nodes, edges, supports, lines.
int64_t orc_merge_to_linetracks(int32_t n_views, const int32_t *img_ids, const int32_t *model_ids, const double *kvec,
                                const double *qvec, const double *tvec, const int64_t *line_off, const double *segs,
                                const double *lines3d, const int64_t *ng_off, const int32_t *ng_ids, double var2d,
                                const LinkerConfig *cfg2d, const LinkerConfig *cfg3d, int64_t *counts) {
  MergeResult &R = g_merge;
  R = MergeResult();
  LineLinker2d linker2d;
  linker2d.config = *cfg2d;
  LineLinker3d linker3d;
  linker3d.config = *cfg3d;
  linker3d.config.set_to_spatial_merging();
  const std::vector<CameraView> views = make_views(n_views, model_ids, kvec, qvec, tvec);
  std::map<int, int> view_of;
  for (int v = 0; v < n_views; ++v) view_of[img_ids[v]] = v;
  const int64_t n_lines = line_off[n_views];
  std::vector<Line2d> l2(n_lines);
  std::vector<Line3d> l3(n_lines);
  std::vector<double> len(n_lines);
  R.unc.resize(n_lines);
  std::vector<int64_t> node_of(n_lines, -1);
  std::vector<std::pair<int, int>> nodes;
  for (int v = 0; v < n_views; ++v)
    for (int64_t g = line_off[v]; g < line_off[v + 1]; ++g) {
      const double *s = segs + 4 * g, *l = lines3d + 6 * g;
      l2[g] = Line2d(V2(s[0], s[1]), V2(s[2], s[3]));
      l3[g] = Line3d(V3(l[0], l[1], l[2]), V3(l[3], l[4], l[5]));
      l3[g].uncertainty = l3[g].computeUncertainty(views[v], var2d);
      R.unc[g] = l3[g].uncertainty;
      len[g] = fit_length(l3[g]);
      if (len[g] == 0) continue;
      node_of[g] = (int64_t)nodes.size();
      nodes.push_back(std::make_pair(img_ids[v], (int)(g - line_off[v])));
      R.node_line.push_back(g);
    }
  // per source view: self pairs (i < j), then cross pairs in (line, neighbour slot, neighbour line) order
  std::vector<std::vector<std::pair<int64_t, int64_t>>> pairs(n_views);
#pragma omp parallel for schedule(dynamic, 1)
  for (int v = 0; v < n_views; ++v) {
    const int64_t b = line_off[v], n = line_off[v + 1] - b;
    for (int64_t i = 0; i < n; ++i) {
      if (len[b + i] == 0) continue;
      for (int64_t j = i + 1; j < n; ++j) {
        if (len[b + j] == 0) continue;
        if (!check_connection3d(linker3d, l3[b + i], l3[b + j])) continue;
        if (!check_connection2d(linker2d, l2[b + i], l2[b + j])) continue;
        pairs[v].push_back(std::make_pair(b + i, b + j));
      }
    }
    const size_t image_id = (size_t)(int64_t)img_ids[v];
    for (int64_t i = 0; i < n; ++i) {
      if (len[b + i] == 0) continue;
      for (int64_t k = ng_off[v]; k < ng_off[v + 1]; ++k) {
        const size_t ng_image_id = (size_t)(int64_t)ng_ids[k];
        const int u = view_of.at(ng_ids[k]);
        const int64_t bu = line_off[u], nu = line_off[u + 1] - bu;
        for (int64_t j = 0; j < nu; ++j) {
          const int key = (int)(image_id + (size_t)i + ng_image_id + (size_t)j); // merging.cc:437-441
          if (key % 2 == 0 && image_id < ng_image_id) continue;
          if (key % 2 == 1 && image_id > ng_image_id) continue;
          if (len[bu + j] == 0) continue;
          if (!check_connection3d(linker3d, l3[b + i], l3[bu + j])) continue;
          if (!check_connection2d(linker2d, l3[b + i].projection(views[u]), l2[bu + j])) continue;
          if (!check_connection2d(linker2d, l3[bu + j].projection(views[v]), l2[b + i])) continue;
          pairs[v].push_back(std::make_pair(b + i, bu + j));
        }
      }
    }
  }
  std::vector<edge_tuple> edges;
  for (int v = 0; v < n_views; ++v)
    for (const auto &p : pairs[v]) {
      const double sim = len[p.first] + len[p.second];
      R.edges.push_back((int32_t)node_of[p.first]);
      R.edges.push_back((int32_t)node_of[p.second]);
      R.sim.push_back(sim);
      edges.push_back(std::make_tuple(sim, (size_t)node_of[p.first], (size_t)node_of[p.second]));
    }
  std::vector<int> labels = ComputeLineTrackLabelsGreedy(nodes, edges);
  int n_tracks = 0;
  for (int x : labels) n_tracks = std::max(n_tracks, x + 1);
  std::vector<std::vector<int64_t>> members(n_tracks);
  for (size_t k = 0; k < nodes.size(); ++k)
    if (labels[k] >= 0) members[labels[k]].push_back((int64_t)k);
  R.track_off.push_back(0);
  for (int t = 0; t < n_tracks; ++t) {
    std::vector<Line3d> ls;
    std::vector<double> sc;
    for (int64_t k : members[t]) {
      R.track_nodes.push_back((int32_t)k);
      ls.push_back(l3[R.node_line[k]]);
      sc.push_back(len[R.node_line[k]]);
    }
    R.track_off.push_back((int64_t)R.track_nodes.size());
    const Line3d a = aggregate_line3d_list(ls, sc, 0);
    const double o[7] = {a.start.x, a.start.y, a.start.z, a.end.x, a.end.y, a.end.z, a.uncertainty};
    R.track_line.insert(R.track_line.end(), o, o + 7);
  }
  counts[0] = (int64_t)nodes.size();
  counts[1] = (int64_t)R.sim.size();
  counts[2] = (int64_t)R.track_nodes.size();
  counts[3] = n_lines;
  return n_tracks;
}

// Copies the result of the last orc_merge_to_linetracks of this thread (sizes from its counts).
void orc_merge_fetch(double *unc, int64_t *node_line, int32_t *edges, double *sim, int64_t *track_off,
                     int32_t *track_nodes, double *track_line) {
  const MergeResult &R = g_merge;
  std::copy(R.unc.begin(), R.unc.end(), unc);
  std::copy(R.node_line.begin(), R.node_line.end(), node_line);
  std::copy(R.edges.begin(), R.edges.end(), edges);
  std::copy(R.sim.begin(), R.sim.end(), sim);
  std::copy(R.track_off.begin(), R.track_off.end(), track_off);
  std::copy(R.track_nodes.begin(), R.track_nodes.end(), track_nodes);
  std::copy(R.track_line.begin(), R.track_line.end(), track_line);
}

} // extern "C"
