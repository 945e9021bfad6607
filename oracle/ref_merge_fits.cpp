// ref_merge_fits.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// C entry points (ctypes) over the REFERENCE'S OWN merging.merging (merging.py:6-21): merging::SetUncertaintySegs3d and
// merging::MergeToLineTracks of its merging.cc / merging_utils.cc, compiled unchanged into oracle/_ref/liblimap_ref.so
// (oracle/Makefile target `ref`). oracle/merge_fits.py compiles this file with the same flags and links it against that
// library into oracle/_ref/liblimap_ref_merge.so, only where the reference source tree exists. Its outputs on the
// seeded cases are stored as tests/golden/ref/merge_to_linetracks_*.npz (tests/golden/make_merge_golden.py).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>
#include <pybind11/eigen.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>
#include <Eigen/Dense>
#include <colmap/scene/camera.h>
#include <colmap/util/logging.h>
#include "limap/base/graph.h"
#include "limap/base/line_linker.h"
#include "limap/merging/merging.h"
#include "limap/merging/merging_utils.h"

using namespace limap;

extern "C" {
struct ref_linker_cfg { // layout of lm_linker_config / orc::LinkerConfig
  double score_th, th_angle, th_overlap, th_smartoverlap, th_smartangle, th_perp, th_innerseg, th_scaleinv;
  int32_t use_angle, use_overlap, use_smartangle, use_perp, use_innerseg, use_scaleinv;
};
}
template <typename L> static void fill_linker(L &l, const ref_linker_cfg &c) {
  l.score_th = c.score_th; l.th_angle = c.th_angle; l.th_overlap = c.th_overlap; l.th_smartoverlap = c.th_smartoverlap;
  l.th_smartangle = c.th_smartangle; l.th_perp = c.th_perp; l.th_innerseg = c.th_innerseg;
  l.use_angle = c.use_angle; l.use_overlap = c.use_overlap; l.use_smartangle = c.use_smartangle; l.use_perp = c.use_perp;
  l.use_innerseg = c.use_innerseg;
}
static LineLinker2dConfig to_linker2d(const ref_linker_cfg &c) { LineLinker2dConfig l; fill_linker(l, c); return l; }
static LineLinker3dConfig to_linker3d(const ref_linker_cfg &c) {
  LineLinker3dConfig l;
  fill_linker(l, c);
  l.th_scaleinv = c.th_scaleinv;
  l.use_scaleinv = c.use_scaleinv;
  return l;
}
static Line2d mk2(const double *s) { return Line2d(V2D(s[0], s[1]), V2D(s[2], s[3])); }
static thread_local std::string g_err;
extern "C" const char *ref_merge_last_error() { return g_err.c_str(); }

// merging.py:6-21 of the reference: SetUncertaintySegs3d per image, then merging::MergeToLineTracks into a fresh Graph.
// Arguments as orc_merge_to_linetracks (orc_merging.cpp); outputs through ref_merge_fetch. With no line of non-zero
// length the reference dereferences max_element of an empty label vector; nothing is called then and the result is
// empty.
namespace {
struct RefMergeResult {
  std::vector<double> unc;
  std::vector<int64_t> node_line;
  std::vector<int32_t> edges;
  std::vector<double> sim;
  std::vector<int64_t> track_off;
  std::vector<int32_t> track_nodes;
  std::vector<double> track_line;
};
thread_local RefMergeResult g_ref_merge;
} // namespace
extern "C" {
int64_t ref_merge_to_linetracks(int32_t n_views, const int32_t *img_ids, const int32_t *model_ids, const double *kvec,
                                const double *qvec, const double *tvec, const int64_t *line_off, const double *segs,
                                const double *lines3d, const int64_t *ng_off, const int32_t *ng_ids, double var2d,
                                const ref_linker_cfg *cfg2d, const ref_linker_cfg *cfg3d, int64_t *counts) {
  RefMergeResult &R = g_ref_merge;
  R = RefMergeResult();
  try {
    std::map<int, Camera> cams;
    std::map<int, CameraImage> imgs;
    std::map<int, int> view_of;
    for (int v = 0; v < n_views; ++v) {
      const double *k = kvec + 4 * v;
      const int model = model_ids ? model_ids[v] : 1;
      std::vector<double> params;
      if (model == 0) params = {k[0], k[2], k[3]};
      else params = {k[0], k[1], k[2], k[3]};
      cams[v] = Camera(model, params, v);
      imgs[img_ids[v]] = CameraImage(v, CameraPose(V4D(qvec[4 * v], qvec[4 * v + 1], qvec[4 * v + 2], qvec[4 * v + 3]),
                                                   V3D(tvec[3 * v], tvec[3 * v + 1], tvec[3 * v + 2])));
      view_of[img_ids[v]] = v;
    }
    ImageCollection imagecols(cams, imgs);
    std::map<int, std::vector<Line2d>> all_lines_2d;
    std::map<int, std::vector<Line3d>> all_lines_3d;
    std::map<int, std::vector<int>> neighbors;
    bool any_node = false;
    for (int v = 0; v < n_views; ++v) {
      std::vector<Line2d> l2;
      std::vector<Line3d> l3;
      for (int64_t g = line_off[v]; g < line_off[v + 1]; ++g) {
        l2.push_back(mk2(segs + 4 * g));
        const double *l = lines3d + 6 * g;
        l3.push_back(Line3d(V3D(l[0], l[1], l[2]), V3D(l[3], l[4], l[5])));
      }
      all_lines_2d[img_ids[v]] = l2;
      all_lines_3d[img_ids[v]] = merging::SetUncertaintySegs3d(l3, imagecols.camview(img_ids[v]), var2d);
      for (size_t k = 0; k < l3.size(); ++k) {
        R.unc.push_back(all_lines_3d[img_ids[v]][k].uncertainty);
        any_node = any_node || all_lines_3d[img_ids[v]][k].length() != 0;
      }
      neighbors[img_ids[v]] = std::vector<int>(ng_ids + ng_off[v], ng_ids + ng_off[v + 1]);
    }
    Graph graph;
    std::vector<LineTrack> tracks;
    if (any_node)
      merging::MergeToLineTracks(graph, tracks, all_lines_2d, imagecols, all_lines_3d, neighbors,
                                 LineLinker(LineLinker2d(to_linker2d(*cfg2d)), LineLinker3d(to_linker3d(*cfg3d))));
    for (PatchNode *node : graph.nodes) R.node_line.push_back(line_off[view_of.at(node->image_idx)] + (int64_t)node->line_idx);
    for (Edge *e : graph.undirected_edges) {
      R.edges.push_back((int32_t)e->node_idx1);
      R.edges.push_back((int32_t)e->node_idx2);
      R.sim.push_back(e->sim);
    }
    R.track_off.push_back(0);
    for (const LineTrack &t : tracks) {
      for (int id : t.node_id_list) R.track_nodes.push_back(id);
      R.track_off.push_back((int64_t)R.track_nodes.size());
      const double o[7] = {t.line.start[0], t.line.start[1], t.line.start[2], t.line.end[0], t.line.end[1], t.line.end[2],
                           t.line.uncertainty};
      R.track_line.insert(R.track_line.end(), o, o + 7);
    }
    counts[0] = (int64_t)R.node_line.size();
    counts[1] = (int64_t)R.sim.size();
    counts[2] = (int64_t)R.track_nodes.size();
    counts[3] = (int64_t)R.unc.size();
    return (int64_t)tracks.size();
  } catch (const std::exception &e) {
    g_err = e.what();
    return -1;
  }
}
void ref_merge_fetch(double *unc, int64_t *node_line, int32_t *edges, double *sim, int64_t *track_off,
                     int32_t *track_nodes, double *track_line) {
  const RefMergeResult &R = g_ref_merge;
  std::copy(R.unc.begin(), R.unc.end(), unc);
  std::copy(R.node_line.begin(), R.node_line.end(), node_line);
  std::copy(R.edges.begin(), R.edges.end(), edges);
  std::copy(R.sim.begin(), R.sim.end(), sim);
  std::copy(R.track_off.begin(), R.track_off.end(), track_off);
  std::copy(R.track_nodes.begin(), R.track_nodes.end(), track_nodes);
  std::copy(R.track_line.begin(), R.track_line.end(), track_line);
}
}

