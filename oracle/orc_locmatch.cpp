// oracle/orc_locmatch.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
// fp64 restatement of the line matching of optimize/hybrid_localization/functions.py, on the compute_epipolar_IoU and
// CameraView::projection of orc_triangulation.h / orc_geom.h (pinned to the reference's compiled functions):
//   match_line_2to2_epipolarIoU (:6-23)      orc_locmatch_2to2
//   filter_line_2to2_epipolarIoU (:26-52)    orc_locmatch_filter
//   reprojection_filter_matches_2to3 (:99-140), one query line: orc_locmatch_reproj_one
// Built by oracle/locmatch.py into oracle/_build/liblimap_orc_locmatch.so.
#include "orc_triangulation.h"
#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

using namespace orc;

namespace {
CameraView mkview(const double *cam /*model,fx,fy,cx,cy,qw,qx,qy,qz,tx,ty,tz*/) {
  CameraView v;
  v.cam.model_id = (int)cam[0];
  for (int k = 0; k < 4; ++k) v.cam.kvec[k] = cam[1 + k];
  v.pose.set(cam + 5, cam + 9);
  return v;
}
Line2d mk2(const double *s) { return Line2d(V2(s[0], s[1]), V2(s[2], s[3])); }
double cross2(const V2 &a, const V2 &b) { return a.x * b.y - a.y * b.x; } // np.cross of two 2-vectors
} // namespace

extern "C" {

// out[k] = (i, j) of every pair with IoU > th, i major; returns the count (out may be NULL)
int64_t orc_locmatch_2to2(int64_t n1, const double *l1, const double *cam1, int64_t n2, const double *l2,
                          const double *cam2, double th, int32_t *out) {
  const CameraView v1 = mkview(cam1), v2 = mkview(cam2);
  int64_t n = 0;
  for (int64_t i = 0; i < n1; ++i)
    for (int64_t j = 0; j < n2; ++j)
      if (compute_epipolar_IoU(mk2(l1 + 4 * i), v1, mk2(l2 + 4 * j), v2) > th) {
        if (out) { out[2 * n] = (int32_t)i; out[2 * n + 1] = (int32_t)j; }
        ++n;
      }
  return n;
}

int64_t orc_locmatch_filter(int64_t n_pairs, const int32_t *pairs, const double *l1, const double *cam1,
                            const double *l2, const double *cam2, double th, int32_t *out) {
  const CameraView v1 = mkview(cam1), v2 = mkview(cam2);
  int64_t n = 0;
  for (int64_t k = 0; k < n_pairs; ++k)
    if (compute_epipolar_IoU(mk2(l1 + 4 * pairs[2 * k]), v1, mk2(l2 + 4 * pairs[2 * k + 1]), v2) > th) {
      out[2 * n] = pairs[2 * k];
      out[2 * n + 1] = pairs[2 * k + 1];
      ++n;
    }
  return n;
}

// The best track of one query line among n candidate track ids (duplicates and any order allowed), -1 when none;
// dist_func 0 perpendicular_dist, 1 midpoint_dist, 2 midpoint_perpendicular_dist.
int32_t orc_locmatch_reproj_one(const double *ref_seg, const double *cam, int64_t n, const int32_t *cand,
                                const double *track_lines, int dist_func, double dist_thres, double sine_thres,
                                double angle_scale) {
  const CameraView view = mkview(cam);
  const Line2d ref = mk2(ref_seg);
  const V2 dir_ref = ref.direction();
  std::vector<int32_t> ids(cand, cand + n); // np.unique: ascending, distinct
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  double min_loss = std::numeric_limits<double>::infinity();
  int32_t best = -1;
  for (int32_t id : ids) {
    const double *L = track_lines + 6 * (int64_t)id;
    const Line2d l2d(view.projection(V3(L[0], L[1], L[2])), view.projection(V3(L[3], L[4], L[5])));
    double dist;
    if (dist_func == 1) {
      dist = (ref.midpoint() - l2d.midpoint()).norm();
    } else if (dist_func == 0) {
      const V2 t = l2d.start, d = l2d.direction();
      dist = 0.5 * (std::abs(cross2(d, t - ref.start)) + std::abs(cross2(d, t - ref.end)));
    } else {
      const V2 t = l2d.start, d = l2d.direction();
      dist = std::abs(cross2(d, t - ref.midpoint())) / ref.length();
    }
    double loss = dist;
    if (dist_func == 1) {
      const V2 d = l2d.direction();
      double c = dir_ref.x * d.x + dir_ref.y * d.y;
      c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c); // np.clip keeps NaN
      const double sine = std::sqrt(1 - c * c);
      loss += angle_scale * l2d.length() * sine;
      if (sine > sine_thres) continue;
    }
    if (dist > dist_thres) continue;
    if (loss < min_loss) {
      min_loss = loss;
      best = id;
    }
  }
  return best;
}

} // extern "C"
