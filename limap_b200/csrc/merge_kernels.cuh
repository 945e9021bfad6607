// merge_kernels.cuh — post-triangulation track filters and the remerge pair test (SURVEY.md §8(f) rank 1).
#pragma once
#include "tri_kernels.cuh"

namespace lm {

// Per-support checks of merging/merging_utils.cc:27-155; one thread per supporting 2D line.
struct SupportParams {
  const ViewD *views;        // [n_views]
  const int64_t *sup_off;    // [T+1]
  const int32_t *sup_view;   // [S]
  const double4 *segs;       // [S] x1,y1,x2,y2
  const double *track_line;  // [T][6]
  int64_t T, S;
  double th_angular2d, th_perp2d, th_sv_angular3d, th_overlap;
  uint8_t *flags;            // [S] bit0 reprojection ok, bit1 sensitivity ok, bit2 overlap ok
};
void launch_support_flags(const SupportParams &p, cudaStream_t s);

// All-pairs LineLinker3d::check_connection of RemergeLineTracks (merging/merging.cc:527-556).
struct RemergeParams {
  const double *lines;       // [T][7] start, end, uncertainty
  const float4 *dirf;        // [T] unit direction in fp32 (gate), w unused
  const float4 *ballf;       // [T] midpoint - origin, grown radius (gate)
  const uint8_t *active;     // [T]
  int64_t T;
  int all_active;
  LinkerDev<double> lk;      // after set_to_spatial_merging()
  float cos_gate;            // cos(th_angle) - margin; gate used only when use_gate
  int use_gate;
  int use_ball;              // use_innerseg: the ball gate is a necessary condition
  uint32_t *edges;           // [capacity][2] (a < b), unordered
  unsigned long long *counter; // [2]: edges found, pairs past the gate
  unsigned long long capacity;
};
void launch_remerge_dirs(const double *lines, int64_t T, const double origin[3], double th_innerseg, float4 *dirf,
                         float4 *ballf, cudaStream_t s);
void launch_remerge_pairs(const RemergeParams &p, cudaStream_t s);

// MergeToLineTracks from per-image 3D fits (merging/merging.cc:347-511).
struct FitView {       // CameraView as Line3d::projection / computeUncertainty evaluate it
  double R[9], t[3];   // row-major rotation, translation
  double fx, fy, cx, cy, f; // f = Camera::uncertainty's focal length
};
struct FitPrepParams {
  const FitView *views;      // [V]
  const int64_t *line_off;   // [V+1]
  const double *lines3d;     // [n][6]
  int32_t V;
  int64_t n;
  double var2d, ox, oy, oz, th_innerseg;
  double *rec;               // [n][7] start, end, uncertainty
  double *len;               // [n] Line3d::length(), bit-exact
  uint8_t *nonzero;          // [n] length != 0: the line is a graph node
  float4 *dirf, *ballf;      // [n] gate records
};
void launch_fit_prep(const FitPrepParams &p, cudaStream_t s);

struct FitTile { int32_t va, vb, slot, tiles; }; // slot < 0: self block of va; tiles = ta << 16 | tb
struct FitPairParams {
  const FitView *views;
  const int64_t *line_off;
  const int32_t *img_ids;
  const double4 *segs;       // [n]
  const double *rec;         // [n][7]
  const uint8_t *nonzero;
  const float4 *dirf, *ballf;
  const FitTile *tiles;
  LinkerDev<double> lk3, lk2; // lk3 after set_to_spatial_merging()
  float cos_gate;
  int use_gate, use_ball;
  unsigned long long *keys;  // [capacity] insertion key
  unsigned long long *pairs; // [capacity] line1 << 32 | line2 (global line indices; node ids keep their order)
  unsigned long long *counter; // [3]: edges, pairs past the gates, pairs tested
  unsigned long long capacity;
};
void launch_fit_pairs(const FitPairParams &p, int64_t n_tiles, cudaStream_t s);
// keys of the greedy order (descending (sim, node1, node2)) of the edges in insertion order; sim[e] = len1 + len2
void launch_fit_order_keys(const unsigned long long *pairs, const double *len, int64_t n,
                           unsigned long long *by_nodes, unsigned long long *by_score, double *sim, cudaStream_t s);

} // namespace lm
