// locmatch_kernels.cuh — line matching of query images against a line map (optimize/hybrid_localization/functions.py):
// the epipolar IoU sweep over (query, target image) items, the IoU filter of given pairs, the grouping of 2D-3D matches
// per query line and the reprojection filter. Host side in engine_locmatch.cu.
#pragma once
#include "lm_math.cuh"

namespace lm {

// One image of a localization scene (all fp64). M = R^T K^-1, C = -R^T t feed the epipolar IoU (lm_math.cuh); R, t and
// k = (fx, fy, cx, cy) feed CameraView::projection (base/camera_view.cc:61-65).
struct LocView {
  double M[9], C[3], R[9], t[3], k[4];
};

struct LocScene {
  const LocView *views;       // [n_images]
  const int64_t *line_off;    // [n_images + 1] first line of every image
  const double4 *lines;       // [n_lines] x1, y1, x2, y2
  const int32_t *line_track;  // [n_lines] track of every line, -1 when untracked (NULL: no map)
  const double *track_lines;  // [n_tracks][6] start, end
};

// The (query image, target image) items, in query order and then retrieval order.
struct LocItems {
  const int2 *items;          // [n_items] (query image, target image)
  const int64_t *row_off;     // [n_items + 1] first (item, query line) row of every item
  int64_t n_items;
};

// Epipolar sweep, pass 1: one warp per (item, query line) row tests the row against every line of the target image,
// writes one bit per target line (IoU > th, and the target line tracked when to_tracks) and the row's count.
void launch_locmatch_sweep_count(const LocScene &s, const LocItems &it, const int64_t *word_off, double th,
                                 int to_tracks, uint32_t *mask, int64_t *cnt, unsigned long long *n_2to2,
                                 cudaStream_t st);
// Pass 2: every row's pairs at its scanned offset, in target-line order. Pairs are (query line, target line), or
// (query line, track) when to_tracks.
void launch_locmatch_sweep_place(const LocScene &s, const LocItems &it, const int64_t *word_off, const uint32_t *mask,
                                 const int64_t *off, int to_tracks, int2 *out, cudaStream_t st);
// Given pairs (query line, target line) per item: flag[k] = kept (IoU > th when use_iou, tracked when to_tracks);
// err is set on an out-of-range line id; n_2to2 counts the pairs past the IoU test, tracked or not.
void launch_locmatch_filter_flags(const LocScene &s, const LocItems &it, const int64_t *pair_off, const int2 *pairs,
                                  int64_t n_pairs, int use_iou, double th, int to_tracks, int64_t *flag, int *err,
                                  unsigned long long *n_2to2, cudaStream_t st);
void launch_locmatch_filter_place(const LocScene &s, const LocItems &it, const int64_t *pair_off, const int2 *pairs,
                                  int64_t n_pairs, const int64_t *pos, int to_tracks, int2 *out, cudaStream_t st);
// item_off[k] = off[first[k]] for k <= n: offsets of the items in a scanned flat list.
void launch_gather_offsets(const int64_t *off, const int64_t *first, int64_t n, int64_t *item_off, cudaStream_t st);

// Grouping of the 2D-3D list E (items contiguous, in item order) by query line, in the order of the reference's
// defaultdict: query lines in order of first appearance, tracks in append order. Queries are runs of items with the
// same query image; (query, line) rows are numbered by qrow_off[query] + line.
struct LocGroup {
  const int2 *E;              // [n_e] (query line, track)
  const int64_t *item_off;    // [n_items + 1]
  const int64_t *q_item_off;  // [n_queries + 1] first item of every query
  const int64_t *qrow_off;    // [n_queries + 1]
  int64_t n_e, n_queries;
  unsigned int *cnt;          // [rows of the items] entries per (item, line)
  unsigned long long *first;  // [rows of the items] first entry per (item, line)
  int64_t *key;               // [rows of the items] output position of the (item, line)'s first entry
  unsigned int *run;          // [rows of the items] entries placed so far
  int64_t *head;              // [n_e] scanned in place: a key's size at its first entry, else 0
  int64_t *qhead;             // [query rows] first entry of every (query, line) (-1: no entry)
  int64_t *qtot;              // [query rows] entries of every (query, line)
};
void launch_group_count(const LocItems &it, const LocGroup &g, cudaStream_t st);
void launch_group_heads(const LocItems &it, const LocGroup &g, int64_t n_qrows, cudaStream_t st);
void launch_group_keys(const LocItems &it, const LocGroup &g, int64_t n_qrows, cudaStream_t st);
void launch_group_place(const LocItems &it, const LocGroup &g, int2 *out, cudaStream_t st);

// reprojection_filter_matches_2to3 (functions.py:96-140): one warp per (query, line) key over the grouped list G; the
// best track lands at sel[key position] (flag[key position] = 1), every other entry of flag is 0.
struct ReprojParams {
  int dist_func;              // 0 perpendicular_dist, 1 midpoint_dist, 2 midpoint_perpendicular_dist
  double dist_thres, sine_thres, angle_scale;
};
void launch_reproj_filter(const LocScene &s, const LocItems &it, const LocGroup &g, const int2 *G,
                          const ReprojParams &rp, int64_t *flag, int32_t *sel, cudaStream_t st);
void launch_reproj_place(const LocGroup &g, const int2 *G, const int64_t *pos, const int32_t *sel, int2 *out,
                         cudaStream_t st);

} // namespace lm
