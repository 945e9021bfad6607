/* limap_b200.h — C ABI of the H100-native (sm_90a) line-triangulation / line-refinement engine.
 *
 * This is the drop-in boundary for the hot path of cvg/limap (SURVEY.md §8b). The
 * reference has no C ABI: its C++ classes are reached through pybind11
 * (src/limap/triangulation/bindings.cc:78-119, src/limap/optimize/{line_refinement,hybrid_bundle_adjustment}/bindings.cc,
 * src/limap/vplib/JLinkage/bindings.cc). Each entry point below names the
 * reference interface it replaces (paths relative to src/limap/ of cvg/limap).
 * Plain pointers and sizes only; no torch / pybind types. All functions return
 * LM_OK (0) or a negative error code; lm_last_error() gives the message
 * (the reference throws std::runtime_error / THROW_CHECK instead).
 *
 * Host pointers unless a parameter is named d_*. Image ids are arbitrary ints
 * (as in ImageCollection); lines of an image are indexed 0..L-1.
 * Limits (same as the reference's Node2d = pair<uint16,uint16>, util/types.h:16):
 * n_views <= 65535, lines per image <= 65535.
 */
#ifndef LIMAP_B200_H
#define LIMAP_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LM_OK 0
#define LM_ERR_INVALID -1   /* bad argument / index out of range */
#define LM_ERR_CUDA -2      /* CUDA runtime failure */
#define LM_ERR_STATE -3     /* call order (e.g. run before scene upload) */
#define LM_ERR_NOGPU -4     /* no usable CUDA device: there is NO CPU fallback */

typedef struct lm_ctx lm_ctx;

/* base/line_linker.h:18-46 (LineLinker2dConfig) and :80-143 (LineLinker3dConfig). */
typedef struct lm_linker_config {
  double score_th, th_angle, th_overlap, th_smartoverlap, th_smartangle, th_perp, th_innerseg,
      th_scaleinv;
  int32_t use_angle, use_overlap, use_smartangle, use_perp, use_innerseg, use_scaleinv;
} lm_linker_config;

/* triangulation/base_line_triangulator.h:22-43 + global_line_triangulator.h:11-25.
 * Field defaults are the C++ defaults; the Python mirror applies a dict over them the way
 * ASSIGN_PYDICT_ITEM does (internal/helpers.h:25-27). */
typedef struct lm_tri_config {
  double min_length_2d, line_tri_angle_threshold, IoU_threshold, sensitivity_threshold, var2d,
      fullscore_th;
  int32_t debug_mode, add_halfpix, use_vp, use_endpoints_triangulation;
  int32_t disable_many_points_triangulation, disable_one_point_triangulation;
  int32_t disable_algebraic_triangulation, disable_vp_triangulation;
  int32_t max_valid_conns, min_num_outer_edges, num_outliers_aggregator;
  int32_t merging_strategy; /* 0 = "greedy" (the only strategy on the hot path) */
  lm_linker_config linker2d, linker3d;
} lm_tri_config;

typedef struct lm_tri_stats {
  int64_t n_rows;        /* match rows tested (the M1 numerator) */
  int64_t n_candidates;  /* surviving 3D candidates */
  int64_t n_valid_edges; /* candidates kept as valid connections */
  int64_t n_nodes;       /* 2D lines in the scene */
  int64_t n_kernel_launches; /* kernels this library launched since ctx creation */
  int64_t n_pairs_gated; /* candidate pairs that passed the fp32 3d pruning gates */
  int64_t n_pairs_exact; /* candidate pairs scored with the exact fp64 reference formulas */
  int64_t max_rows_per_node;
  double last_run_ms;    /* device time of the last lm_tri_run (CUDA events on the ctx stream) */
  double last_node_kernel_ms; /* device time of its fused generate+score kernel alone */
} lm_tri_stats;

const char *lm_last_error(void);
const char *lm_version(void);

/* ---- context ------------------------------------------------------------------------ */
int lm_ctx_create(int device, lm_ctx **out);
void lm_ctx_destroy(lm_ctx *ctx);
/* Run all work of this context on an existing CUDA stream (e.g. torch's current stream). */
int lm_ctx_set_stream(lm_ctx *ctx, void *cuda_stream);
int lm_ctx_synchronize(lm_ctx *ctx);

/* ---- scene: BaseLineTriangulator::Init (triangulation/base_line_triangulator.cc:45-63) +
 *      GlobalLineTriangulator::Init (global_line_triangulator.cc:32-57).
 * model_ids: 0 SIMPLE_PINHOLE, 1 PINHOLE (base/camera_models.h:29-44); kvec = [fx,fy,cx,cy];
 * qvec wxyz, tvec (base/camera.h:89-112); line_off[n_views+1]; segs[sum L][4] = x1,y1,x2,y2. */
int lm_scene_upload(lm_ctx *ctx, int32_t n_views, const int32_t *img_ids, const int32_t *model_ids,
                    const double *kvec, const double *qvec, const double *tvec,
                    const int64_t *line_off, const double *segs);

/* ---- triangulator: GlobalLineTriangulator(config) (global_line_triangulator.h:27-35) */
int lm_tri_configure(lm_ctx *ctx, const lm_tri_config *cfg);
/* SetRanges / UnsetRanges (base_line_triangulator.h:62-66) */
int lm_tri_set_ranges(lm_ctx *ctx, const double lo[3], const double hi[3]);
int lm_tri_unset_ranges(lm_ctx *ctx);
/* InitVPResults (base_line_triangulator.h:56-58): labels[label_off[i]..] per line (-1 none),
 * vps[vp_off[i]..][3] per image. */
int lm_tri_set_vps(lm_ctx *ctx, int32_t n_images, const int32_t *img_ids, const int64_t *label_off,
                   const int32_t *labels, const int64_t *vp_off, const double *vps);

/* TriangulateImage(img_id, map<int, MatrixXi>) (base_line_triangulator.cc:71-109).
 * ng_ids[n_ng], row_off[n_ng+1], pairs[row_off[n_ng]][2] = (line_id, ng_line_id).
 * The work is enqueued; it runs (batched over all enqueued images) at lm_tri_run or at the first
 * getter. Out-of-range line ids fail here like the reference's IndexError (:87-94). */
int lm_tri_add_image_matches(lm_ctx *ctx, int32_t img_id, int32_t n_ng, const int32_t *ng_ids,
                             const int64_t *row_off, const int32_t *pairs);
/* Same, pairs already in device memory (zero-copy ingress from a GPU matcher). */
int lm_tri_add_image_matches_device(lm_ctx *ctx, int32_t img_id, int32_t n_ng, const int32_t *ng_ids,
                                    const int64_t *row_off, const int32_t *d_pairs);
/* TriangulateImageExhaustiveMatch(img_id, neighbors) (base_line_triangulator.cc:111-136). */
int lm_tri_add_image_exhaustive(lm_ctx *ctx, int32_t img_id, int32_t n_ng, const int32_t *ng_ids);
/* Drop all enqueued matches and results (scene and config stay). */
int lm_tri_clear(lm_ctx *ctx);
/* Restrict the next lm_tri_run to source images with view index in [begin, end) of the ascending
 * img_id order (multi-GPU sharding by source image, SURVEY.md §8e). Default: all. end < 0 or end > n_views means
 * n_views; lm_tri_run fails with LM_ERR_INVALID when begin exceeds the resulting end. */
int lm_tri_set_shard(lm_ctx *ctx, int32_t view_begin, int32_t view_end);
/* Split lm_tri_run into n groups of whole source images (default 1): sort + node kernel of group g are issued as
 * soon as the match chunks of its images have arrived on the copy stream, so they can run under the upload of
 * the later groups. Results do not depend on n (nodes are independent). */
int lm_tri_set_pipeline_groups(lm_ctx *ctx, int32_t n_groups);
/* Result sink of the next runs (NULL: none): lm_tri_run copies the node records of every pipeline group into
 * host_nodes[view-order node index] (layout of lm_tri_get_nodes, 96 bytes per 2D line of the scene) as soon as the
 * group's kernel has finished, on a stream of its own, under the kernels of the later groups; all records of the
 * run's shard are there when lm_tri_run returns. Pass page-locked memory (pageable memory makes the copies
 * synchronous). Replaces a lm_tri_get_nodes call after the run for single-GPU callers. */
int lm_tri_set_node_sink(lm_ctx *ctx, void *host_nodes);

/* Candidate generation + scoring + selection for every enqueued image:
 * triangulateOneNode (base_line_triangulator.cc:161-337) + scoreOneNode
 * (global_line_triangulator.cc:71-161), fused, one CTA per 2D line. Work is issued on the ctx stream;
 * the call returns after it completed (device time of the run: lm_tri_stats.last_run_ms).
 * May be called repeatedly on the same staged matches (benchmarking). */
int lm_tri_run(lm_ctx *ctx);
int lm_tri_get_stats(lm_ctx *ctx, lm_tri_stats *out);

/* GetBestScoredTriNode for every line of an image (global_line_triangulator.cc:536-540):
 * out_line[L][10] = start3, end3, depths2, uncertainty, score; out_ng[L][2] = (ng_img_id, ng_line_id);
 * out_ncand[L] = number of candidates of the node (may be NULL). Nodes without candidates return
 * zeros, uncertainty -1, score 0, ng (0,0) (the reference leaves the Line3d uninitialised). */
int lm_tri_get_best(lm_ctx *ctx, int32_t img_id, double *out_line, int32_t *out_ng, int32_t *out_ncand);
/* valid_edges_ of an image (global_line_triangulator.cc:130-142) as (ng_img_id, ng_line_id) in
 * candidate order; off[L+1]. Pass edges = NULL to get the count. Returns count or <0. */
int64_t lm_tri_get_valid_edges(lm_ctx *ctx, int32_t img_id, int64_t *off, int32_t *edges);
/* GetScoredTrisNode (global_line_triangulator.cc:374-378); requires debug_mode. Returns the number
 * of candidates of the node (writes at most cap). */
int lm_tri_get_cands_node(lm_ctx *ctx, int32_t img_id, int32_t line_id, int32_t cap, double *out_line,
                          int32_t *out_ng);

/* Per-node results as one device-resident record array (for the multi-GPU all-gather).
 * Record layout: lm_node_record below. d_out must hold lm_tri_num_nodes records. */
typedef struct lm_node_record {
  double line[9]; /* start3, end3, depths2, uncertainty */
  double score;
  int32_t ng_view, ng_line, n_cand, n_valid;
} lm_node_record;
int64_t lm_tri_num_nodes(lm_ctx *ctx);
int lm_tri_export_nodes(lm_ctx *ctx, int64_t node_begin, int64_t node_end, void *d_out);
int lm_tri_import_nodes(lm_ctx *ctx, int64_t node_begin, int64_t node_end, const void *d_in);
/* Directed valid edges as device-resident (src_node, dst_node) int64 pairs, the ones lm_tri_build_tracks uses: this
 * context's shard after lm_tri_run, every rank's after lm_tri_unpack_messages, and whatever lm_tri_import_edges set.
 * (lm_tri_get_valid_edges / lm_tri_get_all_valid_edges keep reporting the context's own shard.) import with append = 1
 * adds the pairs after this run's own valid connections and earlier imports; append = 0 replaces them. */
int64_t lm_tri_num_valid_edges(lm_ctx *ctx);
int lm_tri_export_edges(lm_ctx *ctx, void *d_out /* int64[n][2] */);
int lm_tri_import_edges(lm_ctx *ctx, int64_t n, const void *d_in /* int64[n][2] */, int32_t append);
/* The same exchange as one fixed-size message per rank, so that a multi-GPU step is pack -> ONE all-gather ->
 * unpack with no host synchronisation (SURVEY.md 8e; replaces nothing in the reference, which is single-process).
 * Message: [int64 n_edges, int64 n_nodes] | lm_node_record[max_nodes] | (uint32 src_node, uint32 dst_node)[cap_edges].
 * pack: this context's shard -> d_msg (device, asynchronous on the ctx stream). unpack: `world` messages laid out
 * back to back (the all-gather output) -> node records of every rank in place and the directed valid connections of
 * all ranks, in rank order, ready for lm_tri_build_tracks; rank_node_begin[r] = first node of rank r's shard.
 * lm_tri_gather_status synchronises and returns 1 when some rank had more than cap_edges connections (repeat the
 * exchange with a larger message), 0 otherwise; *n_edges_total = directed edges now held. An overflow stays set until
 * an exchange that fits or a new lm_tri_run: until then lm_tri_build_tracks, lm_tri_num_valid_edges and
 * lm_tri_export_edges fail with LM_ERR_STATE. */
int64_t lm_tri_gather_message_bytes(int64_t max_nodes, int64_t cap_edges);
int lm_tri_pack_message(lm_ctx *ctx, int64_t max_nodes, int64_t cap_edges, void *d_msg);
int lm_tri_unpack_messages(lm_ctx *ctx, int32_t world, const int64_t *rank_node_begin, int64_t max_nodes,
                           int64_t cap_edges, const void *d_msgs);
int64_t lm_tri_gather_status(lm_ctx *ctx, int64_t *n_edges_total);
/* first node index of a view (ascending img_id order) */
int64_t lm_scene_node_offset(lm_ctx *ctx, int32_t view_index);

/* ---- bulk forms of the calls above (same semantics, one call per scene instead of one per image) ------- */
/* TriangulateImage for many images at once: block b holds the matches of (src_img_ids[b], ng_img_ids[b]) in
 * pairs[row_off[b] .. row_off[b+1]). All blocks of one source image must be given in the same call. */
int lm_tri_add_matches_bulk(lm_ctx *ctx, int32_t n_blocks, const int32_t *src_img_ids, const int32_t *ng_img_ids,
                            const int64_t *row_off, const int32_t *pairs);
/* All node records (lm_tri_num_nodes of them, node order = images ascending, lines ascending); ng_view in the
 * record is the view index (position in the ascending image id list). */
int lm_tri_get_nodes(lm_ctx *ctx, lm_node_record *out);
/* All valid connections: node_off[n_nodes+1], edges[n][2] = (ng_img_id, ng_line_id). edges == NULL: count. */
int64_t lm_tri_get_all_valid_edges(lm_ctx *ctx, int64_t *node_off, int32_t *edges);

/* ComputeLineTracks (global_line_triangulator.cc:353-359): run_clustering (:234-291) +
 * ComputeLineTrackLabelsGreedy (merging/merging.cc:18-103) + Aggregator::aggregate_line3d_list
 * (merging/aggregator.cc:53-101). Returns the number of tracks (>= 0) or <0. */
int64_t lm_tri_build_tracks(lm_ctx *ctx, int64_t *n_support_total);
/* track_off[T+1]; per supporting line: img id, line id, graph node id, line3d[10] (start3,end3,
 * depths2,uncertainty,score); per track: line[7] = start3,end3,uncertainty. */
int lm_tri_get_tracks(lm_ctx *ctx, int64_t *track_off, int32_t *img_ids, int32_t *line_ids,
                      int32_t *node_ids, double *node_line3d, double *track_line);

/* ---- post-triangulation track filters and remerge (SURVEY.md 8(f) rank 1) --------------------------------
 * The steps of runners/line_triangulation.py:171-200 between ComputeLineTracks and the line BA. Tracks are flat
 * arrays like lm_ba_solve's: sup_off[T+1], per supporting line its view index (position in the camera arrays)
 * and 2D segment; cameras as kvec[4] / qvec[4] / tvec[3] per view (model_ids NULL = all PINHOLE). */
typedef struct lm_filter_config {
  double th_angular_2d;    /* CheckReprojection: angle(line2d, projection) > th fails (merging_utils.cc:39-43) */
  double th_perp_2d;       /* ... then endpoint-to-line distance > th fails (:44-49) */
  double th_sv_angular_3d; /* CheckSensitivity: Line3d::sensitivity(view) > th fails (merging_utils.cc:101-107) */
  double th_overlap;       /* FilterTracksByOverlap: compute_overlap(projection, line2d) >= th counts (:147-149) */
} lm_filter_config;
typedef struct lm_merge_stats {
  int64_t n_supports;        /* last lm_tracks_support_flags */
  int64_t n_tracks;          /* last lm_remerge_labels */
  int64_t n_pairs_gated;     /* pairs that passed the fp32 angle gate and were checked in fp64 */
  int64_t n_edges;           /* connected pairs */
  int64_t n_kernel_launches; /* cumulative */
  float last_flags_ms, last_flags_kernel_ms, last_remerge_ms, last_remerge_kernel_ms;
} lm_merge_stats;
/* out_flags[S]: bit0 = CheckReprojection result (merging_utils.cc:27-50), bit1 = CheckSensitivity result (:89-109),
 * bit2 = overlap test of FilterTracksByOverlap (:143-150), each for support s of its track's line
 * track_line[t][6] = start3, end3. The callers' selection logic (FilterSupportingLines :52-87,
 * FilterTracksBySensitivity :111-131, FilterTracksByOverlap :133-155) works on these bits. */
int lm_tracks_support_flags(lm_ctx *ctx, int32_t n_views, const int32_t *model_ids, const double *kvec,
                            const double *qvec, const double *tvec, int64_t T, const int64_t *sup_off,
                            const int32_t *sup_view, const double *segs, const double *track_line,
                            const lm_filter_config *cfg, uint8_t *out_flags);
/* Aggregator::aggregate_line3d_list (merging/aggregator.cc:9-101) for T groups of 3D lines:
 * lines[off[T]][7] = start3, end3, uncertainty; scores[off[T]]; out_line[T][7]. Host arithmetic (a 3x3
 * eigen-problem and a sort per group), no device work. */
int lm_aggregate_lines(int64_t T, const int64_t *off, const double *lines, const double *scores,
                       int32_t num_outliers, double *out_line);
/* One pass of RemergeLineTracks up to the group labels (merging/merging.cc:513-598): all-pairs
 * LineLinker3d::check_connection under set_to_spatial_merging() on the device, union-find with the group-size
 * heuristic on the host. track_line[T][7] = start3, end3, uncertainty; active[T]; out_labels[T] = group of each
 * track (groups numbered by their root track, ascending). T <= 65535 * 256 = 16,776,960 (the pair tiles of one grid;
 * LM_ERR_INVALID past it). Returns the number of groups or <0. */
int64_t lm_remerge_labels(lm_ctx *ctx, int64_t T, const double *track_line, const uint8_t *active,
                          const lm_linker_config *linker3d, int32_t *out_labels, int64_t *out_n_edges);
int lm_merge_get_stats(lm_ctx *ctx, lm_merge_stats *out);

/* ---- fit-and-merge: MergeToLineTracks (merging/merging.cc:347-511) with SetUncertaintySegs3d
 * (merging_utils.cc:15-25), the merge step of merging.merging (merging.py:6-21) ------------------------------------
 * Views in ascending image id order: img_ids, model_ids (0 SIMPLE_PINHOLE, 1 PINHOLE), kvec/qvec/tvec as in
 * lm_scene_upload; line_off[n_views+1]; per line its 2D segment segs[n][4] and 3D fit lines3d[n][6] = start3, end3
 * (failed fits are zeros: lines of length 0 are no graph node). Neighbours of view v: the image ids
 * ng_ids[ng_off[v] .. ng_off[v+1]), in the given order, repeats and the image itself allowed. linker2d is used as
 * given, linker3d under set_to_spatial_merging(). Graph nodes are the non-zero lines in (image, line) order; edges
 * are numbered in the reference's insertion order. Limits (LM_ERR_INVALID past them, they size the sort keys):
 * n_views <= 65535, lines per image <= 65535, neighbours per image <= 32767, nodes and edges < 2^31, finite inputs.
 * Returns the number of tracks (>= 0) or <0; out_counts[3] = graph nodes, graph edges, track supports. */
typedef struct lm_fit_merge_stats {
  int64_t n_lines, n_nodes;
  int64_t n_pairs_tested; /* line pairs the reference's loops hand to check_connection_3d */
  int64_t n_pairs_gated;  /* of these, pairs past the fp32 gates, decided with the fp64 formulas */
  int64_t n_edges, n_tracks;
  int64_t n_retries;      /* reruns of the pair kernel after its edge list overflowed (0 or 1) */
  double pair_kernel_ms;  /* device time of the pair kernel (last run when retried) */
  double total_ms;        /* host arrays in to results on the host, wall clock */
} lm_fit_merge_stats;
int64_t lm_merge_fits_build(lm_ctx *ctx, int32_t n_views, const int32_t *img_ids, const int32_t *model_ids,
                            const double *kvec, const double *qvec, const double *tvec, const int64_t *line_off,
                            const double *segs, const double *lines3d, const int64_t *ng_off, const int32_t *ng_ids,
                            double var2d, const lm_linker_config *linker2d, const lm_linker_config *linker3d,
                            int64_t *out_counts);
/* Results of the last lm_merge_fits_build (sizes from its counts): unc[n] = uncertainty of every line, length[n] =
 * its Line3d::length() (the support score, bit-exact), node_line[nodes] = global line index (line_off[v] + line) of each graph node, edges[n_edges][2] = (node1, node2)
 * and sim[n_edges] in insertion order, track_off[T+1], track_nodes[supports] (node order within a track),
 * track_line[T][7] = start3, end3, uncertainty. Any pointer may be NULL. */
int lm_merge_fits_get(lm_ctx *ctx, double *unc, double *length, int64_t *node_line, int32_t *edges, double *sim, int64_t *track_off,
                      int32_t *track_nodes, double *track_line);
int lm_merge_fits_get_stats(lm_ctx *ctx, lm_fit_merge_stats *out);

/* ---- line refinement / line bundle adjustment (cameras constant) ---------------------------------
 * Replaces HybridBAEngine::{InitLineTracks,SetUp,Solve,GetOutputLineTracks}
 * (optimize/hybrid_bundle_adjustment/hybrid_bundle_adjustment.cc:39-59,156-264,298-310) as called by
 * solve_line_bundle_adjustment (optimize/hybrid_bundle_adjustment/solve.py:31-39), and
 * RefinementEngine::{Initialize,SetUp,Solve,GetLine3d} (optimize/line_refinement/refine.cc:19-198):
 * every track is an independent 4-dof Levenberg-Marquardt problem solved by one warp.
 * config: HybridBAConfig / RefinementConfig fields used on this path
 * (optimize/line_refinement/refinement_config.h:18-92). */
typedef struct lm_ba_config {
  double geometric_alpha;   /* 10.0 */
  double cauchy_scale;      /* CauchyLoss(0.25) */
  int32_t max_num_iterations; /* 100 (runners pass 200) */
  int32_t min_num_images;     /* 4: tracks seen in fewer distinct images stay constant */
  int32_t num_outliers;       /* num_outliers_aggregate = 2 */
  int32_t max_num_consecutive_invalid_steps; /* 10 */
  double vp_multiplier;       /* weight of the VP residual relative to the line weight (yaml: 0.1) */
} lm_ba_config;

typedef struct lm_ba_stats {
  int64_t n_tracks, n_blocks;
  int64_t total_iterations;  /* sum over tracks of LM iterations executed (the M2 numerator) */
  int64_t total_successful;
  double solve_ms;           /* device time of the LM kernel (CUDA events on the ctx stream) */
  double prepare_ms;         /* device time of the block-digest kernel */
} lm_ba_stats;

/* Cameras: kvec[n_views][4], qvec[n_views][4], tvec[n_views][3]. Tracks: sup_off[T+1]; per supporting
 * 2D line k: sup_view[k] (index into the camera arrays; also the image identity for count_images),
 * segs[k][4], line3d[k][6] (track.line3d_list, used only to cut the output segment,
 * base/infinite_line.cc:265-287); line_init[T][6] = track.line. Outputs: out_line[T][6] refined segment,
 * out_minimal[T][6] = (uvec, wvec), out_iters[T][2] = (iterations, successful), out_cost[T][2] =
 * (initial, final) cost. Any output may be NULL; line3d may be NULL only when out_line is NULL or there are no
 * supports (LM_ERR_INVALID otherwise), and cfg->num_outliers < 0 is LM_ERR_INVALID. A track with no supports, or
 * with num_outliers >= 2 * its support count, gets line_init as its segment. sup_vp[k][3] (may be NULL):
 * vanishing point of supporting line k for the VP residual of RefinementEngine::AddVPResiduals
 * (refine.cc:86-127), NaN = none. */
int lm_ba_solve(lm_ctx *ctx, int32_t n_views, const double *kvec, const double *qvec, const double *tvec,
                int64_t n_tracks, const int64_t *sup_off, const int32_t *sup_view, const double *segs,
                const double *line3d, const double *line_init, const double *sup_vp, const lm_ba_config *cfg,
                double *out_line,
                double *out_minimal, int32_t *out_iters, double *out_cost);
int lm_ba_get_stats(lm_ctx *ctx, lm_ba_stats *out);

/* ---- vanishing points: JLinkage::AssociateVPs for a batch of images
 * (vplib/JLinkage/JLinkage.cc:14-127; Python glue vplib/base_vp_detector.py:46-78 fans images out with
 * joblib, here all images go to the GPU in one call). The clustering arithmetic of the reference lives in
 * an external library with an unseeded RNG (B1ueber2y/JLinkage@75dadd5); it is restated with a counter-based
 * RNG (`seed`), see DESIGN.md. config: BaseVPDetectorConfig (vplib/base_vp_detector.h:20-35); NB the
 * reference reads th_perp_supports from the shadowed base-class config, i.e. always 3.0. */
typedef struct lm_vp_config {
  double min_length;        /* 40 px */
  double inlier_threshold;  /* 1 px */
  double th_perp_supports;  /* 3 px */
  int32_t min_num_supports; /* 5 (yaml: 10) */
  int32_t n_models;         /* 5000 */
  uint64_t seed;
} lm_vp_config;
/* line_off[n_images+1], segs[sum L][4]. Outputs: labels[sum L] (-1 = no VP), vp_off[n_images+1],
 * vps[vp_cap][3] (homogeneous, unit norm). Returns the total number of VPs (call again with a larger vp_cap
 * if it exceeds vp_cap) or <0. */
int64_t lm_vp_detect(lm_ctx *ctx, int32_t n_images, const int64_t *line_off, const double *segs,
                     const lm_vp_config *cfg, int32_t *labels, int64_t *vp_off, double *vps, int64_t vp_cap);

/* Same, with image_index[n_images] (NULL = 0..n_images-1): the index that seeds the hypotheses of each image. A
 * rank that detects a subset of a scene's images (vplib/base_vp_detector.py:46-78 fans images out over processes)
 * passes their positions in the full list and gets exactly the labels the single call on all images returns. */
int64_t lm_vp_detect_indexed(lm_ctx *ctx, int32_t n_images, const int64_t *line_off, const double *segs,
                             const lm_vp_config *cfg, const int64_t *image_index, int32_t *labels, int64_t *vp_off,
                             double *vps, int64_t vp_cap);
typedef struct lm_vp_stats {
  int64_t n_images, n_segments, n_vps; /* of the last lm_vp_detect: images, segments of min_length, VPs returned */
  double kernel_ms;                    /* device time of the clustering kernel (CUDA events on the ctx stream) */
} lm_vp_stats;
int lm_vp_get_stats(lm_ctx *ctx, lm_vp_stats *out);

/* ---- visual neighbours and robust ranges from a sparse point model (SURVEY.md 8 f4): the step before the path.
 * Replaces SfmModel::{GetMaxIoUImages (mode 0), GetMaxDiceCoeffImages (mode 1), GetMaxOverlapImages (mode 2)}
 * (pointsfm/sfm_model.cc:88-226; Python glue pointsfm/functions.py:20-55) and SfmModel::ComputeRanges (:228-261).
 * Images are indexed 0..n_images-1 (the caller maps indices to image ids as neighbors_vec_to_map does, :75-86);
 * centres[n_images][3] = projection centres; points xyz[n_points][3] with tracks track_off[n_points+1],
 * track_img[] (image indices). out_neighbors[n_images][num_images] (padded with -1), out_count[n_images]. Pairs whose
 * 75th-percentile triangulation angle is below min_triangulation_angle_deg are dropped; ties of the score are broken
 * by ascending image index (the reference's std::sort leaves them unspecified). */
int lm_sfm_rank_neighbors(lm_ctx *ctx, int32_t n_images, const double *centres, int64_t n_points, const double *xyz,
                          const int64_t *track_off, const int32_t *track_img, int32_t num_images,
                          double min_triangulation_angle_deg, int32_t mode, int32_t *out_neighbors, int32_t *out_count);
/* out[6] = lo3, hi3: per axis the (q_lo, q_hi) quantiles of the float coordinates, stretched by kstretch * (hi - lo). */
int lm_sfm_robust_ranges(lm_ctx *ctx, int64_t n_points, const double *xyz, double q_lo, double q_hi, double kstretch,
                         double out[6]);

/* ---- line-map evaluation: PointCloudEvaluator and RefLineEvaluator of evaluation/
 * (evaluation/point_cloud_evaluator.cc, evaluation/base_evaluator.cc, evaluation/refline_evaluator.cc; Python
 * bindings evaluation/bindings.cc:22-133,226-243). Lines are lines[T][6] = (start, end). fp64 throughout; the
 * nearest neighbour is exact (the reference's nanoflann tree with eps = 0). Non-finite coordinates in points or lines
 * are LM_ERR_INVALID. */
typedef struct lm_eval_stats {
  int64_t n_queries; /* nearest-neighbour queries, or point-line / sample-line pairs, of the last call */
  double kernel_ms;  /* device time of its main kernel (CUDA events on the ctx stream) */
  double total_ms;   /* host time of the whole call, copies included */
} lm_eval_stats;
/* The cloud xyz[n_points][3] and its nearest-neighbour index on the ctx (KDTree::initialize + buildIndex,
 * util/kd_tree.cc; PointCloudEvaluator::Build). n_points in [1, 2^31 - 1]; replaces an earlier cloud. */
int lm_eval_build_index(lm_ctx *ctx, int64_t n_points, const double *xyz);
/* PointCloudEvaluator::ComputeDistPoint (point_cloud_evaluator.cc:11-14) of n queries xyz[n][3]: out[n]. */
int lm_eval_point_dists(lm_ctx *ctx, int64_t n, const double *xyz, double *out);
/* BaseEvaluator::ComputeDistLine (base_evaluator.cc:11-25) of T lines: out_mean[T]. n_samples >= 3. */
int lm_eval_line_dists(lm_ctx *ctx, int64_t T, const double *lines, int32_t n_samples, double *out_mean);
/* BaseEvaluator::ComputeInlierRatio and Compute{Inlier,Outlier}SegsOneLine (base_evaluator.cc:27-152) of T lines:
 * out_counts[n_thresholds][T] = samples with distance <= thresholds[k]; out_flags (may be NULL; needs
 * n_thresholds >= 1) = one bit per sample for thresholds[0], bit (l * n_samples + i) % 32 of word
 * (l * n_samples + i) / 32. n_samples >= 1. */
int lm_eval_line_inliers(lm_ctx *ctx, int64_t T, const double *lines, int32_t n_samples, int32_t n_thresholds,
                         const double *thresholds, int32_t *out_counts, uint32_t *out_flags);
/* PointCloudEvaluator::ComputeDistsforEachPoint (sampled = 0, point_cloud_evaluator.cc:17-36) and
 * ComputeDistsforEachPoint_KDTree (sampled = 1, :38-73) against the cloud of lm_eval_build_index: out[n_points],
 * DBL_MAX for every point when T = 0. sampled = 1 needs T * 1000 <= 2^31 - 1. */
int lm_eval_cloud_line_dists(lm_ctx *ctx, int64_t T, const double *lines, int32_t sampled, double *out);
/* RefLineEvaluator::ComputeRecallLength (refline_evaluator.cc:19-44): out_counts[R] = samples of ref_lines[r] within
 * threshold (strictly) of `lines`, out_lengths[R] (may be NULL) = Line3d::length() of ref_lines[r]. The caller sums
 * length * count / n_samples in reference-line order. n_samples in [2, 16776960]. Needs no index. */
int lm_eval_recall_counts(lm_ctx *ctx, int64_t R, const double *ref_lines, int64_t T, const double *lines,
                          double threshold, int32_t n_samples, int32_t *out_counts, double *out_lengths);
/* MeshEvaluator(filename, mpau) (evaluation/mesh_evaluator.cc:13-29) from arrays: V[n_vertices][3], already scaled
 * by mpau, and F[n_faces][3] (int32, 0-based), with its triangle index on the ctx (igl::AABB::init). n_faces and
 * n_vertices in [1, 2^31 - 1], every index in [0, n_vertices), every coordinate finite; replaces an earlier mesh and
 * lives beside the cloud of lm_eval_build_index. */
int lm_eval_build_mesh(lm_ctx *ctx, int64_t n_vertices, const double *V, int64_t n_faces, const int32_t *F);
/* MeshEvaluator::ComputeDistPoint (mesh_evaluator.cc:31-40) of n queries xyz[n][3]: out[n], sqrt of the least
 * igl::point_simplex_squared_distance over all faces, exact (DESIGN.md §3.9). LM_ERR_STATE without a mesh. */
int lm_eval_mesh_point_dists(lm_ctx *ctx, int64_t n, const double *xyz, double *out);
/* BaseEvaluator::ComputeDistLine (base_evaluator.cc:11-25) against the mesh; as lm_eval_line_dists. */
int lm_eval_mesh_line_dists(lm_ctx *ctx, int64_t T, const double *lines, int32_t n_samples, double *out_mean);
/* BaseEvaluator::ComputeInlierRatio and the samples of Compute{Inlier,Outlier}SegsOneLine (base_evaluator.cc:27-120)
 * against the mesh; as lm_eval_line_inliers. */
int lm_eval_mesh_line_inliers(lm_ctx *ctx, int64_t T, const double *lines, int32_t n_samples, int32_t n_thresholds,
                              const double *thresholds, int32_t *out_counts, uint32_t *out_flags);
/* The query count and times of the last lm_eval_* call, cloud or mesh. */
int lm_eval_get_stats(lm_ctx *ctx, lm_eval_stats *out);

/* ---- query pose refinement from 2D-3D point and line matches (cameras of the map constant) --------
 * Replaces JointLocEngine / LineLocEngine::{Initialize,SetUp,Solve,GetFinalQ,GetFinalT,GetInitialCost,GetFinalCost,
 * IsSolutionUsable} (optimize/hybrid_localization/hybrid_localization.{h,cc}) as called by solve_jointloc[_merged] /
 * solve_lineloc[_merged] (optimize/hybrid_localization/solve.py:71-198) and by the ransac.method = None path of
 * _pl_estimate_absolute_pose (estimators/absolute_pose/_pl_estimate_absolute_pose.py:48-80), for many queries in one
 * launch: every query is an independent 6-dof Levenberg-Marquardt problem (qvec on the QuaternionManifold, tvec free,
 * PINHOLE intrinsics constant) solved by one warp.
 * config: LineLocConfig (hybrid_localization_config.h) with the loss object bound in ceresbase/bindings.cc. */
typedef struct lm_loc_config {
  int32_t cost_function;   /* LineLocCostFunction: 0 E2DMidpointDist2, 1 E2DMidpointAngleDist3, 2 E2DPerpendicularDist2,
                              3 E2DPerpendicularDist4, 4 E3DLineLineDist2, 5 E3DPlaneLineDist2 */
  int32_t weight_function; /* LineLocCostFunctionWeight: 0 none, 1 cosine, 2 line3dpp, 3 length, 4 inverse length */
  int32_t loss_kind;       /* 0 TrivialLoss, 1 HuberLoss, 2 SoftLOneLoss, 3 CauchyLoss */
  int32_t points_3d_dist;  /* point residual as a 3D ray distance (set by the engines for the E3D* costs) */
  double loss_scale;       /* the loss's argument a (unused by TrivialLoss) */
  double weight_point;     /* 1.0 */
  double weight_line;      /* 1.0 */
  int32_t max_num_iterations;                /* 100 */
  int32_t max_num_consecutive_invalid_steps; /* 10 */
} lm_loc_config;

typedef struct lm_loc_stats {
  int64_t n_queries, n_blocks;
  int64_t total_iterations, total_successful;
  double kernel_ms; /* device time of the prepare and solve kernels */
  double total_ms;  /* host wall time of the call, copies included */
} lm_loc_stats;

/* Queries: kvec[Q][4] = fx, fy, cx, cy; qvec[Q][4] (w, x, y, z), tvec[Q][3]: the start poses. Points: pt_off[Q+1] into
 * p3d[][3], p2d[][2]. Lines: grp_off[Q+1] into the 3D lines l3d[G][6] (start, end) of each query, l2d_off[G+1] into the
 * 2D lines l2d[][4] matched to each 3D line (the groups of get_line_pairs, solve.py:55-66). Every offset array starts at
 * 0 and is non-decreasing. Outputs: qvec_out[Q][4], tvec_out[Q][3]; out_iters[Q][2] = (iterations, successful steps);
 * out_cost[Q][2] = (initial, final) Ceres cost, 1/2 the sum of the scaled losses; out_flags[Q]: bit0 solved (false when
 * the query has no residuals: its pose is returned unchanged, as Solve() returns false), bit1 the solution is usable.
 * Any output may be NULL. */
int lm_loc_solve(lm_ctx *ctx, int64_t n_queries, const double *kvec, const double *qvec, const double *tvec,
                 const int64_t *pt_off, const double *p3d, const double *p2d, const int64_t *grp_off, const double *l3d,
                 const int64_t *l2d_off, const double *l2d, const lm_loc_config *cfg, double *qvec_out,
                 double *tvec_out, int32_t *out_iters, double *out_cost, uint8_t *out_flags);
/* Sizes, iteration totals and times of the last lm_loc_solve. */
int lm_loc_get_stats(lm_ctx *ctx, lm_loc_stats *out);

/* ---- line matching of query images against a line map (localization) --------------------------------------------
 * Replaces the Python double loops of optimize/hybrid_localization/functions.py as runners/hybrid_localization.py calls
 * them, for every query and every retrieved database image in one pass. An item is a (query image, target image) pair;
 * items come in query order, then retrieval order, and a query is a run of items with the same query image. Every
 * output list keeps the reference's order. Outputs stay on the device until lm_locmatch_get: a caller sizes its buffers
 * from the returned count, then fetches. */
typedef struct lm_locmatch_stats {
  int64_t n_items, n_tests;  /* items and IoU tests of the last sweep or filter */
  int64_t n_pairs_2to2;      /* pairs past the IoU test (tracked or not) */
  int64_t n_out;             /* pairs in the last result */
  double kernel_ms;          /* device time of the last call's kernels, host waits between them excluded */
  double test_ms;            /* device time of the IoU test kernel of the last sweep or filter */
  double total_ms;           /* host wall time of the last call, copies included */
} lm_locmatch_stats;

/* The scene: n_images images with kvec[n][4] = fx, fy, cx, cy, qvec[n][4] (w, x, y, z), tvec[n][3]; their 2D lines as
 * line_off[n+1] into lines[][4]; line_track[] the track of every line (-1: untracked; the inverse id map of
 * base.get_invert_idmap_from_linetracks, base/functions.py:50-72; NULL without a map) and the tracks' lines
 * track_lines[n_tracks][6] (start, end). */
int lm_locmatch_set_scene(lm_ctx *ctx, int32_t n_images, const double *kvec, const double *qvec, const double *tvec,
                          const int64_t *line_off, const double *lines, const int32_t *line_track, int64_t n_tracks,
                          const double *track_lines);
/* match_line_2to2_epipolarIoU (functions.py:6-23) of every item items[n][2] = (query image, target image): the pairs
 * (query line, target line) with compute_epipolar_IoU > IoU_threshold, query line major. to_tracks: fused with
 * match_line_2to3 (functions.py:55-66), pairs (query line, track) of the tracked target lines only. Returns the number
 * of pairs; lm_locmatch_get gives them with offsets per item. */
int64_t lm_locmatch_sweep(lm_ctx *ctx, int64_t n_items, const int32_t *items, double IoU_threshold, int32_t to_tracks);
/* filter_line_2to2_epipolarIoU (functions.py:26-52) of given pairs: pair_off[n_items+1] into pairs[][2] = (query line,
 * target line) per item, kept in order when compute_epipolar_IoU > IoU_threshold (every pair when use_iou is 0).
 * to_tracks as for lm_locmatch_sweep. Returns the number of pairs kept. */
int64_t lm_locmatch_filter(lm_ctx *ctx, int64_t n_items, const int32_t *items, const int64_t *pair_off,
                           const int32_t *pairs, int32_t use_iou, double IoU_threshold, int32_t to_tracks);
/* The (query line, track) pairs of the last to_tracks sweep or filter, grouped per query as the runner's defaultdict
 * all_line_pairs_2to3 holds them (runners/hybrid_localization.py:284-346): query lines in order of first appearance,
 * tracks in append order, duplicates kept. dist_func -1 returns that list; 0 perpendicular_dist, 1 midpoint_dist,
 * 2 midpoint_perpendicular_dist apply reprojection_filter_matches_2to3 (functions.py:96-140) with the query image's
 * camera and dist_thres, sine_thres, angle_scale, one pair per query line at most. Returns the number of pairs;
 * lm_locmatch_get gives them with offsets per query. */
int64_t lm_locmatch_group(lm_ctx *ctx, int32_t dist_func, double dist_thres, double sine_thres, double angle_scale);
/* The last result: off[n+1] (n items for sweep / filter, n queries for group) and pairs[cap][2]; cap must hold them. */
int lm_locmatch_get(lm_ctx *ctx, int64_t *off, int32_t *pairs, int64_t cap);
int lm_locmatch_get_stats(lm_ctx *ctx, lm_locmatch_stats *out);

#ifdef __cplusplus
}
#endif
#endif /* LIMAP_B200_H */
