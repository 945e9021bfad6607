"""limap.optimize.hybrid_localization.functions: 2D line matching of query images against a line map.

Mirrors src/limap/optimize/hybrid_localization/functions.py. The epipolar matcher `match_line_2to2_epipolarIoU`, its
filter `filter_line_2to2_epipolarIoU` and `reprojection_filter_matches_2to3` run on the GPU (lm_locmatch_*, include/
limap_b200.h): every (query line, target line) IoU test is one fp64 evaluation of compute_epipolar_IoU in an all-pairs
sweep, and outputs keep the reference's order. `match_line_2to3`, the three distance functions and
`get_reprojection_dist_func` are host code, as in the reference; callers pass the distance functions by identity.

`match_queries_to_linemap` is an extension: the matching stage of runners/hybrid_localization.py for all queries and all
their retrieved images in one pass over the device.

Out of scope: learned line extraction and matching (their `matches_{qid}.npy` files are read, not produced), hloc's point
correspondences and the RANSAC estimators.
"""
import ctypes as C

import numpy as np

from . import _cabi, base
from ._cabi import check, lib, ptr

_ctx = None  # created on the first call


def _context():
    global _ctx
    if _ctx is None:
        _ctx = _cabi.Context(0)
    return _ctx


def _pose(p):
    return p if isinstance(p, base.CameraPose) else base.CameraPose(p[0], p[1])


def _lines_array(lines):
    if isinstance(lines, np.ndarray):
        return np.ascontiguousarray(lines, np.float64).reshape(-1, 4)
    return np.array([np.concatenate([np.asarray(l.start, np.float64), np.asarray(l.end, np.float64)])
                     if hasattr(l, "start") else np.asarray(l, np.float64).reshape(4) for l in lines],
                    np.float64).reshape(-1, 4)


def _track_lines(linetracks):
    out = np.zeros((len(linetracks), 6))
    for i, t in enumerate(linetracks):
        line = t.line if hasattr(t, "line") else t
        out[i, :3], out[i, 3:] = line.start, line.end
    return out


class _Scene:
    """The flat arrays of lm_locmatch_set_scene: one entry per image (camera, pose, 2D lines, line -> track)."""

    def __init__(self):
        self.kvec, self.qvec, self.tvec, self.lines, self.tracks = [], [], [], [], []

    def add(self, cam, pose, lines, track_ids=None):
        pose = _pose(pose)
        self.kvec.append(np.asarray(cam.kvec(), np.float64))
        self.qvec.append(np.asarray(pose.qvec, np.float64))
        self.tvec.append(np.asarray(pose.tvec, np.float64))
        arr = _lines_array(lines)
        self.lines.append(arr)
        if track_ids is None:
            track_ids = np.full(len(arr), -1, np.int32)
        track_ids = np.asarray(track_ids, np.int32).reshape(-1)
        if len(track_ids) != len(arr):
            raise ValueError(f"{len(track_ids)} track ids for {len(arr)} lines: line2track must hold one entry per line")
        self.tracks.append(track_ids)
        return len(self.kvec) - 1

    def upload(self, ctx, track_lines=None):
        n = len(self.kvec)
        f = lambda a, k: np.ascontiguousarray(np.array(a, np.float64).reshape(-1, k))
        self._keep = dict(kvec=f(self.kvec, 4), qvec=f(self.qvec, 4), tvec=f(self.tvec, 3),
                          line_off=np.r_[0, np.cumsum([len(a) for a in self.lines])].astype(np.int64),
                          lines=f(np.concatenate(self.lines) if n else np.zeros((0, 4)), 4),
                          track=np.ascontiguousarray(np.concatenate(self.tracks) if n else np.zeros(0), np.int32),
                          tl=f(track_lines if track_lines is not None else np.zeros((0, 6)), 6))
        k = self._keep
        check(lib().lm_locmatch_set_scene(ctx.handle, n, ptr(k["kvec"]), ptr(k["qvec"]), ptr(k["tvec"]),
                                          ptr(k["line_off"]), ptr(k["lines"]), ptr(k["track"]), len(k["tl"]),
                                          ptr(k["tl"])))


def _fetch(ctx, count, n_off):
    off = np.zeros(n_off + 1, np.int64)
    pairs = np.zeros((max(count, 0), 2), np.int32)
    check(lib().lm_locmatch_get(ctx.handle, ptr(off), ptr(pairs), len(pairs)))
    return off, pairs


def _items(items):
    return np.ascontiguousarray(np.array(items, np.int32).reshape(-1, 2))


def _sweep(ctx, items, th, to_tracks):
    it = _items(items)
    n = check(lib().lm_locmatch_sweep(ctx.handle, len(it), ptr(it), float(th), int(to_tracks)))
    return _fetch(ctx, n, len(it))


def _filter(ctx, items, pair_lists, use_iou, th, to_tracks):
    it = _items(items)
    pair_off = np.r_[0, np.cumsum([len(p) for p in pair_lists])].astype(np.int64)
    pairs = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int64).reshape(-1, 2)[:, :2] for p in pair_lists])
                                 if len(pair_lists) else np.zeros((0, 2)), np.int32)
    n = check(lib().lm_locmatch_filter(ctx.handle, len(it), ptr(it), ptr(pair_off), ptr(pairs), int(bool(use_iou)),
                                       float(th), int(to_tracks)))
    return n


_DIST_CODE = {}  # distance function -> lm_locmatch_group's dist_func


def _group(ctx, n_queries, dist_func=None, dist_thres=10, sine_thres=0.4, angle_scale=1.0):
    code = -1 if dist_func is None else _DIST_CODE.get(dist_func)
    if code is None:
        raise ValueError(f"reprojection_filter_matches_2to3: {dist_func!r} is none of perpendicular_dist, midpoint_dist "
                         "and midpoint_perpendicular_dist; other distance functions are not supported (no CPU path)")
    n = check(lib().lm_locmatch_group(ctx.handle, code, float(dist_thres), float(sine_thres), float(angle_scale)))
    return _fetch(ctx, n, n_queries)


def stats():
    """Counts and times of the last lm_locmatch_* call (n_tests, n_pairs_2to2, n_out, kernel_ms, test_ms, total_ms)."""
    st = _cabi.LocMatchStats()
    check(lib().lm_locmatch_get_stats(_context().handle, C.byref(st)))
    return {k: getattr(st, k) for k, _ in _cabi.LocMatchStats._fields_}


def _tuples(pairs):
    return [(int(a), int(b)) for a, b in pairs.tolist()]


def match_line_2to2_epipolarIoU(ref_lines, tgt_lines, ref_cam, ref_pose, tgt_cam, tgt_pose, IoU_threshold):
    """functions.py:6-23: the (ref line, tgt line) pairs with compute_epipolar_IoU > IoU_threshold, ref line major."""
    ctx, sc = _context(), _Scene()
    sc.add(ref_cam, ref_pose, ref_lines)
    sc.add(tgt_cam, tgt_pose, tgt_lines)
    sc.upload(ctx)
    return _tuples(_sweep(ctx, [(0, 1)], IoU_threshold, False)[1])


def filter_line_2to2_epipolarIoU(pairs, ref_lines, tgt_lines, ref_cam, ref_pose, tgt_cam, tgt_pose, IoU_threshold):
    """functions.py:26-52: the given pairs whose compute_epipolar_IoU > IoU_threshold, in their order."""
    ctx, sc = _context(), _Scene()
    sc.add(ref_cam, ref_pose, ref_lines)
    sc.add(tgt_cam, tgt_pose, tgt_lines)
    sc.upload(ctx)
    n = _filter(ctx, [(0, 1)], [list(pairs)], True, IoU_threshold, False)
    return _tuples(_fetch(ctx, n, 1)[1])


def match_line_2to3(pairs_2to2, line2track, tgt_img_id):  # functions.py:55-66
    track_ids = line2track[tgt_img_id]
    pairs_2to3 = []
    for pair in pairs_2to2:
        ref_line_id, tgt_line_id = int(pair[0]), int(pair[1])
        if track_ids[tgt_line_id] != -1:
            pairs_2to3.append((ref_line_id, track_ids[tgt_line_id]))
    return pairs_2to3


def midpoint_dist(ref_line, tgt_line):  # functions.py:69-70
    return np.linalg.norm(ref_line.midpoint() - tgt_line.midpoint())


def midpoint_perpendicular_dist(ref_line, tgt_line):  # functions.py:73-78
    m = ref_line.midpoint()
    t, d = tgt_line.start, tgt_line.direction()
    return np.abs(d[0] * (t - m)[1] - d[1] * (t - m)[0]) / ref_line.length()


def perpendicular_dist(ref_line, tgt_line):  # functions.py:81-86
    s, e = ref_line.start, ref_line.end
    t, d = tgt_line.start, tgt_line.direction()
    return 0.5 * (np.abs(d[0] * (t - s)[1] - d[1] * (t - s)[0]) + np.abs(d[0] * (t - e)[1] - d[1] * (t - e)[0]))


_DIST_CODE.update({perpendicular_dist: 0, midpoint_dist: 1, midpoint_perpendicular_dist: 2})
_DIST_NAMES = {"Perpendicular": perpendicular_dist, "Midpoint": midpoint_dist,
               "Midpoint_Perpendicular": midpoint_perpendicular_dist}


def get_reprojection_dist_func(func_name):  # functions.py:89-96
    if func_name in _DIST_NAMES:
        return _DIST_NAMES[func_name]
    raise ValueError(f"[Error] Unknown dist function: {func_name}")


def reprojection_filter_matches_2to3(ref_lines, ref_camview, all_pairs_2to3, linetracks, dist_thres=10,
                                     sine_thres=0.4, angle_scale=1.0, dist_func=midpoint_dist):
    """functions.py:99-140: for every query line (in the order of all_pairs_2to3), the track whose projection into
    ref_camview has the least loss under the distance and angle gates; ties go to the lowest track id. dist_func must be
    one of this module's three distance functions."""
    if dist_func not in _DIST_CODE:
        _group(None, 0, dist_func)  # raises
    ctx, sc = _context(), _Scene()
    keys = list(all_pairs_2to3)
    cand = [int(t) for k in keys for t in all_pairs_2to3[k]]
    if any(t < 0 or t >= len(linetracks) for t in cand):
        raise IndexError("a track id of all_pairs_2to3 is outside linetracks")
    sc.add(ref_camview.cam, ref_camview.pose, ref_lines)
    # the candidates as the given pairs of one item: a target image whose j-th line is on the j-th candidate's track
    sc.add(ref_camview.cam, ref_camview.pose, np.zeros((len(cand), 4)), cand)
    sc.upload(ctx, _track_lines(linetracks))
    pairs = [(int(k), j) for j, k in enumerate(int(k) for k in keys for _ in all_pairs_2to3[k])]
    _filter(ctx, [(0, 1)], [pairs], False, 0.0, True)
    return _tuples(_group(ctx, 1, dist_func, dist_thres, sine_thres, angle_scale)[1])


def match_queries_to_linemap(query_views, query_lines, db_views, db_lines, retrieval, linetracks, line2track,
                             IoU_threshold=0.2, line_pairs_2to2=None, epipolar_filter=False, reprojection_filter=None,
                             dist_thres=2, sine_thres=0.4, angle_scale=1.0, as_arrays=False):
    """The 2D-3D line matches of runners/hybrid_localization.py:284-346 for every query in one pass over the device.

    query_views / db_views: {image id: CameraView} (the query poses are the coarse ones), query_lines / db_lines:
    {image id: 2D lines}, retrieval: {query id: [db image ids]} in retrieval order, linetracks: the line map,
    line2track: base.get_invert_idmap_from_linetracks(db_lines, linetracks). Matcher: the epipolar one when
    line_pairs_2to2 is None, else the given pairs {query id: {db image id: [(query line, db line), ...]}}, filtered by
    the epipolar IoU when epipolar_filter. reprojection_filter: None or a get_reprojection_dist_func name.

    Returns {query id: [(query line, track id), ...]} in the order the reference runner builds it (numpy [n, 2] int32
    arrays with as_arrays)."""
    dist_func = None if reprojection_filter is None else get_reprojection_dist_func(reprojection_filter)
    ctx, sc = _context(), _Scene()
    qids = list(query_views)
    qidx = {q: sc.add(query_views[q].cam, query_views[q].pose, query_lines[q]) for q in qids}
    dbidx = {}
    for q in qids:
        for t in retrieval[q]:
            if t not in dbidx:
                dbidx[t] = sc.add(db_views[t].cam, db_views[t].pose, db_lines[t], line2track[t])
    sc.upload(ctx, _track_lines(linetracks))
    items = [(qidx[q], dbidx[t]) for q in qids for t in retrieval[q]]
    if line_pairs_2to2 is None:
        _sweep(ctx, items, IoU_threshold, True)
    else:
        _filter(ctx, items, [line_pairs_2to2[q][t] for q in qids for t in retrieval[q]], epipolar_filter,
                IoU_threshold, True)
    # queries with no retrieved image have no items and no matches
    with_items = [q for q in qids if len(retrieval[q])]
    off, pairs = _group(ctx, len(with_items), dist_func, dist_thres, sine_thres, angle_scale)
    out = {q: (pairs[:0] if as_arrays else []) for q in qids}
    for i, q in enumerate(with_items):
        seg = pairs[off[i]:off[i + 1]]
        out[q] = seg if as_arrays else _tuples(seg)
    return out
