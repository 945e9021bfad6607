"""Localization line matching on the GPU (lm_locmatch_*, locmatch_kernels.cu) against the reference's functions.py
(tests/golden/ref/loc_matching.npz) and the fp64 oracle (oracle/orc_locmatch.cpp): the same pair lists in the same
order; and runners.hybrid_localization end to end against the per-query composition."""
import os
import sys

import numpy as np
import pytest

from limap_b200 import base
from limap_b200 import hybrid_localization_functions as fn
from oracle import locmatch as om

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import locmatch_cases as lc  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "loc_matching.npz")
CASES = {"seed0": dict(seed=0), "seed1_planted": dict(seed=1, planted=True)}
MODEL = {0: "SIMPLE_PINHOLE", 1: "PINHOLE"}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _as_list(a):
    return [tuple(map(int, p)) for p in np.asarray(a).reshape(-1, 2)]


def _camera(c):
    K = np.array([[c[1], 0, c[3]], [0, c[2], c[4]], [0, 0, 1.0]])
    return base.Camera(MODEL[int(c[0])], K, 0, (600, 800))


def _pose(c, as_tuple):
    return (c[5:9], c[9:12]) if as_tuple else base.CameraPose(c[5:9], c[9:12])


def _view(c):
    return base.CameraView(_camera(c), base.CameraPose(c[5:9], c[9:12]))


def _lines(a):
    return [base.Line2d(s[:2], s[2:]) for s in a]


@pytest.mark.parametrize("tag", sorted(CASES))
def test_2to2_and_filter_equal_reference_and_oracle(golden, tag):
    case = lc.make_case(**CASES[tag])
    cams, lines = case["cams"], case["lines"]
    k = 0
    for q in case["q_ids"]:
        for d in case["retrieval"][q]:
            k += 1
            as_tuple = bool(k % 2)  # poses alternately as CameraPose and as (qvec, tvec)
            for th in lc.THRESHOLDS:
                got = fn.match_line_2to2_epipolarIoU(_lines(lines[q]), lines[d], _camera(cams[q]),
                                                     _pose(cams[q], as_tuple), _camera(cams[d]),
                                                     _pose(cams[d], not as_tuple), th)
                assert got == _as_list(golden[f"{tag}/m22/{q}/{d}/{th}"]), (q, d, th)
                assert got == om.match_2to2(lines[q], cams[q], lines[d], cams[d], th)
            got = fn.filter_line_2to2_epipolarIoU(case["pairs"][q][d], lines[q], _lines(lines[d]), _camera(cams[q]),
                                                  _pose(cams[q], as_tuple), _camera(cams[d]), _pose(cams[d], as_tuple),
                                                  0.2)
            assert got == _as_list(golden[f"{tag}/f22/{q}/{d}"]), (q, d)


@pytest.mark.parametrize("tag", sorted(CASES))
@pytest.mark.parametrize("mode", ["epipolar", "learned", "learned_filter"])
@pytest.mark.parametrize("rf", [None] + list(lc.REPROJ_FUNCS))
def test_batched_matching_equals_reference_order(golden, tag, mode, rf):
    case = lc.make_case(**CASES[tag])
    tracks = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in case["tracks"]]
    got = fn.match_queries_to_linemap(
        {q: _view(case["cams"][q]) for q in case["q_ids"]}, {q: case["lines"][q] for q in case["q_ids"]},
        {d: _view(case["cams"][d]) for d in case["db_ids"]}, case["lines"], case["retrieval"], tracks,
        {d: list(v) for d, v in case["line2track"].items()}, IoU_threshold=0.2,
        line_pairs_2to2=None if mode == "epipolar" else case["pairs"], epipolar_filter=mode == "learned_filter",
        reprojection_filter=rf)
    for q in case["q_ids"]:
        assert got[q] == _as_list(golden[f"{tag}/run/{mode}/{rf}/{q}"]), q


def test_batched_matching_equals_per_call_composition():
    case = lc.make_case(seed=0)
    cams, lines = case["cams"], case["lines"]
    l2t = {d: list(map(int, v)) for d, v in case["line2track"].items()}
    tracks = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in case["tracks"]]
    got = fn.match_queries_to_linemap({q: _view(cams[q]) for q in case["q_ids"]}, lines,
                                      {d: _view(cams[d]) for d in case["db_ids"]}, lines, case["retrieval"],
                                      tracks, l2t, IoU_threshold=0.1, reprojection_filter="Midpoint")
    for q in case["q_ids"]:
        acc = {}
        for d in case["retrieval"][q]:
            p22 = fn.match_line_2to2_epipolarIoU(lines[q], lines[d], _camera(cams[q]), _pose(cams[q], True),
                                                 _camera(cams[d]), _pose(cams[d], True), 0.1)
            for i, t in fn.match_line_2to3(p22, l2t, d):
                acc.setdefault(i, []).append(t)
        want = fn.reprojection_filter_matches_2to3(_lines(lines[q]), _view(cams[q]), acc, tracks, dist_thres=2,
                                                   dist_func=fn.midpoint_dist)
        assert got[q] == want, q


def _boundary(decide, lo=0.0, hi=1e6):
    """The smallest double threshold at which decide(th) is True (decide monotone), by bisection on the bit pattern."""
    a, b = int(np.float64(lo).view(np.int64)), int(np.float64(hi).view(np.int64))  # (non-negative doubles)
    assert not decide(lo) and decide(hi)
    while b - a > 1:
        m = (a + b) // 2
        if decide(float(np.int64(m).view(np.float64))):
            b = m
        else:
            a = m
    return float(np.int64(b).view(np.float64))


def _behind(cam, X):
    """The point whose camera-frame coordinates are those of X negated: it projects behind the camera."""
    from limap_b200.base import _quat_to_R
    R, t = _quat_to_R(cam[5:9]), cam[9:12]
    return R.T @ (-(R @ X + t) - t)


@pytest.mark.parametrize("rf", lc.REPROJ_FUNCS)
def test_reprojection_filter_boundaries(rf):
    case = lc.make_case(seed=0)
    q = case["q_ids"][1]
    cam, qlines = case["cams"][q], case["lines"][q]
    T = case["tracks"]
    n = len(T)
    # tracks n, n+1: copies of track 3 (equal loss: the lowest id wins); n+2: track 3 behind the camera
    tracks = np.concatenate([T, T[3:4], T[3:4], np.r_[_behind(cam, T[3, :3]), _behind(cam, T[3, 3:])][None]])
    view = _view(cam)
    tl = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in tracks]
    dist_func = fn.get_reprojection_dist_func(rf)
    cand = {i: [n + 1, 3, n + 2, n, 5, 5, 7] for i in range(len(qlines))}
    for kw in (dict(dist_thres=1e9, sine_thres=1.5), dict(dist_thres=10.0), dict(dist_thres=2.0, sine_thres=0.1)):
        got = fn.reprojection_filter_matches_2to3(_lines(qlines), view, cand, tl, dist_func=dist_func, **kw)
        want = om.reproj_filter(qlines, cam, cand, tracks, rf, **kw)
        assert got == want, kw
        assert all(t != n + 1 and t != n for _, t in got)  # ties go to the lowest id (3)
    # the distance gate and the sine gate hit exactly: at the boundary double and the one below it
    for i in range(4):
        one = {i: [3]}
        dth = _boundary(lambda th: om.reproj_filter(qlines, cam, one, tracks, rf, dist_thres=th, sine_thres=2.0) != [])
        for th in (dth, np.nextafter(dth, -np.inf)):
            got = fn.reprojection_filter_matches_2to3(_lines(qlines), view, one, tl, dist_thres=th, sine_thres=2.0,
                                                      dist_func=dist_func)
            assert got == om.reproj_filter(qlines, cam, one, tracks, rf, dist_thres=th, sine_thres=2.0), (i, th)
        if rf == "Midpoint":
            sth = _boundary(lambda th: om.reproj_filter(qlines, cam, one, tracks, rf, dist_thres=1e300,
                                                        sine_thres=th) != [], 0.0, 2.0)
            for th in (sth, np.nextafter(sth, -np.inf)):
                got = fn.reprojection_filter_matches_2to3(_lines(qlines), view, one, tl, dist_thres=1e300,
                                                          sine_thres=th, dist_func=dist_func)
                assert got == om.reproj_filter(qlines, cam, one, tracks, rf, dist_thres=1e300, sine_thres=th)
    with pytest.raises(ValueError):
        fn.reprojection_filter_matches_2to3(_lines(qlines), view, cand, tl, dist_func=lambda a, b: 0.0)


# ---- runners.hybrid_localization end to end ------------------------------------------------------------------------
def _loc_set(tmp, case, learned):
    from limap_b200.util import io as limapio
    seg_dir = os.path.join(tmp, "line_detections", "lsd", "segments")
    os.makedirs(seg_dir)
    for img, segs in case["lines"].items():
        limapio.save_txt_segments(seg_dir, img, segs)
    cams, imgs_db, imgs_q = {}, {}, {}
    for img, c in case["cams"].items():
        cam = _camera(c)
        cam.cam_id = img
        cams[img] = cam
        im = base.CameraImage(img, base.CameraPose(c[5:9], c[9:12]), case["names"][img])
        (imgs_q if img in case["q_ids"] else imgs_db)[img] = im
    col_db = base.ImageCollection({i: cams[i] for i in imgs_db}, imgs_db)
    col_q = base.ImageCollection({i: cams[i] for i in imgs_q}, imgs_q)
    tracks = []
    for tid, t in enumerate(case["tracks"]):
        obs = [(d, j) for d in case["db_ids"] for j, v in enumerate(case["line2track"][d]) if v == tid]
        tracks.append(base.LineTrack(base.Line3d(t[:3], t[3:]), [o[0] for o in obs], [o[1] for o in obs],
                                     [base.Line2d(case["lines"][o[0]][o[1]][:2], case["lines"][o[0]][o[1]][2:])
                                      for o in obs]))
    rng = np.random.default_rng(5)
    corresp = {}
    for q in case["q_ids"]:
        X = rng.uniform(-1, 1, (30, 3))
        view = _view(case["cams"][q])
        corresp[q] = dict(p3ds=X, p2ds=np.array([view.projection(x) for x in X]) + rng.normal(size=(30, 2)))
    if learned:
        folder = os.path.join(tmp, "line_matchings", "lsd", "feats_sold2", "sold2_n5_top0")
        os.makedirs(folder)
        for q in case["q_ids"]:
            limapio.save_npy(os.path.join(folder, f"matches_{q}.npy"),
                             {d: np.array(p, np.int64).reshape(-1, 2) for d, p in case["pairs"][q].items()})
    retrieval = {case["names"][q]: [case["names"][d] for d in case["retrieval"][q]] for q in case["q_ids"]}
    return col_db, col_q, corresp, tracks, retrieval


def _cfg(tmp, matcher, rf, ransac=None):
    return {"dir_save": tmp, "dir_load": tmp, "load_det": True, "n_neighbors_loc": 5,
            "line2d": {"detector": {"method": "lsd"}},
            "localization": {"2d_matcher": matcher, "epipolar_filter": False, "IoU_threshold": 0.2,
                             "reprojection_filter": rf, "skip_exists": False, "ransac": {"method": ransac},
                             "line_cost_func": "PerpendicularDist", "line_weight": 1.0,
                             "optimize": {"loss_func": "HuberLoss", "loss_func_args": [1.0]}}}


@pytest.mark.parametrize("matcher", ["epipolar", "sold2"])
@pytest.mark.parametrize("rf", [None, "Perpendicular"])
def test_runner_end_to_end(tmp_path, matcher, rf):
    import pathlib

    import limap
    import limap.estimators as est
    case = lc.make_case(seed=0, empty_images=False)  # the segment files of the runner need at least one line each
    tmp = str(tmp_path)
    col_db, col_q, corresp, tracks, retrieval = _loc_set(tmp, case, matcher != "epipolar")
    cfg = _cfg(tmp, matcher, rf)
    results = pathlib.Path(tmp) / "results.txt"
    poses = limap.runners.hybrid_localization(cfg, col_db, col_q, corresp, tracks, retrieval, results)
    # per-query composition: oracle matching in the runner's order, then pl_estimate_absolute_pose
    want = om.match_queries({q: (case["cams"][q], case["lines"][q]) for q in case["q_ids"]},
                            {d: (case["cams"][d], case["lines"][d]) for d in case["db_ids"]}, case["retrieval"],
                            case["line2track"], case["tracks"], 0.2,
                            pairs_2to2=None if matcher == "epipolar" else case["pairs"], reprojection_filter=rf)
    lines_out = []
    for q in case["q_ids"]:
        pairs = want[q]
        l3ds = [t.line for t in tracks]
        l2ds = [base.Line2d(case["lines"][q][i][:2], case["lines"][q][i][2:]) for i, _ in pairs]
        cam = col_q.cam(col_q.camimage(q).cam_id)
        pose, _ = est.pl_estimate_absolute_pose(cfg["localization"], l3ds, [t for _, t in pairs], l2ds,
                                                corresp[q]["p3ds"], corresp[q]["p2ds"], cam, col_q.campose(q))
        assert np.abs(poses[q].qvec - pose.qvec).max() <= 1e-9 and np.abs(poses[q].tvec - pose.tvec).max() <= 1e-9
        lines_out.append(" ".join([case["names"][q]] + [str(x) for x in poses[q].qvec] +
                                  [str(x) for x in poses[q].tvec]) + "\n")
    assert results.read_text() == "".join(lines_out)
    with pytest.raises(NotImplementedError, match="PoseLib"):
        limap.runners.hybrid_localization(_cfg(tmp, matcher, rf, "hybrid"), col_db, col_q, corresp, tracks,
                                          retrieval, pathlib.Path(tmp) / "r2.txt")
    assert not (pathlib.Path(tmp) / "r2.txt").exists()


def test_many_queries_without_2to3_matches():
    """40 queries against an untracked map under the reprojection filter: no 2D-3D entry at all, and the per-query
    offsets still cover every query; the next call on the same context is unaffected."""
    case = lc.make_case(seed=0, empty_images=False)
    cams, lines = case["cams"], case["lines"]
    q0 = case["q_ids"][0]
    qids = list(range(1000, 1040))
    views = {q: _view(cams[q0]) for q in qids}
    untracked = {d: [-1] * len(lines[d]) for d in case["db_ids"]}
    tracks = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in case["tracks"]]
    for rf in lc.REPROJ_FUNCS:
        got = fn.match_queries_to_linemap(views, {q: lines[q0] for q in qids}, {d: _view(cams[d]) for d in case["db_ids"]},
                                          lines, {q: case["db_ids"][:2] for q in qids}, tracks, untracked,
                                          IoU_threshold=0.0, reprojection_filter=rf)
        assert got == {q: [] for q in qids}
    # the same context afterwards: the reference's order on the planted case
    golden = dict(np.load(GOLDEN))
    test_batched_matching_equals_reference_order(golden, "seed1_planted", "epipolar", "Midpoint")


def test_results_need_a_tracks_pass_and_line2track_matches_lines():
    from limap_b200 import _cabi
    case = lc.make_case(seed=0)
    cams, lines = case["cams"], case["lines"]
    q, d = case["q_ids"][0], case["db_ids"][0]
    fn.match_line_2to2_epipolarIoU(lines[q], lines[d], _camera(cams[q]), _pose(cams[q], True), _camera(cams[d]),
                                   _pose(cams[d], True), 0.2)  # a plain 2to2 result: nothing to group
    with pytest.raises(_cabi.LimapB200Error, match="to_tracks"):
        fn._group(fn._context(), 1)
    tracks = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in case["tracks"]]
    l2t = {k: list(v) for k, v in case["line2track"].items()}
    l2t[d] = l2t[d][:-1]
    with pytest.raises(ValueError, match="one entry per line"):
        fn.match_queries_to_linemap({q: _view(cams[q])}, lines, {d: _view(cams[d])}, lines, {q: [d]}, tracks, l2t)


def test_filter_counts_pairs_past_the_iou_test(golden):
    """n_pairs_2to2 of a filter with to_tracks counts the pairs past the IoU test, tracked or not."""
    case = lc.make_case(seed=0)
    tracks = [base.LineTrack(base.Line3d(t[:3], t[3:]), [], [], []) for t in case["tracks"]]
    q = case["q_ids"][0]
    fn.match_queries_to_linemap({q: _view(case["cams"][q])}, case["lines"],
                                {d: _view(case["cams"][d]) for d in case["db_ids"]}, case["lines"],
                                {q: case["retrieval"][q]}, tracks, {d: list(v) for d, v in case["line2track"].items()},
                                line_pairs_2to2=case["pairs"], epipolar_filter=True)
    # the stats of the last call are the group's; rerun the filter alone
    order = list(dict.fromkeys(case["retrieval"][q]))  # the scene's database images, in order of first retrieval
    fn._filter(fn._context(), [(0, 1 + order.index(d)) for d in case["retrieval"][q]],
               [case["pairs"][q][d] for d in case["retrieval"][q]], True, 0.2, True)
    st = fn.stats()
    assert st["n_pairs_2to2"] == sum(len(golden[f"seed0/f22/{q}/{d}"]) for d in case["retrieval"][q])
    assert 0 < st["test_ms"] <= st["kernel_ms"]


def test_query_endpoint_at_the_epipole():
    """A query line starting exactly at the (rounded) epipole of the target: F x of that endpoint carries no correct
    digit in any evaluation order, so only the other query lines' pairs are held to the oracle; the call itself runs."""
    case = lc.make_case(seed=0)
    cams, lines = case["cams"], case["lines"]
    q, d = case["q_ids"][0], case["db_ids"][1]
    ql = lines[q].copy()
    ql[0, :2] -= np.array([0.6, 0.8])  # back onto the projected camera centre (locmatch_cases places it 1 px off)
    for th in lc.THRESHOLDS:
        got = fn.match_line_2to2_epipolarIoU(ql, lines[d], _camera(cams[q]), _pose(cams[q], False), _camera(cams[d]),
                                             _pose(cams[d], False), th)
        want = om.match_2to2(ql, cams[q], lines[d], cams[d], th)
        assert [p for p in got if p[0] != 0] == [p for p in want if p[0] != 0], th
