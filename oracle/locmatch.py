"""ctypes wrapper of the localization line-matching oracle (oracle/orc_locmatch.cpp). TEST INFRASTRUCTURE ONLY: imported
by tests/ and scripts/, never by limap_b200/.

  match_2to2 / filter_2to2 / reproj_one   the fp64 restatements of functions.py's three GPU functions
  match_queries                           the runner's matching stage (runners/hybrid_localization.py:284-346) composed
                                          from them in the reference's order: per query, per retrieved image, 2to2
                                          pairs, then match_line_2to3 into a defaultdict, then the optional
                                          reprojection filter or the flat list
  ref_count                               the reference's compiled compute_epipolar_IoU in a C loop on all host cores
                                          (oracle/ref_locmatch.cpp -> oracle/_ref/liblimap_ref_locmatch.so; built only
                                          where the reference source tree exists), for scripts/bench_loc_matching.py"""
import ctypes as C
import os
from collections import defaultdict

import numpy as np

from . import evaluation as _ev
from . import ref as _ref

_HERE = os.path.dirname(os.path.abspath(__file__))
ORC_SRC = os.path.join(_HERE, "orc_locmatch.cpp")
ORC_LIB = os.path.join(_HERE, "_build", "liblimap_orc_locmatch.so")
_DEPS = [ORC_SRC, os.path.join(_HERE, "orc_triangulation.h"), os.path.join(_HERE, "orc_geom.h")]
REF_SRC = os.path.join(_HERE, "ref_locmatch.cpp")
REF_LIB = os.path.join(_HERE, "_ref", "liblimap_ref_locmatch.so")
_P = C.c_void_p
_lib = None
_ref_lib = None
DIST_FUNCS = {"Perpendicular": 0, "Midpoint": 1, "Midpoint_Perpendicular": 2}


def build(force=False):
    if force or _ev._stale(ORC_LIB, _DEPS):
        os.makedirs(os.path.dirname(ORC_LIB), exist_ok=True)
        _ev._run([_ev._CXX] + _ev._ORC_FLAGS + ["-shared", "-o", ORC_LIB, ORC_SRC])
    if _ref.can_build() and _ref.available() and (force or _ev._stale(REF_LIB, [REF_SRC, _ref.LIB_PATH])):
        _ev._run([_ev._CXX, "-O3", "-fopenmp", "-fPIC", "-shared", "-o", REF_LIB, REF_SRC,
                  "-L" + os.path.dirname(_ref.LIB_PATH), "-llimap_ref", "-Wl,-rpath,$ORIGIN"])
    return ORC_LIB


def ref_count(cams, item_cams, line_off, lines, item_lines, th):
    """Matched pairs per item by the reference's compiled compute_epipolar_IoU in a C loop on all host cores
    (oracle/_ref/liblimap_ref_locmatch.so, built only where the reference source tree exists)."""
    global _ref_lib
    if _ref_lib is None:
        build()
        if not os.path.exists(REF_LIB):
            raise RuntimeError(f"{REF_LIB} is missing (built only where the reference source tree exists)")
        _ref_lib = C.CDLL(REF_LIB)
        _ref_lib.ref_locmatch_count.restype = None
        _ref_lib.ref_locmatch_count.argtypes = [C.c_int64, _P, _P, _P, _P, _P, C.c_double, _P]
    i64 = lambda a: np.ascontiguousarray(a, np.int64)
    ic, lo, il = i64(item_cams), i64(line_off), i64(item_lines)
    cm, ln = _f64(cams, 12), _f64(lines, 4)
    out = np.zeros(len(ic), np.int64)
    _ref_lib.ref_locmatch_count(len(ic), _p(ic), _p(cm), _p(lo), _p(ln), _p(il), float(th), _p(out))
    return out


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(ORC_LIB)
        L.orc_locmatch_2to2.restype = C.c_int64
        L.orc_locmatch_2to2.argtypes = [C.c_int64, _P, _P, C.c_int64, _P, _P, C.c_double, _P]
        L.orc_locmatch_filter.restype = C.c_int64
        L.orc_locmatch_filter.argtypes = [C.c_int64, _P, _P, _P, _P, _P, C.c_double, _P]
        L.orc_locmatch_reproj_one.restype = C.c_int32
        L.orc_locmatch_reproj_one.argtypes = [_P, _P, C.c_int64, _P, _P, C.c_int, C.c_double, C.c_double, C.c_double]
        _lib = L
    return _lib


def _f64(a, n):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, n))


def _p(a):
    return a.ctypes.data_as(_P)


def cam_array(model, kvec, qvec, tvec):
    """The oracle's camera layout: model, fx, fy, cx, cy, qvec, tvec."""
    return np.ascontiguousarray(np.r_[model, kvec, qvec, tvec], np.float64)


def match_2to2(l1, cam1, l2, cam2, th):
    l1, l2 = _f64(l1, 4), _f64(l2, 4)
    out = np.zeros((len(l1) * len(l2) + 1, 2), np.int32)
    n = lib().orc_locmatch_2to2(len(l1), _p(l1), _p(cam1), len(l2), _p(l2), _p(cam2), float(th), _p(out))
    return [tuple(map(int, p)) for p in out[:n]]


def filter_2to2(pairs, l1, cam1, l2, cam2, th):
    l1, l2 = _f64(l1, 4), _f64(l2, 4)
    pr = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    out = np.zeros((len(pr) + 1, 2), np.int32)
    n = lib().orc_locmatch_filter(len(pr), _p(pr), _p(l1), _p(cam1), _p(l2), _p(cam2), float(th), _p(out))
    return [tuple(map(int, p)) for p in out[:n]]


def reproj_one(ref_seg, cam, cand, track_lines, dist_func, dist_thres=10.0, sine_thres=0.4, angle_scale=1.0):
    seg = _f64(ref_seg, 4)
    c = np.ascontiguousarray(np.asarray(cand, np.int32))
    tl = _f64(track_lines, 6)
    return int(lib().orc_locmatch_reproj_one(_p(seg), _p(cam), len(c), _p(c), _p(tl), DIST_FUNCS[dist_func],
                                             float(dist_thres), float(sine_thres), float(angle_scale)))


def reproj_filter(ref_lines, cam, all_pairs_2to3, track_lines, dist_func, dist_thres=10.0, sine_thres=0.4,
                  angle_scale=1.0):
    """reprojection_filter_matches_2to3 over a {query line: [track ids]} dict, in its key order."""
    ref_lines = _f64(ref_lines, 4)
    out = []
    for k, cand in all_pairs_2to3.items():
        best = reproj_one(ref_lines[k], cam, cand, track_lines, dist_func, dist_thres, sine_thres, angle_scale)
        if best >= 0:
            out.append((int(k), best))
    return out


def match_queries(queries, scenes, retrieval, line2track, track_lines, IoU_threshold, pairs_2to2=None,
                  epipolar_filter=False, reprojection_filter=None, dist_thres=2.0):
    """queries: {qid: (cam_array, lines[n][4])}; scenes: {db id: (cam_array, lines)}; retrieval {qid: [db ids]};
    line2track {db id: [track per line]}; pairs_2to2 {qid: {db id: pairs}} for the learned matchers. Returns
    {qid: [(query line, track id)]} in the runner's order."""
    out = {}
    for qid, (qcam, qlines) in queries.items():
        acc = defaultdict(list)
        for t in retrieval[qid]:
            tcam, tlines = scenes[t]
            if pairs_2to2 is None:
                p22 = match_2to2(qlines, qcam, tlines, tcam, IoU_threshold)
            elif epipolar_filter:
                p22 = filter_2to2(pairs_2to2[qid][t], qlines, qcam, tlines, tcam, IoU_threshold)
            else:
                p22 = [tuple(map(int, p[:2])) for p in pairs_2to2[qid][t]]
            for i, j in p22:  # match_line_2to3
                if line2track[t][j] != -1:
                    acc[i].append(int(line2track[t][j]))
        if reprojection_filter is not None:
            out[qid] = reproj_filter(qlines, qcam, acc, track_lines, reprojection_filter, dist_thres)
        else:
            out[qid] = [(x, y) for x in acc for y in acc[x]]
    return out
