"""Writes tests/golden/ref/loc_matching.npz: the reference's own line matching for the localization runner, on the seeded
cases of tests/locmatch_cases.py. Runs only where the reference source tree and oracle/_ref exist.

The reference's optimize/hybrid_localization/functions.py is read from the reference tree and executed unchanged, with
`limap.base` / `limap.triangulation` stand-ins whose geometry is the reference's compiled code in oracle/_ref
(compute_epipolar_IoU, CameraView::projection, Line2d::direction / length). The runner's 2to3 and grouping loop
(runners/hybrid_localization.py:284-346) is composed around it in the runner's order.

    python tests/golden/make_locmatch_golden.py
"""
import os
import sys
import types
from collections import defaultdict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import locmatch_cases as lc  # noqa: E402
from oracle import ref  # noqa: E402

FUNCTIONS = os.path.join(ref.REFERENCE_SRC, "limap", "optimize", "hybrid_localization", "functions.py")


def _p(a):
    return a.ctypes.data_as(ref._P)


def _stand_ins():
    L = ref.lib()
    f64 = lambda a: np.ascontiguousarray(a, np.float64)

    class Line2d:
        def __init__(self, s, e):
            self.start, self.end = f64(s), f64(e)

        def _seg(self):
            return f64(np.r_[self.start, self.end])

        def length(self):
            return L.ref_line2d_length(_p(self._seg()))

        def direction(self):
            out = np.zeros(2)
            L.ref_line2d_direction(_p(self._seg()), _p(out))
            return out

        def midpoint(self):
            return 0.5 * (self.start + self.end)

    class CameraPose:
        def __init__(self, q, t):
            self.q, self.t = f64(q), f64(t)

    class CameraView:
        def __init__(self, cam, pose):
            self.cam = f64(np.r_[cam[:5], pose.q, pose.t])

        def projection(self, X):
            out = np.zeros(2)
            L.ref_project_point(_p(self.cam), _p(f64(X)), _p(out))
            return out

    def compute_epipolar_IoU(l1, v1, l2, v2):
        return L.ref_compute_epipolar_IoU(_p(l1._seg()), _p(v1.cam), _p(l2._seg()), _p(v2.cam))

    base = types.ModuleType("limap.base")
    base.Line2d, base.CameraPose, base.CameraView = Line2d, CameraPose, CameraView
    tri = types.ModuleType("limap.triangulation")
    tri.compute_epipolar_IoU = compute_epipolar_IoU
    pkg = types.ModuleType("limap")
    pkg.base, pkg.triangulation = base, tri
    sys.modules.update({"limap": pkg, "limap.base": base, "limap.triangulation": tri})
    fn = types.ModuleType("reference_functions")
    exec(compile(open(FUNCTIONS).read(), FUNCTIONS, "exec"), fn.__dict__)
    return base, fn


class _Track:
    def __init__(self, base, row):
        self.line = types.SimpleNamespace(start=row[:3], end=row[3:])


def run_case(base, fn, case, out, tag):
    cams, lines = case["cams"], case["lines"]
    L2 = {k: [base.Line2d(s[:2], s[2:]) for s in v] for k, v in lines.items()}
    pose = lambda k: (cams[k][5:9], cams[k][9:12])  # poses as tuples: the functions build CameraPose themselves
    tracks = [_Track(base, r) for r in case["tracks"]]
    line2track = {k: [int(x) for x in v] for k, v in case["line2track"].items()}
    for q in case["q_ids"]:
        for d in case["retrieval"][q]:
            for th in lc.THRESHOLDS:
                p = fn.match_line_2to2_epipolarIoU(L2[q], L2[d], cams[q], pose(q), cams[d], pose(d), th)
                out[f"{tag}/m22/{q}/{d}/{th}"] = np.array(p, np.int32).reshape(-1, 2)
            p = fn.filter_line_2to2_epipolarIoU(case["pairs"][q][d], L2[q], L2[d], cams[q], pose(q), cams[d], pose(d),
                                                0.2)
            out[f"{tag}/f22/{q}/{d}"] = np.array(p, np.int32).reshape(-1, 2)
    # runners/hybrid_localization.py:284-346 for the epipolar matcher and the learned one (with and without the
    # epipolar filter), each without and with every reprojection filter
    for mode in ("epipolar", "learned", "learned_filter"):
        for rf in (None,) + lc.REPROJ_FUNCS:
            for q in case["q_ids"]:
                acc = defaultdict(list)
                for d in case["retrieval"][q]:
                    if mode == "epipolar":
                        p22 = fn.match_line_2to2_epipolarIoU(L2[q], L2[d], cams[q], pose(q), cams[d], pose(d), 0.2)
                    elif mode == "learned_filter":
                        p22 = fn.filter_line_2to2_epipolarIoU(case["pairs"][q][d], L2[q], L2[d], cams[q], pose(q),
                                                              cams[d], pose(d), 0.2)
                    else:
                        p22 = case["pairs"][q][d]
                    for qi, tr in fn.match_line_2to3(p22, line2track, d):
                        acc[qi].append(tr)
                if rf is not None:
                    view = base.CameraView(cams[q], base.CameraPose(*pose(q)))
                    res = fn.reprojection_filter_matches_2to3(L2[q], view, acc, tracks, dist_thres=2,
                                                              dist_func=fn.get_reprojection_dist_func(rf))
                else:
                    res = [(x, y) for x in acc for y in acc[x]]
                out[f"{tag}/run/{mode}/{rf}/{q}"] = np.array(res, np.int64).reshape(-1, 2)


def main():
    ref.build()
    base, fn = _stand_ins()
    out = {}
    for tag, kw in (("seed0", dict(seed=0)), ("seed1_planted", dict(seed=1, planted=True))):
        run_case(base, fn, lc.make_case(**kw), out, tag)
    path = os.path.join(HERE, "ref", "loc_matching.npz")
    np.savez_compressed(path, **out)
    print(path, len(out))


if __name__ == "__main__":
    main()
