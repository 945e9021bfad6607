"""ctypes wrapper of the CPU oracle (oracle/_build/liblimap_oracle.so). TEST INFRASTRUCTURE ONLY:
imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
Pinning status per component: oracle/orc_geom.h (pinned to oracle/_ref), orc_lm.h (solver loop unpinned), orc_vp.h and
orc_sfm.cpp (third-party algorithms restated: PARITY UNPINNED)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "liblimap_oracle.so")
_lib = None
_P = C.c_void_p


def usable_cpus():
    """CPUs this process may really use: affinity mask capped by the cgroup quota. OpenMP's default
    (every core the machine has) oversubscribes badly inside a CPU-limited container."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            q, p = f.read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:
        pass
    return max(1, n)


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cpp", ".h"))]
    if force or not os.path.exists(LIB_PATH) or any(
            os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs):
        env = dict(os.environ)
        env.pop("CXX", None)
        subprocess.run(["make", "-C", _HERE, "-B" if force else "-s"], check=True, env=env,
                       stdout=subprocess.DEVNULL)
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        L = C.CDLL(LIB_PATH)
        L.orc_last_error.restype = C.c_char_p
        L.orc_tri_create.restype = _P
        L.orc_tri_create.argtypes = [_P]
        L.orc_tri_destroy.argtypes = [_P]
        L.orc_tri_set_node_parallel.argtypes = [_P, C.c_int]
        L.orc_tri_init.argtypes = [_P, C.c_int] + [_P] * 7
        L.orc_tri_set_ranges.argtypes = [_P, _P, _P]
        L.orc_tri_unset_ranges.argtypes = [_P]
        L.orc_tri_triangulate_image.argtypes = [_P, C.c_int, C.c_int, _P, _P, _P]
        L.orc_tri_triangulate_image_exhaustive.argtypes = [_P, C.c_int, C.c_int, _P]
        L.orc_tri_rows_tested.restype = C.c_longlong
        L.orc_tri_rows_tested.argtypes = [_P]
        L.orc_tri_get_best.argtypes = [_P, C.c_int, _P, _P, _P]
        L.orc_tri_get_valid_edges.restype = C.c_longlong
        L.orc_tri_get_valid_edges.argtypes = [_P, C.c_int, _P, _P]
        L.orc_tri_get_tris_node.argtypes = [_P, C.c_int, C.c_int, C.c_int, _P, _P]
        L.orc_tri_compute_tracks.argtypes = [_P, _P]
        L.orc_tri_get_tracks.argtypes = [_P] * 7
        L.orc_tri_get_graph.restype = C.c_longlong
        L.orc_tri_get_graph.argtypes = [_P] * 5
        L.orc_line2d_length.restype = C.c_double
        L.orc_line2d_length.argtypes = [_P]
        L.orc_line2d_direction.argtypes = [_P, _P]
        L.orc_compute_epipolar_IoU.restype = C.c_double
        L.orc_compute_epipolar_IoU.argtypes = [_P] * 4
        L.orc_triangulate_line.argtypes = [_P, _P, _P, _P, C.c_int, _P]
        L.orc_project_point.argtypes = [_P, _P, _P]
        L.orc_score_3d.restype = C.c_double
        L.orc_score_3d.argtypes = [_P, _P, _P]
        L.orc_score_2d.restype = C.c_double
        L.orc_score_2d.argtypes = [_P, _P, _P]
        L.orc_set_num_threads.argtypes = [C.c_int]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(_P)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


class OracleTri:
    """fp64 CPU restatement of GlobalLineTriangulator, same array-level interface as
    limap_b200.engine.TriEngine."""

    _PREFIX = "orc_"

    @staticmethod
    def _library():
        return lib()

    def _c(self, name):
        return getattr(self._library(), self._PREFIX + name)

    def __init__(self, cfg=None, threads=None, node_parallel=False):
        """node_parallel=False keeps the reference's OpenMP schedule (inside one node); True moves the OpenMP loop out to
        the 2D lines of the image -- same results, the schedule a throughput-tuned CPU implementation would use."""
        from limap_b200.config import make_tri_config
        self.cfg = make_tri_config(cfg) if not hasattr(cfg, "_fields_") else cfg
        # parity runs do not need many threads; the reference's OpenMP regions are tiny (one node each)
        self._c("set_num_threads")(int(threads) if threads else min(8, usable_cpus()))
        self._h = self._c("tri_create")(C.byref(self.cfg))
        if not self._h:
            raise RuntimeError(self._c("last_error")().decode())
        if node_parallel:
            self._c("tri_set_node_parallel")(self._h, 1)

    def __del__(self):
        if getattr(self, "_h", None):
            self._c("tri_destroy")(self._h)
            self._h = None

    def upload_scene(self, img_ids, model_ids, kvec, qvec, tvec, line_off, segs):
        self.img_ids = np.ascontiguousarray(img_ids, np.int32)
        self.line_off = np.ascontiguousarray(line_off, np.int64)
        self._view = {int(i): v for v, i in enumerate(self.img_ids)}
        a = [self.img_ids, np.ascontiguousarray(model_ids, np.int32), _f64(kvec), _f64(qvec), _f64(tvec),
             self.line_off, _f64(segs)]
        self._c("tri_init")(self._h, len(self.img_ids), *[_p(x) for x in a])

    def upload(self, scene):
        self.upload_scene(scene.img_ids, scene.model_ids, scene.kvec, scene.qvec, scene.tvec,
                          scene.line_off, scene.segs)

    def n_lines(self, img_id):
        v = self._view[int(img_id)]
        return int(self.line_off[v + 1] - self.line_off[v])

    def set_ranges(self, lo, hi):
        self._c("tri_set_ranges")(self._h, _p(_f64(lo)), _p(_f64(hi)))

    def set_vps(self, vpresults, img_ids=None, line_off=None):
        """InitVPResults: {img_id: object with .labels and .vps}."""
        ids = [int(i) for i in self.img_ids if int(i) in vpresults]
        label_off, vp_off, labels, vps = [0], [0], [], []
        for i in ids:
            r = vpresults[i]
            lab = np.asarray(r.labels, np.int32).reshape(-1)
            v = np.asarray(r.vps, np.float64).reshape(-1, 3)
            labels.append(lab)
            vps.append(v)
            label_off.append(label_off[-1] + len(lab))
            vp_off.append(vp_off[-1] + len(v))
        labels = np.ascontiguousarray(np.concatenate(labels) if labels else np.zeros(0, np.int32))
        vps = np.ascontiguousarray(np.concatenate(vps) if vps else np.zeros((0, 3)))
        self._c("tri_set_vps").argtypes = [_P, C.c_int, _P, _P, _P, _P, _P]
        self._c("tri_set_vps")(self._h, len(ids), _p(np.asarray(ids, np.int32)), _p(np.asarray(label_off, np.int64)),
                          _p(labels), _p(np.asarray(vp_off, np.int64)), _p(vps))

    def add_image_matches(self, img_id, ng_ids, row_off, pairs):
        ng_ids = np.ascontiguousarray(ng_ids, np.int32)
        row_off = np.ascontiguousarray(row_off, np.int64)
        pairs = np.ascontiguousarray(pairs, np.int32)
        rc = self._c("tri_triangulate_image")(self._h, int(img_id), len(ng_ids), _p(ng_ids), _p(row_off),
                                             _p(pairs))
        if rc:
            raise RuntimeError(self._c("last_error")().decode())

    def add_image_exhaustive(self, img_id, neighbors):
        ng = np.ascontiguousarray(neighbors, np.int32)
        rc = self._c("tri_triangulate_image_exhaustive")(self._h, int(img_id), len(ng), _p(ng))
        if rc:
            raise RuntimeError(self._c("last_error")().decode())

    def rows_tested(self):
        return int(self._c("tri_rows_tested")(self._h))

    def get_best(self, img_id):
        L = self.n_lines(img_id)
        line = np.zeros((L, 10))
        ng = np.zeros((L, 2), np.int32)
        nc = np.zeros(L, np.int32)
        self._c("tri_get_best")(self._h, int(img_id), _p(line), _p(ng), _p(nc))
        return line, ng, nc

    def get_valid_edges(self, img_id):
        L = self.n_lines(img_id)
        off = np.zeros(L + 1, np.int64)
        n = self._c("tri_get_valid_edges")(self._h, int(img_id), _p(off), None)
        edges = np.zeros((max(n, 1), 2), np.int32)
        self._c("tri_get_valid_edges")(self._h, int(img_id), _p(off), _p(edges))
        return off, edges[:n]

    def get_cands_node(self, img_id, line_id, cap=4096):
        line = np.zeros((cap, 10))
        ng = np.zeros((cap, 2), np.int32)
        n = self._c("tri_get_tris_node")(self._h, int(img_id), int(line_id), cap, _p(line), _p(ng))
        if n > cap:
            return self.get_cands_node(img_id, line_id, n)
        return line[:n], ng[:n]

    def build_tracks(self):
        tot = C.c_int64(0)
        T = self._c("tri_compute_tracks")(self._h, C.byref(tot))
        n = tot.value
        track_off = np.zeros(T + 1, np.int64)
        img = np.zeros(max(n, 1), np.int32)
        line = np.zeros(max(n, 1), np.int32)
        node = np.zeros(max(n, 1), np.int32)
        l3d = np.zeros((max(n, 1), 10))
        tl = np.zeros((max(T, 1), 7))
        self._c("tri_get_tracks")(self._h, _p(track_off), _p(img), _p(line), _p(node), _p(l3d), _p(tl))
        return dict(track_off=track_off, img_ids=img[:n], line_ids=line[:n], node_ids=node[:n],
                    line3d=l3d[:n], track_line=tl[:T])


def cam_array(model, kvec, qvec, tvec):
    return _f64([model, *kvec, *qvec, *tvec])


class LMCfg(C.Structure):
    _fields_ = [("geometric_alpha", C.c_double), ("cauchy_scale", C.c_double),
                ("max_num_iterations", C.c_int32), ("min_num_images", C.c_int32),
                ("num_outliers", C.c_int32), ("mode", C.c_int32), ("parallel_tracks", C.c_int32),
                ("max_num_consecutive_invalid_steps", C.c_int32), ("vp_multiplier", C.c_double)]


def refine_tracks(ts, max_num_iterations=100, min_num_images=4, num_outliers=2, geometric_alpha=10.0,
                  cauchy_scale=0.25, mode=0, parallel_tracks=True, threads=None, sup_vp=None, vp_multiplier=1.0,
                  max_num_consecutive_invalid_steps=10):
    """CPU restatement of solve_line_bundle_adjustment / per-track RefinementEngine on a TrackSet. `term` holds each
    track's exit (LMSummary::termination: 0 not solved, 1 iteration cap, 2 radius, 3 zero gradient, 4 consecutive
    invalid steps, 5 zero step, 6 zero cost change)."""
    L = lib()
    L.orc_set_num_threads(int(threads) if threads else min(8, usable_cpus()))
    L.orc_refine_tracks.argtypes = [C.c_int] + [_P] * 15
    T = ts.n_tracks
    cfg = LMCfg(geometric_alpha, cauchy_scale, max_num_iterations, min_num_images, num_outliers, mode,
                int(parallel_tracks), int(max_num_consecutive_invalid_steps), float(vp_multiplier))
    out_line = np.zeros((T, 6))
    out_min = np.zeros((T, 6))
    iters = np.zeros((T, 2), np.int32)
    cost = np.zeros((T, 2))
    term = np.zeros(T, np.int32)
    a = [np.ascontiguousarray(ts.sup_off, np.int64), _f64(ts.segs), _f64(ts.kvec), _f64(ts.qvec), _f64(ts.tvec),
         np.ascontiguousarray(ts.img_ids, np.int32), _f64(ts.line3d), _f64(ts.line_init),
         None if sup_vp is None else _f64(sup_vp)]
    L.orc_refine_tracks(T, *[_p(x) for x in a], C.byref(cfg), _p(out_line), _p(out_min), _p(iters), _p(cost),
                        _p(term))
    return dict(line=out_line, minimal=out_min, iters=iters, cost=cost, term=term)


class VPCfg(C.Structure):
    _fields_ = [("min_length", C.c_double), ("inlier_threshold", C.c_double), ("th_perp_supports", C.c_double),
                ("min_num_supports", C.c_int32), ("n_models", C.c_int32), ("seed", C.c_uint64)]


def detect_vps(line_off, segs, min_length=40.0, inlier_threshold=1.0, min_num_supports=5, th_perp_supports=3.0,
               n_models=5000, seed=0, threads=None, image_index=None):
    """CPU restatement of JLinkage::AssociateVPs over a batch of images (flat segments)."""
    L = lib()
    L.orc_set_num_threads(int(threads) if threads else min(8, usable_cpus()))
    L.orc_vp_detect_indexed.restype = C.c_longlong
    L.orc_vp_detect_indexed.argtypes = [C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_longlong]
    idx = None if image_index is None else np.ascontiguousarray(image_index, np.int64)
    line_off = np.ascontiguousarray(line_off, np.int64)
    segs = _f64(segs)
    n = len(line_off) - 1
    cfg = VPCfg(min_length, inlier_threshold, th_perp_supports, min_num_supports, n_models, seed)
    labels = np.full(int(line_off[-1]), -1, np.int32)
    vp_off = np.zeros(n + 1, np.int64)
    cap = 64 * max(n, 1)
    vps = np.zeros((cap, 3))
    tot = L.orc_vp_detect_indexed(n, _p(line_off), _p(segs), C.byref(cfg), None if idx is None else _p(idx), _p(labels),
                                  _p(vp_off), _p(vps), cap)
    if tot > cap:  # more VPs than the first guess: run again with room for all of them
        vps = np.zeros((tot, 3))
        L.orc_vp_detect_indexed(n, _p(line_off), _p(segs), C.byref(cfg), None if idx is None else _p(idx), _p(labels),
                                _p(vp_off), _p(vps), tot)
    return labels, vp_off, vps[:tot]


# ---- track filters + remerge (orc_merging.cpp) -----------------------------------------------------------
class OrcLinkerCfg(C.Structure):  # orc::LinkerConfig
    _fields_ = [(n, C.c_double) for n in ("score_th", "th_angle", "th_overlap", "th_smartoverlap", "th_smartangle",
                                           "th_perp", "th_innerseg", "th_scaleinv")] + \
               [(n, C.c_int) for n in ("use_angle", "use_overlap", "use_smartangle", "use_perp", "use_innerseg",
                                       "use_scaleinv")]


def track_support_flags(model_ids, kvec, qvec, tvec, sup_off, sup_view, segs, track_line, th_angular_2d=8.0,
                        th_perp_2d=5.0, th_sv_angular_3d=75.0, th_overlap=0.5, threads=None):
    """CheckReprojection / CheckSensitivity / overlap bits per supporting line (merging_utils.cc:27-155)."""
    L = lib()
    L.orc_set_num_threads(int(threads) if threads else min(8, usable_cpus()))
    L.orc_track_support_flags.argtypes = [C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P] + [C.c_double] * 4 + [_P]
    sup_off = np.ascontiguousarray(sup_off, np.int64)
    sup_view = np.ascontiguousarray(sup_view, np.int32)
    model_ids = None if model_ids is None else np.ascontiguousarray(model_ids, np.int32)
    kvec, qvec, tvec, segs, track_line = map(_f64, (kvec, qvec, tvec, segs, track_line))
    flags = np.zeros(int(sup_off[-1]), np.uint8)
    L.orc_track_support_flags(len(kvec), _p(model_ids), _p(kvec), _p(qvec), _p(tvec), len(sup_off) - 1, _p(sup_off),
                              _p(sup_view), _p(segs), _p(track_line), th_angular_2d, th_perp_2d, th_sv_angular_3d,
                              th_overlap, _p(flags))
    return flags


def aggregate_lines(off, lines, scores, num_outliers):
    L = lib()
    L.orc_aggregate_lines.argtypes = [C.c_int64, _P, _P, _P, C.c_int32, _P]
    off = np.ascontiguousarray(off, np.int64)
    lines, scores = _f64(lines), _f64(scores)
    out = np.zeros((len(off) - 1, 7))
    L.orc_aggregate_lines(len(off) - 1, _p(off), _p(lines), _p(scores), int(num_outliers), _p(out))
    return out


def remerge_labels(track_line, active, linker, threads=None):
    """One RemergeLineTracks pass up to the group labels. linker: dict of LineLinker3dConfig fields."""
    L = lib()
    L.orc_set_num_threads(int(threads) if threads else min(8, usable_cpus()))
    L.orc_remerge_labels.restype = C.c_int64
    L.orc_remerge_labels.argtypes = [C.c_int64, _P, _P, _P, _P, _P]
    d = dict(score_th=0.5, th_angle=10.0, th_overlap=0.01, th_smartoverlap=0.1, th_smartangle=1.0, th_perp=0.02,
             th_innerseg=0.02, th_scaleinv=0.01, use_angle=1, use_overlap=1, use_smartangle=1, use_perp=0,
             use_innerseg=1, use_scaleinv=0)  # line_linker.h:85-111
    d.update({k: v for k, v in linker.items() if k in d})
    cfg = OrcLinkerCfg(*[float(d[n]) if t is C.c_double else int(bool(d[n])) for n, t in OrcLinkerCfg._fields_])
    track_line = _f64(track_line)
    active = np.ascontiguousarray(active, np.uint8)
    labels = np.zeros(len(track_line), np.int32)
    ne = C.c_int64(0)
    ng = L.orc_remerge_labels(len(track_line), _p(track_line), _p(active), C.byref(cfg), _p(labels), C.byref(ne))
    return labels, int(ng), int(ne.value)


# ---- visual neighbours / robust ranges (orc_sfm.cpp) ---------------------------------------------------------------
def rank_neighbors(centres, xyz, track_off, track_img, num_images, min_triangulation_angle=1.0, mode=0):
    L = lib()
    L.orc_rank_neighbors.argtypes = [C.c_int, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_double, C.c_int, _P, _P]
    centres, xyz = _f64(centres), _f64(xyz)
    track_off = np.ascontiguousarray(track_off, np.int64)
    track_img = np.ascontiguousarray(track_img, np.int32)
    n = len(centres)
    out = np.full((n, int(num_images)), -1, np.int32)
    cnt = np.zeros(n, np.int32)
    L.orc_rank_neighbors(n, _p(centres), len(xyz), _p(xyz), _p(track_off), _p(track_img), int(num_images),
                         float(min_triangulation_angle), int(mode), _p(out), _p(cnt))
    return out, cnt


def robust_ranges(xyz, q_lo, q_hi, kstretch):
    L = lib()
    L.orc_robust_ranges.argtypes = [C.c_int64, _P, C.c_double, C.c_double, C.c_double, _P]
    xyz = _f64(xyz)
    out = np.zeros(6)
    L.orc_robust_ranges(len(xyz), _p(xyz), float(q_lo), float(q_hi), float(kstretch), _p(out))
    return out[:3].copy(), out[3:].copy()
