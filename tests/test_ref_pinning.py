"""Pins the oracle (oracle/*.h, the restatement every GPU parity test compares against) to the REFERENCE'S OWN
COMPILED CODE. The reference's outputs come from its hot-path sources built unchanged (oracle/Makefile target `ref`;
Eigen / COLMAP / glog / PoseLib come from the header shims in oracle/ref_shim/) run on the seeded inputs built below;
they are stored in tests/golden/ref/ (tests/golden/make_ref_golden.py regenerates them where the reference source tree
is available), so the pinning runs anywhere. Where an input set is large, the reference's outputs are stored for a fixed
sample of it (every k-th item) and the oracle still runs on the whole set.

  * whole pipeline: limap::triangulation::GlobalLineTriangulator (Init -> TriangulateImage -> ComputeLineTracks) against
    OracleTri on seeded scenes and the configuration families the GPU tests use (the GPU configuration matrix also moves
    single thresholds -- score_th, min_length_2d, the phase-A angle and sensitivity cut-offs -- around the families
    pinned here) -- candidate lists, scores, valid connections, best candidates, graph-ordered track membership
    bit-exact, coordinates to 1e-9;
  * decision boundaries (tests/boundary_scenes.py): 2D lengths equal to min_length_2d, 3D angles and scale-invariant
    distances planted at threshold * (1 -+ delta) for delta 1e-6, 1e-9, 1e-11;
  * function level on 2e4..1e5 random inputs each: compute_epipolar_IoU, triangulate_line (plane pair and endpoints),
    triangulate_line_with_direction, LineLinker2d/3d::compute_score, Line3d::sensitivity / computeUncertainty,
    CameraView::projection / ray_direction, Aggregator::aggregate_line3d_list, MinimalInfiniteLine3d,
    GetLineSegmentFromInfiniteLine3d, CheckReprojection / CheckSensitivity / overlap, RemergeLineTracks."""
import ctypes as C
import os

import numpy as np
import pytest

from limap_b200.config import DEFAULT_YAML_TRIANGULATION
from limap_b200.synth import make_scene

from parity_utils import compare_nodes, compare_tracks

from oracle import oracle as orc
from oracle import ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")
TOL = 1e-9


def _gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _feed(t, sc, exhaustive=False, ranges=True, vp=None):
    t.upload(sc)
    if ranges:
        t.set_ranges(*sc.ranges)
    if vp is not None:
        t.set_vps(vp, sc.img_ids, sc.line_off)
    for i in sc.img_ids:
        if exhaustive:
            t.add_image_exhaustive(int(i), sc.neighbors[int(i)])
        else:
            t.add_image_matches(int(i), *sc.flat_matches(int(i)))
    return t


def _cfg(**kw):
    c = dict(DEFAULT_YAML_TRIANGULATION, debug_mode=True)
    c.update(kw)
    return c


def _vps(sc, seed):
    rng = np.random.default_rng(seed)
    out = {}

    class R:
        pass
    for v, i in enumerate(sc.img_ids):
        L = int(sc.line_off[v + 1] - sc.line_off[v])
        q = rng.normal(size=(3, 3))
        q[:, :2] *= 1000.0
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        lab = rng.integers(0, 3, L)
        lab[rng.random(L) < 0.4] = -1
        r = R()
        r.labels, r.vps = lab.astype(np.int32), q
        out[int(i)] = r
    return out


CASES = {
    "default_yaml": (dict(V=8, L=120, N=5, K=6, seed=201), {}, {}),
    "cpp_defaults_outer_edge_filter": (dict(V=8, L=120, N=5, K=5, seed=202), None, {}),
    "asset_units_gaps_shuffled": (dict(V=8, L=100, N=5, K=4, seed=203, scale=100.0, id_stride=7, shuffle_rows=True), {}, {}),
    "mixed_cameras": (dict(V=8, L=100, N=5, K=5, seed=204, camera_mix=True), {}, {}),
    "endpoints_halfpix_no_ranges": (dict(V=6, L=80, N=4, K=4, seed=205), dict(use_endpoints_triangulation=True, add_halfpix=True), dict(ranges=False)),
    "max_valid_conns": (dict(V=6, L=60, N=5, K=8, seed=206), dict(max_valid_conns=3), {}),
    "exhaustive": (dict(V=5, L=40, N=3, K=2, seed=207), {}, dict(exhaustive=True)),
    "vp_proposals": (dict(V=6, L=60, N=4, K=3, seed=208), dict(use_vp=True), dict(vp=9)),
    "innerseg_2d_linker": (dict(V=6, L=80, N=4, K=4, seed=209), dict(linker2d_config=dict(use_innerseg=True, th_innerseg=3.0)), {}),
    # sub-tests of both linkers switched off or moved: no perpendicular / smart-angle test, 2D and 3D angles above the
    # 14.4775 deg switch of the asin^2 series, other score thresholds and scale invariance
    "linker_flag_variants": (dict(V=7, L=80, N=4, K=4, seed=210), dict(
        linker2d_config=dict(DEFAULT_YAML_TRIANGULATION["linker2d_config"], use_perp=False, use_smartangle=False,
                             th_angle=20.0, score_th=0.3),
        linker3d_config=dict(DEFAULT_YAML_TRIANGULATION["linker3d_config"], th_angle=20.0, th_scaleinv=0.05,
                             score_th=0.8)), {}),
    "linker_no_overlap_no_angle": (dict(V=7, L=80, N=4, K=4, seed=211), dict(
        linker2d_config=dict(DEFAULT_YAML_TRIANGULATION["linker2d_config"], use_overlap=False, use_angle=False),
        linker3d_config=dict(DEFAULT_YAML_TRIANGULATION["linker3d_config"], th_angle=90.0, th_scaleinv=0.002)), {}),
    # the gates of phase A at their off values, and the rank of every candidate deciding the valid connections
    "phase_a_gates_off": (dict(V=7, L=80, N=4, K=4, seed=212), dict(
        line_tri_angle_threshold=0.0, sensitivity_threshold=90.0, IoU_threshold=0.0, min_length_2d=-1.0), {}),
    "rank_all_valid": (dict(V=6, L=60, N=5, K=6, seed=213), dict(fullscore_th=0.0, max_valid_conns=2), {}),
}


def _pipeline_case(name):
    kw, over, run = CASES[name]
    sc = make_scene(**kw)
    cfg = dict(debug_mode=True) if over is None else _cfg(**over)
    run = dict(run)
    if "vp" in run:
        run["vp"] = _vps(sc, run["vp"])
    return sc, cfg, run


CAND_LINES_EVERY = 2  # candidate ids are stored for every node, candidate coordinates for every 2nd node


def _record_tri(t, sc, every=CAND_LINES_EVERY):
    """Everything compare_nodes / compare_tracks read from a triangulator, as flat arrays (candidate coordinates of
    every `every`-th node)."""
    best, ng, nc, ecnt, edges, ccnt, cline, cng = [], [], [], [], [], [], [], []
    for i in sc.img_ids:
        l, g, c = t.get_best(int(i))
        best.append(l); ng.append(g); nc.append(c)
        off, e = t.get_valid_edges(int(i))
        ecnt.append(np.diff(off)); edges.append(e.reshape(-1, 2))
        for k in range(len(c)):
            cl, cg = t.get_cands_node(int(i), k)
            ccnt.append(len(cl)); cng.append(cg.reshape(-1, 2))
            if (len(ccnt) - 1) % every == 0:
                cline.append(cl.reshape(-1, 10))
    out = dict(best_line=np.concatenate(best), best_ng=np.concatenate(ng), best_nc=np.concatenate(nc),
               edge_cnt=np.concatenate(ecnt), edges=np.concatenate(edges).astype(np.int32),
               cand_cnt=np.asarray(ccnt, np.int64), cand_line=np.concatenate(cline), cand_ng=np.concatenate(cng).astype(np.int32))
    out.update({"tracks_" + k: v for k, v in t.build_tracks().items()})
    return out


class _StoredTri:
    """The reference triangulator's answers, replayed from _record_tri's arrays."""

    def __init__(self, z, sc, every=CAND_LINES_EVERY):
        self.z, self.every = z, every
        n = np.diff(sc.line_off)
        self.first = {int(i): int(o) for i, o in zip(sc.img_ids, np.concatenate([[0], np.cumsum(n)]))}
        self.n = {int(i): int(k) for i, k in zip(sc.img_ids, n)}
        self.eoff = np.concatenate([[0], np.cumsum(z["edge_cnt"])]).astype(np.int64)
        self.coff = np.concatenate([[0], np.cumsum(z["cand_cnt"])]).astype(np.int64)
        self.loff = np.concatenate([[0], np.cumsum(z["cand_cnt"][::every])]).astype(np.int64)

    def get_best(self, i):
        a, b = self.first[i], self.first[i] + self.n[i]
        return self.z["best_line"][a:b], self.z["best_ng"][a:b], self.z["best_nc"][a:b]

    def get_valid_edges(self, i):
        a, b = self.first[i], self.first[i] + self.n[i]
        off = self.eoff[a:b + 1]
        return off - off[0], self.z["edges"][off[0]:off[-1]]

    def get_cands_node(self, i, l):
        """(candidate coordinates, or None where they are not stored; candidate ids)"""
        n = self.first[i] + l
        a, b = self.coff[n], self.coff[n + 1]
        lines = None
        if n % self.every == 0:
            k = n // self.every
            lines = self.z["cand_line"][self.loff[k]:self.loff[k + 1]]
        return lines, self.z["cand_ng"][a:b]

    def build_tracks(self):
        return {k[len("tracks_"):]: self.z[k] for k in self.z.files if k.startswith("tracks_")}


def _ref_pipeline(name):
    sc, cfg, run = _pipeline_case(name)
    return _record_tri(_feed(ref.RefTri(cfg, threads=1), sc, **run), sc)


def compare_stored(sc, r, o, endpoint_tol, score_tol=1e-9):
    """The stored reference `r` against a triangulator `o`: candidate lists in reference order, valid connections, best
    candidates and graph-ordered tracks bit-exact; coordinates within endpoint_tol, scores within score_tol."""
    import parity_utils
    old = parity_utils.ENDPOINT_TOL, parity_utils.SCORE_TOL
    parity_utils.ENDPOINT_TOL, parity_utils.SCORE_TOL = endpoint_tol, score_tol
    try:
        st = compare_nodes(sc, r, o)  # scores, valid connections, best candidates
        for i in sc.img_ids:  # candidate lists in reference order
            for l in range(r.n[int(i)]):
                cl, cng = r.get_cands_node(int(i), l)
                ol, ong = o.get_cands_node(int(i), l)
                assert np.array_equal(cng, ong), f"candidate list differs at node ({i},{l})"
                if cl is not None and len(ol):
                    assert np.abs(cl[:, :9] - ol[:, :9]).max() <= endpoint_tol
                    assert np.abs(cl[:, 9] - ol[:, 9]).max() <= score_tol
        tr = compare_tracks(r, o)
        assert tr["exact_order"]
    finally:
        parity_utils.ENDPOINT_TOL, parity_utils.SCORE_TOL = old
    return dict(st, tracks=tr["tracks"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_whole_pipeline_oracle_equals_compiled_reference(name, capfd):
    sc, cfg, run = _pipeline_case(name)
    o = _feed(orc.OracleTri(cfg, threads=1), sc, **run)
    r = _StoredTri(_gold("pipeline_" + name), sc)
    st = compare_stored(sc, r, o, 1e-7 * (100.0 if CASES[name][0].get("scale") else 1.0))
    assert st["candidates"] > 200 and st["valid_edges"] > 20 and st["tracks"] > 5


def _ref_boundary_min_length():
    from boundary_scenes import min_length_cfg, min_length_scene
    sc, _ = min_length_scene()
    return _record_tri(_feed(ref.RefTri(min_length_cfg(), threads=1), sc), sc, every=1)


def _ref_boundary_3d(name):
    from boundary_scenes import boundary_3d_cfg, boundary_3d_scene
    sc, _ = boundary_3d_scene(name)
    return _record_tri(_feed(ref.RefTri(boundary_3d_cfg(name), threads=1), sc), sc, every=1)


@pytest.mark.parametrize("name", ["angle_10", "angle_14.4775", "angle_20", "scaleinv"])
def test_boundary_3d_oracle_equals_compiled_reference(name):
    """3D angle and scale-invariant endpoint distance planted at threshold * (1 -+ delta), delta 1e-6 / 1e-9 / 1e-11,
    at depths ~1 and ~1e3 and at asset-unit coordinates (tests/boundary_scenes.py): the reference's compiled code scores
    the +delta pairs 0 and the -delta pairs >= score_th, and the oracle reproduces it."""
    from boundary_scenes import boundary_3d_cfg, check_planted, checked_boundary_3d_scene
    sc, planted = checked_boundary_3d_scene(name)
    o = _feed(orc.OracleTri(boundary_3d_cfg(name), threads=1), sc)
    r = _StoredTri(_gold("boundary_3d_" + name), sc, every=1)
    check_planted(r, sc, planted)
    compare_stored(sc, r, o, 1e-7)


def test_boundary_min_length_oracle_equals_compiled_reference():
    """2D segments of length exactly min_length_2d, as source lines and as matched lines: rejected by `<=`."""
    from boundary_scenes import min_length_cfg, min_length_scene
    sc, planted = min_length_scene()
    o = _feed(orc.OracleTri(min_length_cfg(), threads=1), sc)
    r = _StoredTri(_gold("boundary_min_length"), sc, every=1)
    st = compare_stored(sc, r, o, 1e-7)
    assert st["candidates"] > 1000
    nc = np.concatenate([r.get_best(int(i))[2] for i in sc.img_ids])
    assert (nc[planted] == 0).all()


# ---- function level --------------------------------------------------------------------------------------------
def _rand_cam(rng, mixed=True):
    f = rng.uniform(400, 900)
    model = int(rng.integers(0, 2)) if mixed else 0
    fy = f * rng.uniform(0.9, 1.1) if model == 1 else f
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return orc.cam_array(model, [f, fy, rng.uniform(300, 500), rng.uniform(200, 400)], q, rng.normal(size=3) * 3)


def _look_at_cam(rng, target, dist):
    from limap_b200.synth import _rot_to_quat
    c = target + dist * (lambda v: v / np.linalg.norm(v))(rng.normal(size=3))
    z = (target - c) / np.linalg.norm(target - c)
    x = np.cross(z, rng.normal(size=3))
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z], 0)
    f = rng.uniform(500, 800)
    return orc.cam_array(0, [f, f, 400, 300], _rot_to_quat(R), -R @ c), R, -R @ c, f


def _proj(R, t, f, X):
    Xc = R @ X + t
    return Xc[:2] / Xc[2] * f + np.array([400.0, 300.0])


def _pairs_of_views(rng, n):
    """(l1, cam1, l2, cam2): projections of a random 3D segment into two looking-at cameras, with pixel noise."""
    out = []
    for _ in range(n):
        X0, X1 = rng.uniform(-2, 2, 3), rng.uniform(-2, 2, 3)
        c1, R1, t1, f1 = _look_at_cam(rng, (X0 + X1) / 2, rng.uniform(6, 12))
        c2, R2, t2, f2 = _look_at_cam(rng, (X0 + X1) / 2, rng.uniform(6, 12))
        l1 = np.concatenate([_proj(R1, t1, f1, X0), _proj(R1, t1, f1, X1)]) + rng.normal(scale=1.0, size=4)
        l2 = np.concatenate([_proj(R2, t2, f2, X0), _proj(R2, t2, f2, X1)]) + rng.normal(scale=1.0, size=4)
        out.append((np.ascontiguousarray(l1), c1, np.ascontiguousarray(l2), c2))
    return out


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.all((np.abs(a - b) <= tol * (1 + np.abs(b))) | (np.isnan(a) & np.isnan(b)))


def _orc_lib():
    L = orc.lib()
    L.orc_triangulate_line_with_direction.argtypes = [C.c_void_p] * 6
    for f in ("orc_line3d_sensitivity", "orc_line3d_uncertainty"):
        getattr(L, f).restype = C.c_double
    L.orc_line3d_sensitivity.argtypes = [C.c_void_p] * 2
    L.orc_line3d_uncertainty.argtypes = [C.c_void_p, C.c_void_p, C.c_double]
    L.orc_ray_direction.argtypes = [C.c_void_p] * 3
    L.orc_minimal_from_line.argtypes = [C.c_void_p] * 2
    L.orc_infinite_from_minimal.argtypes = [C.c_void_p] * 3
    L.orc_segment_from_minimal.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    L.orc_geometric_residual.argtypes = [C.c_void_p] * 5 + [C.c_double] + [C.c_void_p] * 2
    L.orc_vp_residual.argtypes = [C.c_void_p] * 6
    return L


def _fn(lib, prefix, name):
    return getattr(lib, prefix + name)


TWO_VIEW_EVERY = 10


def _two_view_inputs():
    rng = np.random.default_rng(301)
    pairs = _pairs_of_views(rng, 20000)
    dirs = []
    for _ in pairs:
        d = rng.normal(size=3)
        dirs.append(d / np.linalg.norm(d))
    return pairs, dirs


def _two_view(lib, prefix, pairs, dirs, idx):
    """Per pair: [IoU, triangulate_line by planes (9), by endpoints (9), triangulate_line_with_direction (9)]."""
    p = orc._p
    out = np.zeros((len(idx), 28))
    for r, k in enumerate(idx):
        l1, c1, l2, c2 = pairs[k]
        out[r, 0] = _fn(lib, prefix, "compute_epipolar_IoU")(p(l1), p(c1), p(l2), p(c2))
        for by_end in (0, 1):
            o = np.zeros(9)
            _fn(lib, prefix, "triangulate_line")(p(l1), p(c1), p(l2), p(c2), by_end, p(o))
            out[r, 1 + 9 * by_end:10 + 9 * by_end] = o
        o = np.zeros(9)
        _fn(lib, prefix, "triangulate_line_with_direction")(p(l1), p(c1), p(l2), p(c2), p(dirs[k]), p(o))
        out[r, 19:28] = o
    return out


def _ref_two_view():
    pairs, dirs = _two_view_inputs()
    return dict(out=_two_view(ref.lib(), "ref_", pairs, dirs, range(0, len(pairs), TWO_VIEW_EVERY)))


def test_two_view_functions_on_random_pairs():
    pairs, dirs = _two_view_inputs()
    a = _two_view(_orc_lib(), "orc_", pairs, dirs, range(len(pairs)))
    b = _gold("two_view")["out"]
    s = a[::TWO_VIEW_EVERY]
    assert len(s) == len(b) and _close(s[:, 0], b[:, 0])
    for c in (1, 10, 19):
        assert np.array_equal(s[:, c + 8], b[:, c + 8])  # score: 1 on success, -1 on failure -- the same decision
        ok = b[:, c + 8] > 0
        assert _close(s[ok, c:c + 9], b[ok, c:c + 9], 1e-8)
    assert int((a[:, 9] > 0).sum() + (a[:, 18] > 0).sum()) > 20000


CAMERA_EVERY = 10


def _camera_inputs():
    rng = np.random.default_rng(302)
    out = []
    for _ in range(50000):
        cam = _rand_cam(rng)
        X = rng.normal(size=3) * 5
        px = rng.uniform(0, 800, 2)
        l3 = np.concatenate([rng.normal(size=6) * 3, rng.uniform(1, 9, 2), [0.1]])
        out.append((cam, X, px, l3))
    return out


def _camera(lib, prefix, items):
    """Per item: [projection (2), ray direction (3), Line3d sensitivity, uncertainty]."""
    p = orc._p
    out = np.zeros((len(items), 7))
    for r, (cam, X, px, l3) in enumerate(items):
        a, d = np.zeros(2), np.zeros(3)
        _fn(lib, prefix, "project_point")(p(cam), p(X), p(a))
        _fn(lib, prefix, "ray_direction")(p(cam), p(px), p(d))
        out[r, :2], out[r, 2:5] = a, d
        out[r, 5] = _fn(lib, prefix, "line3d_sensitivity")(p(l3), p(cam))
        out[r, 6] = _fn(lib, prefix, "line3d_uncertainty")(p(l3), p(cam), 2.0)
    return out


def _ref_camera():
    return dict(out=_camera(ref.lib(), "ref_", _camera_inputs()[::CAMERA_EVERY]))


def test_camera_and_line3d_functions():
    a = _camera(_orc_lib(), "orc_", _camera_inputs()[::CAMERA_EVERY])
    b = _gold("camera")["out"]
    assert len(a) == len(b)
    assert _close(a[:, :2], b[:, :2], 1e-9) and _close(a[:, 2:5], b[:, 2:5], 1e-12)
    assert _close(a[:, 5], b[:, 5], 1e-9) and _close(a[:, 6], b[:, 6], 1e-12)


LINKER_EVERY = 5


def _linker_inputs():
    rng = np.random.default_rng(303)
    variants = [dict(), dict(use_perp=1, use_innerseg=0), dict(use_scaleinv=1, use_overlap=0, use_innerseg=0),
                dict(use_innerseg=1, use_perp=1, use_scaleinv=1), dict(use_angle=0, use_smartangle=0)]
    out = []
    for k in range(100000):
        v = dict(variants[k % len(variants)])
        v.update(score_th=0.5, th_angle=rng.uniform(3, 12), th_overlap=rng.uniform(0.01, 0.2), th_smartoverlap=0.25,
                 th_smartangle=1.0, th_perp=rng.uniform(0.5, 3), th_innerseg=rng.uniform(0.5, 3), th_scaleinv=0.05)
        # 2D: a segment and a noisy, shifted, maybe flipped copy
        a = rng.uniform(0, 600, 4)
        d = (a[2:] - a[:2]) / np.linalg.norm(a[2:] - a[:2])
        s = rng.uniform(-0.5, 0.5, 2) * np.linalg.norm(a[2:] - a[:2])
        b = np.concatenate([a[:2] + d * s[0], a[2:] + d * s[1]]) + rng.normal(scale=rng.choice([0.3, 3.0]), size=4)
        if rng.random() < 0.5:
            b = b[[2, 3, 0, 1]]
        # 3D: start3, end3, depths2, uncertainty
        A = np.concatenate([rng.normal(size=6) * 2, rng.uniform(2, 9, 2), [rng.uniform(0.01, 0.2)]])
        dd = (A[3:6] - A[:3]) / np.linalg.norm(A[3:6] - A[:3])
        B = A.copy()
        B[:3] += dd * rng.uniform(-0.5, 0.5) + rng.normal(scale=rng.choice([0.005, 0.1]), size=3)
        B[3:6] += dd * rng.uniform(-0.5, 0.5) + rng.normal(scale=rng.choice([0.005, 0.1]), size=3)
        out.append((v, np.ascontiguousarray(a), np.ascontiguousarray(b), A, B))
    return out


def _linker(lib, prefix, items):
    """Per item: [LineLinker2d score, LineLinker3d score]."""
    p = orc._p
    out = np.zeros((len(items), 2))
    for r, (v, a, b, A, B) in enumerate(items):
        cfg = ref.linker_cfg(v)
        out[r, 0] = _fn(lib, prefix, "score_2d")(C.byref(cfg), p(a), p(b))
        out[r, 1] = _fn(lib, prefix, "score_3d")(C.byref(cfg), p(A), p(B))
    return out


def _ref_linker():
    return dict(out=_linker(ref.lib(), "ref_", _linker_inputs()[::LINKER_EVERY]))


def test_linker_scores_on_random_pairs():
    a = _linker(_orc_lib(), "orc_", _linker_inputs())
    b = _gold("linker")["out"]
    s = a[::LINKER_EVERY]
    assert len(s) == len(b) and _close(s, b, 1e-9)
    assert (a[:, 1] > 0).sum() > 10000


AGG_EVERY = 10


def _aggregate_inputs():
    rng = np.random.default_rng(304)
    # aggregate_line3d_list: groups of 1..12 noisy copies of a segment
    sizes = rng.integers(1, 13, 20000)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    base = rng.normal(size=(len(sizes), 6)) * 3
    lines = np.repeat(base, sizes, 0) + rng.normal(scale=0.02, size=(off[-1], 6))
    lines = np.concatenate([lines, rng.uniform(0.01, 0.3, (off[-1], 1))], 1)
    scores = rng.uniform(0, 5, off[-1])
    groups = []
    for no in (0, 2):
        ok = sizes * 2 - 1 - no >= no
        o2 = np.concatenate([[0], np.cumsum(sizes[ok])]).astype(np.int64)
        sel = np.repeat(ok, sizes)
        groups.append((o2, lines[sel], scores[sel], no))
    # MinimalInfiniteLine3d round trip + segment cut
    cuts = []
    for _ in range(20000):
        line = rng.normal(size=6) * 4
        n = int(rng.integers(2, 9))
        l3 = np.ascontiguousarray(np.tile(line, (n, 1)) + rng.normal(scale=0.05, size=(n, 6)))
        cuts.append((line, n, l3))
    return groups, cuts


def _minimal_chain(lib, prefix, line, n, l3, x=None):
    """[minimal (6), direction (3), moment (3), segment cut (6)]; the last three start from `x` if given (else the
    library's own minimal form)."""
    p = orc._p
    xm, d, m, s = np.zeros(6), np.zeros(3), np.zeros(3), np.zeros(6)
    _fn(lib, prefix, "minimal_from_line")(p(line), p(xm))
    x = xm if x is None else np.ascontiguousarray(x)
    _fn(lib, prefix, "infinite_from_minimal")(p(x), p(d), p(m))
    _fn(lib, prefix, "segment_from_minimal")(p(x), p(l3), n, 1, p(s))
    return np.concatenate([xm, d, m, s])


def _ref_aggregate():
    groups, cuts = _aggregate_inputs()
    out = {f"agg_{g[3]}": ref.aggregate_lines(*g)[::AGG_EVERY] for g in groups}
    out["minimal"] = np.stack([_minimal_chain(ref.lib(), "ref_", *c) for c in cuts[::AGG_EVERY]])
    return out


def test_aggregator_minimal_line_and_segment_cut():
    groups, cuts = _aggregate_inputs()
    z = _gold("aggregate")
    for g in groups:
        a, b = orc.aggregate_lines(*g)[::AGG_EVERY], z[f"agg_{g[3]}"]
        assert len(a) == len(b)
        d = np.minimum(np.abs(a[:, :6] - b[:, :6]).max(1), np.abs(a[:, :6] - b[:, [3, 4, 5, 0, 1, 2]]).max(1))
        assert d.max() < 1e-8 and np.abs(a[:, 6] - b[:, 6]).max() == 0
    L, ref_rows = _orc_lib(), z["minimal"]
    assert len(ref_rows) == len(cuts[::AGG_EVERY])
    for c, b in zip(cuts[::AGG_EVERY], ref_rows):
        xb = b[:6]
        a = _minimal_chain(L, "orc_", *c, x=xb)
        xa = a[:6]
        assert _close(xa, xb, 1e-9) or _close(np.concatenate([-xa[:4], xa[4:]]), xb, 1e-9)  # q == -q
        assert _close(a[6:9], b[6:9], 1e-12) and _close(a[9:12], b[9:12], 1e-10)
        assert _close(a[12:], b[12:], 1e-9)


RESIDUAL_EVERY = 10


def _residual_inputs():
    rng = np.random.default_rng(306)
    L = _orc_lib()
    p = orc._p
    out = []
    for it in range(20000):
        model = it & 1
        f = rng.uniform(300, 900)
        params = np.array([f, rng.uniform(300, 400), rng.uniform(200, 300)]) if model == 0 else \
            np.array([f, f * rng.uniform(0.9, 1.1), rng.uniform(300, 400), rng.uniform(200, 300)])
        kvec = np.array([params[0], params[0], params[1], params[2]]) if model == 0 else params.copy()
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        q *= rng.choice([1.0, 1.0, 0.7, 1.3])     # ceres::QuaternionToRotation normalises: not assumed unit
        t = rng.normal(size=3) * 2
        line = rng.normal(size=6) * 3
        x = np.zeros(6)
        L.orc_minimal_from_line(p(line), p(x))
        x += rng.normal(scale=0.01, size=6)       # off the manifold too: the functors are ambient
        seg = rng.uniform(0, 700, 4)
        alpha = float(rng.choice([10.0, 0.0, 3.0]))
        vp = rng.normal(size=3)
        vp /= np.linalg.norm(vp)
        out.append((model, x, seg, params, kvec, q, t, alpha, vp))
    return out


def _ref_residuals():
    R = ref.lib()
    p = orc._p
    rows = []
    for model, x, seg, params, kvec, q, t, alpha, vp in _residual_inputs()[::RESIDUAL_EVERY]:
        rb, jb, vb, vjb = np.zeros(2), np.zeros(12), np.zeros(1), np.zeros(6)
        R.ref_geometric_residual(model, p(x), p(seg), p(params), p(q), p(t), alpha, p(rb), p(jb))
        R.ref_vp_residual(model, p(x), p(vp), p(params), p(q), p(vb), p(vjb))
        rows.append(np.concatenate([rb, jb, vb, vjb]))
    return dict(out=np.stack(rows))


def test_refinement_residual_functors():
    """a14/a15: the reference's GeometricRefinementFunctor / VPConstraintsFunctor (cost_functions.h), compiled and
    evaluated on forward-mode jets, against the restatement the LM oracle is built from: residuals AND the 6-column
    Jacobians, PINHOLE and SIMPLE_PINHOLE, unnormalised quaternions included."""
    L = _orc_lib()
    p = orc._p
    gold = _gold("residuals")["out"]
    items = _residual_inputs()[::RESIDUAL_EVERY]
    assert len(items) == len(gold)
    worst = 0.0
    for it, ((model, x, seg, params, kvec, q, t, alpha, vp), g) in enumerate(zip(items, gold)):
        rb, jb, vb, vjb = g[:2], g[2:14], g[14:15], g[15:21]
        ra, ja = np.zeros(2), np.zeros(12)
        L.orc_geometric_residual(p(x), p(seg), p(kvec), p(q), p(t), alpha, p(ra), p(ja))
        s = max(1.0, np.abs(rb).max())
        assert np.abs(ra - rb).max() <= 1e-9 * s, (it, ra, rb)
        sj = max(1.0, np.abs(jb).max())
        assert np.abs(ja - jb).max() <= 1e-8 * sj, (it, ja, jb)
        worst = max(worst, np.abs(ja - jb).max() / sj)
        va, vja = np.zeros(1), np.zeros(6)
        L.orc_vp_residual(p(x), p(vp), p(kvec), p(q), p(va), p(vja))
        assert abs(va[0] - vb[0]) <= 1e-10, (it, va, vb)
        assert np.abs(vja - vjb).max() <= 1e-8 * max(1.0, np.abs(vjb).max()), (it, vja, vjb)
    assert worst < 1e-8


FILTER_KW = (dict(), dict(th_angular_2d=2.0, th_perp_2d=1.0, th_sv_angular_3d=60.0, th_overlap=0.9))
REMERGE_LK = dict(score_th=0.5, th_angle=5.0, th_overlap=0.001, th_smartoverlap=0.1, th_smartangle=1.0, th_perp=1.0,
                  th_innerseg=1.0)


def _filter_inputs():
    from limap_b200.synth import make_track_lines, make_tracks
    ts = make_tracks(T=400, S=10, V=40, seed=305, noise_px=2.0)
    views, first = np.unique(ts.img_ids, return_index=True)
    remap = np.zeros(int(views.max()) + 1, np.int32)
    remap[views] = np.arange(len(views), dtype=np.int32)
    rng = np.random.default_rng(305)
    tl = ts.gt + rng.normal(scale=0.03, size=ts.gt.shape)
    a = (None, ts.kvec[first], ts.qvec[first], ts.tvec[first], ts.sup_off, remap[ts.img_ids], ts.segs, tl)
    TL = make_track_lines(3000, dup_frac=0.4, seed=7, extent=8.0)
    acts = (np.ones(3000, np.uint8), (rng.random(3000) < 0.7).astype(np.uint8))
    return a, TL, acts


def _ref_filters():
    a, TL, acts = _filter_inputs()
    out = {f"flags_{k}": ref.track_support_flags(*a, **kw) for k, kw in enumerate(FILTER_KW)}
    for k, act in enumerate(acts):
        group, n_out = ref.remerge_groups(TL, act, REMERGE_LK)
        out[f"group_{k}"], out[f"n_groups_{k}"] = group, np.int64(n_out)
    return out


def test_track_filters_and_remerge():
    a, TL, acts = _filter_inputs()
    z = _gold("filters")
    for k, kw in enumerate(FILTER_KW):
        fa, fb = orc.track_support_flags(*a, **kw), z[f"flags_{k}"]
        assert np.array_equal(fa, fb) and 0 < (fa == 7).sum() < len(fa)
    for k, act in enumerate(acts):
        labels, ng, ne = orc.remerge_labels(TL, act, REMERGE_LK, threads=1)
        group, n_out = z[f"group_{k}"], int(z[f"n_groups_{k}"])
        # same partition: oracle labels <-> reference groups are in bijection
        pairs = set(zip(labels.tolist(), group.tolist()))
        assert len(pairs) == len(set(labels.tolist())) == len(set(group.tolist())) == ng == n_out
        assert ng < 3000


SFM_SEEDS = ((71, 30, 4000), (72, 12, 300))
SFM_RANKINGS = ((8, 1.0), (100, 0.5), (3, 6.0))
SFM_QUANTILES = ((0.05, 0.95, 1.25), (0.0, 0.999, 0.5), (0.25, 0.5, 2.0))


def _sfm_inputs(seed, V, n_pts):
    from limap_b200.base import CameraPose
    from limap_b200.synth import make_sfm_points
    sc = make_scene(V=V, L=10, N=3, K=1, seed=seed)
    _, xyz, off, img = make_sfm_points(sc, n_points=n_pts, seed=seed)
    R = np.stack([CameraPose(sc.qvec[v], sc.tvec[v]).R() for v in range(V)])
    return R, sc.tvec, xyz, off, img


def _ref_sfm():
    out = {}
    for seed, V, n_pts in SFM_SEEDS:
        R, T, xyz, off, img = _sfm_inputs(seed, V, n_pts)
        for mode in (0, 1, 2):
            for k, (n_nb, ang) in enumerate(SFM_RANKINGS):
                b, cb = ref.sfm_rank_neighbors(R, T, xyz, off, img, n_nb, min_triangulation_angle=ang, mode=mode)
                out[f"rank_{seed}_{mode}_{k}"], out[f"count_{seed}_{mode}_{k}"] = b, cb
        for k, q in enumerate(SFM_QUANTILES):
            out[f"lo_{seed}_{k}"], out[f"hi_{seed}_{k}"] = ref.sfm_robust_ranges(xyz, *q)
    return out


def test_sfm_model_neighbour_ranking_and_ranges():
    """f4: the reference's compiled pointsfm/sfm_model.cc (ranking loops, IoU / Dice formulas, sorts, ComputeRanges float
    arithmetic; COLMAP's mvs::Model statistics restated in oracle/ref_shim) against the oracle restatement the CUDA path
    is tested with. The reference orders equal scores with an UNSTABLE sort, the restatement keeps ascending image index:
    lists are compared exactly where the scores are distinct and by score sequence where they tie."""
    z = _gold("sfm")
    for seed, V, n_pts in SFM_SEEDS:
        R, T, xyz, off, img = _sfm_inputs(seed, V, n_pts)
        centres = ref.colmap_float_centres(R, T)
        xyz32 = xyz.astype(np.float32).astype(np.float64)  # Model::Point keeps float coordinates
        # scores per (i, j) for the tie analysis
        shared = np.zeros((V, V), np.int64)
        npts = np.bincount(img, minlength=V)
        for p in range(len(off) - 1):
            t = img[off[p]:off[p + 1]]
            shared[np.ix_(t, t)] += 1
        np.fill_diagonal(shared, 0)
        for mode in (0, 1, 2):
            union = npts[:, None] + npts[None, :] - shared
            score = (shared / np.maximum(union, 1), 2 * shared / np.maximum(union + shared, 1), shared.astype(float))[mode]
            for k, (n_nb, ang) in enumerate(SFM_RANKINGS):
                a, ca = orc.rank_neighbors(centres, xyz32, off, img, n_nb, min_triangulation_angle=ang, mode=mode)
                b, cb = z[f"rank_{seed}_{mode}_{k}"], z[f"count_{seed}_{mode}_{k}"]
                assert np.array_equal(ca, cb), (seed, mode, n_nb, ang)
                n_exact = 0
                for i in range(V):
                    la, lb = a[i, :ca[i]], b[i, :cb[i]]
                    sa, sb = score[i, la], score[i, lb]
                    assert np.array_equal(sa, sb), (seed, mode, n_nb, ang, i)  # same scores in the same order
                    row = score[i, shared[i] > 0]
                    if all((row == v).sum() == 1 for v in sa):  # no listed score ties with any other co-visible image
                        assert np.array_equal(la, lb), (seed, mode, n_nb, ang, i)
                        n_exact += 1
                assert n_exact > 0 or mode == 2
        for k, q in enumerate(SFM_QUANTILES):
            lo_a, hi_a = orc.robust_ranges(xyz, *q)
            lo_b, hi_b = z[f"lo_{seed}_{k}"], z[f"hi_{seed}_{k}"]
            assert np.array_equal(lo_a, lo_b) and np.array_equal(hi_a, hi_b), q  # float arithmetic, bit for bit


VP_KW = (dict(), dict(min_length=20.0, min_num_supports=8, th_perp_supports=1.0), dict(inlier_threshold=2.5))


def _vp_inputs():
    from limap_b200.synth import make_vp_images
    imgs = make_vp_images(6, 120, seed=81) + make_vp_images(2, 25, seed=82) + [np.zeros((0, 4))]
    return [np.ascontiguousarray(s, np.float64).reshape(-1, 4) for s in imgs]


def _ref_vp():
    out = {}
    for idx, segs in enumerate(_vp_inputs()):
        for k, kw in enumerate(VP_KW):
            out[f"labels_{idx}_{k}"], out[f"vps_{idx}_{k}"] = ref.vp_associate(segs, seed=7, image_index=idx, **kw)
    return out


def test_jlinkage_wrapper_filtering_renumbering_and_vp_fit():
    """a18: limap's own J-Linkage wrapper (vplib/JLinkage/JLinkage.cc + base_vp_detector.cc: min_length filter, the 2 x
    max(min_num_supports, 10) guard, cluster filtering with count_valid_supports_2d, label renumbering, VP = last right
    singular vector of the stacked line coordinates) compiled unchanged, over a JLinkage-library shim that forwards the
    sampling / clustering to the restated core -- against the restatement of the same wrapper in oracle/orc_vp.h.
    (The JLinkage library itself is an absent submodule: its core stays restated, DESIGN.md 6.)"""
    z = _gold("vp")
    n_vp_total = 0
    for idx, segs in enumerate(_vp_inputs()):
        for k, kw in enumerate(VP_KW):
            la, va = z[f"labels_{idx}_{k}"], z[f"vps_{idx}_{k}"]
            off = np.array([0, len(segs)], np.int64)
            lb, _, vb = orc.detect_vps(off, segs, n_models=5000, seed=7, image_index=[idx], threads=1, **kw)
            assert np.array_equal(la, lb), (idx, kw)
            assert len(va) == len(vb)
            for a, b in zip(va, vb):
                assert min(np.abs(a - b).max(), np.abs(a + b).max()) < 1e-7, (idx, kw, a, b)  # sign of a singular vector
            n_vp_total += len(va)
    assert n_vp_total >= 10


def _linetrack_inputs():
    rng = np.random.default_rng(91)
    cases = []
    for case in range(6):
        n = int(rng.integers(1, 9))
        line = rng.normal(size=6) * 3
        if case == 4:
            line[1] = np.nan  # written as 0 (linetrack.cc:137-152)
        img = rng.integers(0, 5, n).astype(np.int32)
        lid = rng.integers(0, 400, n).astype(np.int32)
        node = rng.integers(0, 10 ** 6, n).astype(np.int32)
        score = rng.uniform(0, 5, n)
        l2d = rng.uniform(0, 800, (n, 4))
        l3d = rng.normal(size=(n, 6)) * 2
        aux = case != 5  # case 5: a track without node ids / scores / 3D lines
        cases.append((n, line, img, lid, node, score, l2d, l3d, aux))
    return cases, rng.uniform(0, 800, (200, 4))


def _mirror_linetrack(c, path):
    import limap.base as base
    n, line, img, lid, node, score, l2d, l3d, aux = c
    t = base.LineTrack()
    t.line = base.Line3d(line[:3], line[3:])
    t.image_id_list, t.line_id_list = img.tolist(), lid.tolist()
    t.line2d_list = [base.Line2d(r[:2], r[2:]) for r in l2d]
    if aux:
        t.node_id_list, t.score_list = node.tolist(), score.tolist()
        t.line3d_list = [base.Line3d(r[:3], r[3:]) for r in l3d]
    t.Write(path)


def _ref_linetrack():
    import tempfile
    L = ref.lib()
    p = orc._p
    cases, segs = _linetrack_inputs()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for k, c in enumerate(cases):
            n, line, img, lid, node, score, l2d, l3d, aux = c
            f_ref = os.path.join(tmp, f"ref_{k}.txt").encode()
            L.ref_linetrack_write(f_ref, p(line), n, p(img), p(lid), p(node) if aux else None, p(score) if aux else None,
                                  p(l2d), p(l3d) if aux else None)
            out[f"file_{k}"] = np.frombuffer(open(f_ref, "rb").read(), np.uint8)
            # what the reference reads back from the mirror's file
            f_py = os.path.join(tmp, f"py_{k}.txt")
            _mirror_linetrack(c, f_py)
            o = dict(line=np.zeros(6), img=np.zeros(n, np.int32), lid=np.zeros(n, np.int32), node=np.zeros(n, np.int32),
                     score=np.zeros(n), l2d=np.zeros((n, 4)), l3d=np.zeros((n, 6)), ni=np.zeros(1, np.int32))
            got = L.ref_linetrack_read(f_py.encode(), n, *[p(o[x]) for x in ("line", "img", "lid", "node", "score", "l2d", "l3d", "ni")])
            out.update({f"read_{k}_{x}": v for x, v in o.items()})
            out[f"read_{k}_got"] = np.int64(got)
    w = np.zeros(200)
    L.ref_line_weights(200, p(segs), p(w))
    out["line_weights"] = w
    return out


def test_linetrack_file_format_and_line_weights(tmp_path):
    """a19: LineTrack::Write / LineTrack::Read of the reference's compiled base/linetrack.cc against the Python mirror
    (limap_b200.base.LineTrack): each side reads the other's file and the mirror's writer reproduces the reference's
    bytes; ComputeLineWeights (the loss weight of a supporting line in the refinement) = length / 30."""
    import limap.base as base
    z = _gold("linetrack")
    cases, segs = _linetrack_inputs()
    for case, c in enumerate(cases):
        n, line, img, lid, node, score, l2d, l3d, aux = c
        f_ref = tmp_path / f"ref_{case}.txt"
        f_ref.write_bytes(z[f"file_{case}"].tobytes())
        f_py = str(tmp_path / f"py_{case}.txt")
        _mirror_linetrack(c, f_py)
        assert open(f_py, "rb").read() == f_ref.read_bytes(), case  # byte for byte
        # the mirror reads the reference's file
        t2 = base.LineTrack()
        t2.Read(str(f_ref))
        assert t2.image_id_list == img.tolist() and t2.line_id_list == lid.tolist() and t2.count_images() == len(set(img))
        assert np.allclose([np.concatenate([l.start, l.end]) for l in t2.line2d_list], l2d, atol=1e-9)
        if aux:
            assert t2.node_id_list == node.tolist() and np.allclose(t2.score_list, score, atol=1e-9)
            assert np.allclose([np.concatenate([l.start, l.end]) for l in t2.line3d_list], l3d, atol=1e-9)
        # the reference read the mirror's file
        r = {x: z[f"read_{case}_{x}"] for x in ("line", "img", "lid", "node", "score", "l2d", "l3d", "ni", "got")}
        assert int(r["got"]) == n and np.array_equal(r["img"], img) and np.array_equal(r["lid"], lid) and r["ni"][0] == len(set(img))
        assert np.allclose(r["line"], np.nan_to_num(line), atol=1e-9) and np.allclose(r["l2d"], l2d, atol=1e-9)
        if aux:
            assert np.array_equal(r["node"], node) and np.allclose(r["score"], score, atol=1e-9) and np.allclose(r["l3d"], l3d, atol=1e-9)
    w = z["line_weights"]
    dx, dy = segs[:, 2] - segs[:, 0], segs[:, 3] - segs[:, 1]
    assert np.allclose(w, np.sqrt(dx * dx + dy * dy) / 30.0, rtol=1e-15, atol=0)


def _value_type_inputs():
    import limap.base as base
    rng = np.random.default_rng(92)
    out = []
    for it in range(3000):
        model = it & 1
        f = rng.uniform(300, 900)
        fy = f if model == 0 else f * rng.uniform(0.9, 1.1)
        cx, cy = rng.uniform(300, 400), rng.uniform(200, 300)
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        t = rng.normal(size=3) * 3
        cam_arr = np.array([model, f, fy, cx, cy, *q, *t])
        cam = base.Camera("SIMPLE_PINHOLE", [f, cx, cy], 0, (600, 800)) if model == 0 else \
            base.Camera("PINHOLE", [f, fy, cx, cy], 0, (600, 800))
        view = base.CameraView(cam, base.CameraPose(q, t))
        X = rng.normal(size=3) * 2 + view.pose.center() + view.R().T @ np.array([0, 0, 6.0])
        px = rng.uniform(0, 700, 2)
        seg = rng.uniform(0, 700, 4)
        Y = rng.normal(size=3) * 2 + view.pose.center() + view.R().T @ np.array([0, 0, 7.0])
        l3_arr = np.array([*X, *Y, view.pose.projdepth(X), view.pose.projdepth(Y), 0.1])
        out.append((view, cam_arr, X, px, seg, Y, l3_arr))
    return out


def _ref_value_types():
    L = ref.lib()
    p = orc._p
    rows = []
    for view, cam_arr, X, px, seg, Y, l3_arr in _value_type_inputs():
        b, r, d = np.zeros(2), np.zeros(3), np.zeros(2)
        L.ref_project_point(p(cam_arr), p(X), p(b))
        L.ref_ray_direction(p(cam_arr), p(px), p(r))
        L.ref_line2d_direction(p(seg), p(d))
        rows.append(np.concatenate([b, r, [L.ref_line2d_length(p(seg))], d, [L.ref_line3d_sensitivity(p(l3_arr), p(cam_arr))],
                                    [L.ref_line3d_uncertainty(p(l3_arr), p(cam_arr), 5.0)]]))
    return dict(out=np.stack(rows))


def test_python_value_types_against_compiled_reference():
    """a1 / a19: the Python value types of the mirror (limap_b200.base: Camera, CameraPose, CameraView, Line2d, Line3d) --
    the objects a runner handles -- against the reference's compiled base/{camera,pose,camera_view,linebase}.cc:
    projection, ray_direction, Line2d length / direction, Line3d sensitivity and uncertainty."""
    import limap.base as base
    gold = _gold("value_types")["out"]
    items = _value_type_inputs()
    assert len(items) == len(gold)
    for it, ((view, cam_arr, X, px, seg, Y, l3_arr), g) in enumerate(zip(items, gold)):
        b, r_ref, len_ref, d_ref, sens_ref, unc_ref = g[:2], g[2:5], g[5], g[6:8], g[8], g[9]
        a = np.asarray(view.projection(X))
        assert np.abs(a - b).max() <= 1e-9 * max(1.0, np.abs(b).max()), (it, a, b)
        assert np.abs(np.asarray(view.ray_direction(px)) - r_ref).max() <= 1e-12
        l2 = base.Line2d(seg[:2], seg[2:])
        assert abs(l2.length() - len_ref) <= 1e-12 and np.abs(np.asarray(l2.direction()) - d_ref).max() <= 1e-12
        l3 = base.Line3d(X, Y, 1.0, float(l3_arr[6]), float(l3_arr[7]), 0.1)
        assert abs(l3.sensitivity(view) - sens_ref) <= 1e-7
        assert abs(l3.computeUncertainty(view, 5.0) - unc_ref) <= 1e-10 * max(1.0, abs(l3_arr[6]))


def _flatten_tracks(tracks, view_of):
    off, tl, act, view, lid, node, score, l2d, l3d = [0], [], [], [], [], [], [], [], []
    l9 = lambda l: [*l.start, *l.end, l.depths[0], l.depths[1], l.uncertainty]
    for t in tracks:
        tl.append(l9(t.line))
        act.append(1 if t.active else 0)
        for k in range(t.count_lines()):
            view.append(view_of[int(t.image_id_list[k])])
            lid.append(int(t.line_id_list[k]))
            node.append(int(t.node_id_list[k]))
            score.append(float(t.score_list[k]))
            l2d.append([*t.line2d_list[k].start, *t.line2d_list[k].end])
            l3d.append(l9(t.line3d_list[k]))
        off.append(len(view))
    f = lambda a, dt, shp: np.ascontiguousarray(np.asarray(a, dt).reshape(shp))
    return (f(off, np.int64, -1), f(tl, np.float64, (-1, 9)), f(act, np.uint8, -1), f(view, np.int32, -1), f(lid, np.int32, -1),
            f(node, np.int32, -1), f(score, np.float64, -1), f(l2d, np.float64, (-1, 4)), f(l3d, np.float64, (-1, 9)))


def _ref_track_filter(op, a, b, n, lk, cams, flat):
    L = ref.lib()
    p = orc._p
    off, tl, act, view, lid, node, score, l2d, l3d = flat
    T, S = len(off) - 1, len(view)
    o = (np.zeros(T + 1, np.int64), np.zeros((max(T, 1), 9)), np.zeros(max(T, 1), np.uint8), np.zeros(max(S, 1), np.int32),
         np.zeros(max(S, 1), np.int32), np.zeros(max(S, 1), np.int32), np.zeros(max(S, 1)), np.zeros((max(S, 1), 4)),
         np.zeros((max(S, 1), 9)))
    model_ids, kvec, qvec, tvec = cams
    cfg = ref.linker_cfg(lk or {})
    To = L.ref_track_filter(op, float(a), float(b), int(n), C.byref(cfg), len(kvec), p(model_ids), p(kvec), p(qvec), p(tvec), T,
                            p(off), p(tl), p(act), p(view), p(lid), p(node), p(score), p(l2d), p(l3d), *[p(x) for x in o])
    S_o = int(o[0][To])
    return (o[0][:To + 1], o[1][:To], o[2][:To], o[3][:S_o], o[4][:S_o], o[5][:S_o], o[6][:S_o], o[7][:S_o], o[8][:S_o])


TRACK_FILTER_LK = dict(score_th=0.5, th_angle=8.0, th_overlap=0.01, th_smartoverlap=0.1, th_smartangle=1.0, th_perp=1.0,
                       th_innerseg=1.0)
# (name, reference operator, a, b, n, linker) of the chain reprojection -> remerge -> sensitivity -> overlap
TRACK_FILTER_STEPS = (("reprojection", 0, 4.0, 2.0, 0, None), ("remerge", 3, 0, 0, 0, TRACK_FILTER_LK),
                      ("sensitivity", 1, 75.0, 0, 4, None), ("overlap", 2, 0.5, 0, 4, None))


def _track_filter_chain():
    """The mirror's post-triangulation operators on the tracks of a triangulated scene (triangulation served by the oracle
    stand-in): the input tracks of every step and the mirror's output, with what the reference needs to rerun the step."""
    import limap.base as base
    import limap.merging as merging
    import limap.triangulation as triangulation
    from runner_utils import imagecols_of
    sc = make_scene(V=10, L=120, N=5, K=4, seed=93, noise_px=1.0, camera_mix=True)
    imagecols = imagecols_of(sc)
    tri = triangulation.GlobalLineTriangulator(dict(DEFAULT_YAML_TRIANGULATION))
    tri.SetRanges(sc.ranges)
    tri.Init({int(i): [base.Line2d(s[:2], s[2:]) for s in sc.lines_of(v)] for v, i in enumerate(sc.img_ids)}, imagecols)
    for i in sc.img_ids:
        tri.TriangulateImage(int(i), sc.matches[int(i)])
    t0 = tri.ComputeLineTracks()
    t1 = merging.filter_tracks_by_reprojection(t0, imagecols, 4.0, 2.0, num_outliers=0)
    t2 = merging.remerge(base.LineLinker3d(TRACK_FILTER_LK), t1, num_outliers=0)
    t3 = merging.filter_tracks_by_sensitivity(t2, imagecols, 75.0, 4)
    t4 = merging.filter_tracks_by_overlap(t3, imagecols, 0.5, 4)
    view_of = {int(i): v for v, i in enumerate(sc.img_ids)}
    cams = (np.ascontiguousarray(sc.model_ids, np.int32), sc.kvec, sc.qvec, sc.tvec)
    return [t0, t1, t2, t3, t4], view_of, cams


def _ref_track_filters():
    from runner_utils import install_oracle_backend
    with pytest.MonkeyPatch.context() as mp:
        install_oracle_backend(mp)
        chain, view_of, cams = _track_filter_chain()
    out = {}
    for k, (name, op, a, b, n, lk) in enumerate(TRACK_FILTER_STEPS):
        for j, arr in enumerate(_ref_track_filter(op, a, b, n, lk, cams, _flatten_tracks(chain[k], view_of))):
            out[f"{name}_{j}"] = arr
    return out


def test_track_level_filters_and_remerge_against_compiled_reference(monkeypatch):
    """f1 at track level: the mirror's post-triangulation operators (limap_b200.merging: list surgery in Python on top of the
    engine's per-support predicates, here served by the oracle stand-in so that the test runs without a GPU) against the
    reference's compiled FilterSupportingLines / FilterTracksBySensitivity / FilterTracksByOverlap / iterated
    RemergeLineTracks, on the tracks of a triangulated scene: same tracks in the same order, same supports, same lines."""
    from runner_utils import install_oracle_backend
    install_oracle_backend(monkeypatch)
    chain, view_of, cams = _track_filter_chain()
    assert len(chain[0]) > 30
    z = _gold("track_filters")

    def same(py_tracks, tag):
        flat_ref = [z[f"{tag}_{j}"] for j in range(9)]
        a = _flatten_tracks(py_tracks, view_of)
        assert np.array_equal(a[0], flat_ref[0]), tag                       # track boundaries
        for k in (3, 4, 5):                                                  # views, line ids, node ids in order
            assert np.array_equal(a[k], flat_ref[k]), (tag, k)
        assert np.array_equal(a[2], flat_ref[2]), tag                        # active flags
        assert np.allclose(a[6], flat_ref[6], atol=1e-12) and np.allclose(a[7], flat_ref[7], atol=1e-12)
        d = np.minimum(np.abs(a[1][:, :6] - flat_ref[1][:, :6]).max(1, initial=0),
                       np.abs(a[1][:, :6] - flat_ref[1][:, [3, 4, 5, 0, 1, 2]]).max(1, initial=0))
        assert d.max(initial=0) < 1e-8, (tag, d.max())
        return len(py_tracks)

    n = [len(chain[0])] + [same(chain[k + 1], s[0]) for k, s in enumerate(TRACK_FILTER_STEPS)]
    assert n[0] >= n[1] >= n[2] >= n[3] >= n[4] > 5 and n[4] < n[0]


def _max_image_dim_cases():
    rng = np.random.default_rng(94)
    cases = [(801, 1602, 801), (600, 800, 400), (1000, 3, 500)]  # (h, w, val): the first has ratio * h == 400.5 exactly
    cases += [(int(rng.integers(100, 3000)), int(rng.integers(100, 3000)), int(rng.integers(50, 3500))) for _ in range(400)]
    return cases


def _max_image_dim_params(model):
    return [612.3, 400.5, 299.25] if model == 0 else [612.3, 640.7, 400.5, 299.25]


def _ref_max_image_dim():
    L = ref.lib()
    L.ref_camera_set_max_image_dim.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    cases = _max_image_dim_cases()
    hw_out, params_out = np.zeros((len(cases), 2, 2), np.int32), np.zeros((len(cases), 2, 4))
    for k, (h, w, val) in enumerate(cases):
        for model in (0, 1):
            params = _max_image_dim_params(model)
            pr = np.array(params + [0.0] * (4 - len(params)))
            hw = np.array([h, w], np.int32)
            L.ref_camera_set_max_image_dim(model, orc._p(pr), orc._p(hw), val)
            hw_out[k, model], params_out[k, model] = hw, pr
    return dict(hw=hw_out, params=params_out)


def test_camera_set_max_image_dim_rounding():
    """Camera::set_max_image_dim (the runner's max_image_dim): the new size is C round() of ratio * size (halves away from
    zero, not to even), the intrinsics follow colmap::Camera::Rescale."""
    import limap.base as base
    z = _gold("max_image_dim")
    cases = _max_image_dim_cases()
    assert len(cases) == len(z["hw"])
    n_half = 0
    for k, (h, w, val) in enumerate(cases):
        for model in (0, 1):
            params = _max_image_dim_params(model)
            cam = base.Camera("SIMPLE_PINHOLE" if model == 0 else "PINHOLE", list(params), 0, (h, w))
            cam.set_max_image_dim(val)
            hw, pr = z["hw"][k, model], z["params"][k, model]
            assert (cam.h(), cam.w()) == (int(hw[0]), int(hw[1])), (h, w, val)
            assert np.allclose(cam.params, pr[:len(params)], rtol=1e-15, atol=0), (h, w, val)
        r = val / max(h, w)
        n_half += r < 1 and (abs(r * h % 1 - 0.5) < 1e-12 or abs(r * w % 1 - 0.5) < 1e-12)
    assert n_half >= 1


# golden file name -> the reference's outputs on this module's inputs (tests/golden/make_ref_golden.py)
REFERENCE_OUTPUTS = {**{"pipeline_" + name: (lambda name=name: _ref_pipeline(name)) for name in CASES},
                     "boundary_min_length": _ref_boundary_min_length,
                     **{"boundary_3d_" + name: (lambda name=name: _ref_boundary_3d(name))
                        for name in ("angle_10", "angle_14.4775", "angle_20", "scaleinv")},
                     "two_view": _ref_two_view, "camera": _ref_camera, "linker": _ref_linker, "aggregate": _ref_aggregate,
                     "residuals": _ref_residuals, "filters": _ref_filters, "sfm": _ref_sfm, "vp": _ref_vp,
                     "linetrack": _ref_linetrack, "value_types": _ref_value_types, "track_filters": _ref_track_filters,
                     "max_image_dim": _ref_max_image_dim}
