"""Scenes with decisions planted exactly on a threshold, for the pinning (CPU) and parity (GPU) tests.

min_length_scene: both 2D length tests of phase A, `!(length <= min_length_2d)` on the source line
(base_line_triangulator.cc:166) and on the matched line, are decided by exact equality. Planted segments have integer
endpoints and a Pythagorean offset ((12, 16), (16, 12), (20, 0), ...), so their length is exactly 20 in fp64 (the
squares, their sum and the square root are exact): the input data sits on the threshold with no rounding budget at all.
With min_length_2d = 20 the reference rejects them; slightly below 20 they triangulate (the builder asserts both through
the oracle, so the scene cannot silently lose its planted decisions)."""
import numpy as np

from limap_b200.config import DEFAULT_YAML_TRIANGULATION
from limap_b200.synth import make_scene

MIN_LENGTH = 20.0
_OFFSETS = np.array([(12, 16), (16, 12), (20, 0), (0, 20), (12, -16), (16, -12)], np.float64)


def min_length_cfg(min_length=MIN_LENGTH, **kw):
    c = dict(DEFAULT_YAML_TRIANGULATION, debug_mode=True, min_length_2d=min_length)
    c.update(kw)
    return c


def _feed(t, sc):
    t.upload(sc)
    t.set_ranges(*sc.ranges)
    for i in sc.img_ids:
        t.add_image_matches(int(i), *sc.flat_matches(int(i)))
    return t


def min_length_scene(per_view=8, seed=501, check=True):
    """(scene, planted node indices): in every view the `per_view` segments of true lines that triangulate best are
    replaced by a length-20 segment through their integer-rounded midpoint, along the Pythagorean direction closest to
    theirs."""
    sc = make_scene(V=6, L=60, N=4, K=4, seed=seed)
    from oracle.oracle import OracleTri
    o = _feed(OracleTri(min_length_cfg(0.0), threads=1), sc)
    planted = []
    for v, i in enumerate(sc.img_ids):
        _, _, nc = o.get_best(int(i))
        a = int(sc.line_off[v])
        order = [l for l in np.argsort(-nc, kind="stable") if sc.gt_id[a + l] >= 0][:per_view]
        for l in order:
            s = sc.segs[a + l]
            d = (s[2:] - s[:2]) / np.linalg.norm(s[2:] - s[:2])
            off = _OFFSETS[int(np.argmax(np.abs(_OFFSETS @ d)))]
            if off @ d < 0:
                off = -off
            mid = np.round((s[:2] + s[2:]) / 2)
            sc.segs[a + l] = np.concatenate([mid - off / 2, mid + off / 2])
            planted.append(a + l)
    planted = np.asarray(sorted(planted), np.int64)
    seg = sc.segs[planted]
    assert np.all(np.sqrt((seg[:, 0] - seg[:, 2]) ** 2 + (seg[:, 1] - seg[:, 3]) ** 2) == MIN_LENGTH)
    if check:
        below = _feed(OracleTri(min_length_cfg(np.nextafter(MIN_LENGTH, 0.0)), threads=1), sc)
        at = _feed(OracleTri(min_length_cfg(), threads=1), sc)
        nc_below = np.concatenate([below.get_best(int(i))[2] for i in sc.img_ids])
        nc_at = np.concatenate([at.get_best(int(i))[2] for i in sc.img_ids])
        assert (nc_below[planted] > 0).sum() >= len(planted) // 2  # the source-line test decides these nodes
        assert (nc_at[planted] == 0).all()
        assert nc_at.sum() < nc_below.sum() - (nc_below[planted]).sum()  # ... and the neighbour-line test other rows
    return sc, planted


# ---- phase B, 3D linker: pairs planted at threshold * (1 -+ delta) -------------------------------------------------
# Each planted node is a 2D line of a source view with exactly two match rows, one into view a and one into view b, so
# it has two candidates A and B (from different images) and the score of A is the one pair score (A, B). Both 3D lines
# lie in the back-projection plane of the source segment with their endpoints on its two rays; their segments in views
# a and b are their exact fp64 projections, so plane-pair triangulation returns them to rounding (~1e-16 relative).
# The 2D linker is switched off (score 1), so the planted 3D sub-test decides alone.
#
# Budget: every planted decision is a distance or an angle of 10..20 deg between triangulated lines. The reference's own
# rounding of these quantities is below 1e-13 relative (the triangulation returns the lines to ~1e-16; acos at 10 deg
# amplifies 1e-16 to ~1e-15), so all three tiers, 1e-6, 1e-9 and 1e-11 relative, are decided by the geometry and not by
# rounding. The builder asserts this through the oracle for every planted pair: A scores 0 at +delta and >= score_th at
# -delta.
DELTAS = (1e-6, 1e-9, 1e-11)
# (depth of the planted lines, offset of the group's source camera from the world origin): depth ~1, depth ~1e3, and
# depth ~1e3 at asset-unit coordinates (|X| ~ 1e3, the asset-scale x100 scenes)
GEOMETRIES = ((1.0, 0.0), (1e3, 0.0), (1e3, 700.0))
EPS = 1e-12
SCORE_TH = 0.5
# name -> (3D linker th_angle, th_scaleinv, planted decisions); th_angle 14.4775 puts the decision on the switch of
# pair_score_fast from the asin^2 series (sin^2 <= 1/16) to acos
BOUNDARY_3D = {
    "angle_10": (10.0, 10.0, ("angle",)),
    "angle_14.4775": (14.4775, 10.0, ("angle",)),
    "angle_20": (20.0, 10.0, ("angle",)),
    "scaleinv": (30.0, 0.015, ("scaleinv_start", "scaleinv_end")),
}


def boundary_3d_cfg(name):
    th_angle, th_scaleinv, _ = BOUNDARY_3D[name]
    return dict(DEFAULT_YAML_TRIANGULATION, debug_mode=True, fullscore_th=0.25, min_length_2d=0.0,
                linker2d_config=dict(score_th=SCORE_TH, use_angle=False, use_overlap=False, use_perp=False,
                                     use_smartangle=False),
                linker3d_config=dict(DEFAULT_YAML_TRIANGULATION["linker3d_config"], score_th=SCORE_TH,
                                     th_angle=th_angle, th_scaleinv=th_scaleinv))


def _look_at(C, target, rng):
    from limap_b200.base import CameraPose
    from limap_b200.synth import _rot_to_quat
    z = (target - C) / np.linalg.norm(target - C)
    x = np.cross(z, np.array([0.0, 0.0, 1.0]) + rng.normal(scale=0.1, size=3))
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z], 0)
    q = _rot_to_quat(R)
    t = -R @ C
    return q, t, CameraPose(q, t).R()  # project with R as the engine and the reference rebuild it from q


def _project(K, R, t, X):
    h = R @ X + t
    return np.array([h[0] / (h[2] + EPS) * K[0] + K[2], h[1] / (h[2] + EPS) * K[1] + K[3]])


def _angle(u, v):
    c = np.cross(u, v)
    return np.degrees(np.arctan2(np.linalg.norm(c), abs(float(u @ v))))


def boundary_3d_scene(name, seed=601):
    """(scene, planted) with planted = [(node index, decision, delta, sign)], sign +1: A must score 0, -1: >= score_th."""
    from limap_b200.synth import Scene
    th_angle, th_si, decisions = BOUNDARY_3D[name]
    rng = np.random.default_rng(seed)
    f = 692.82
    K = np.array([f, f, 400.0, 300.0])
    kvec, qvec, tvec, segs, line_off, planted, matches = [], [], [], [], [0], [], {}
    for depth, origin in GEOMETRIES:
        C0 = origin + rng.normal(size=3) * depth * 0.1
        fwd = rng.normal(size=3)
        fwd /= np.linalg.norm(fwd)
        focus = C0 + depth * fwd
        side = np.cross(fwd, rng.normal(size=3))
        side /= np.linalg.norm(side)
        Ca, Cb = C0 + 0.35 * depth * side, C0 - 0.3 * depth * side + 0.1 * depth * fwd
        cams = [_look_at(C, focus, rng) for C in (C0, Ca, Cb)]
        R0, t0 = cams[0][2], cams[0][1]
        rows = [(d, dl, s) for d in decisions for dl in DELTAS for s in (1, -1)]
        ls, la, lb = [], [], []
        for k, (dec, dl, sgn) in enumerate(rows):
            # the base line A: depth ~ `depth`, length depth / 2, roughly across the view
            M = C0 + depth * (fwd + 0.15 * rng.normal(size=3))
            while True:  # not near an epipolar plane of view a or b (the ray-plane angle test of phase A)
                u = np.cross(M - C0, rng.normal(size=3))
                u /= np.linalg.norm(u)
                if min(_angle(u, C - C0) for C in (Ca, Cb)) > 40.0:
                    break
            S, E = M - u * depth * 0.25, M + u * depth * 0.25
            rs, re_ = (S - C0) / np.linalg.norm(S - C0), (E - C0) / np.linalg.norm(E - C0)
            lam_s, lam_e = float(np.linalg.norm(S - C0)), float(np.linalg.norm(E - C0))
            S, E = C0 + lam_s * rs, C0 + lam_e * re_
            zs, ze = float((R0 @ S + t0)[2]), float((R0 @ E + t0)[2])
            SB, EB = S, E
            if dec == "angle":
                target = th_angle * (1 + sgn * dl)
                lo, hi = lam_e, lam_e * 4
                for _ in range(200):  # bisection on the end point along the end ray: the angle grows with mu
                    mu = 0.5 * (lo + hi)
                    if _angle(E - S, C0 + mu * re_ - S) < target:
                        lo = mu
                    else:
                        hi = mu
                EB = C0 + 0.5 * (lo + hi) * re_
            elif dec == "scaleinv_start":
                SB = C0 + (lam_s + th_si * (zs + EPS) * (1 + sgn * dl)) * rs
            else:
                EB = C0 + (lam_e + th_si * (ze + EPS) * (1 + sgn * dl)) * re_
            ls.append(np.concatenate([_project(K, R0, t0, S), _project(K, R0, t0, E)]))
            la.append(np.concatenate([_project(K, cams[1][2], cams[1][1], S), _project(K, cams[1][2], cams[1][1], E)]))
            lb.append(np.concatenate([_project(K, cams[2][2], cams[2][1], SB), _project(K, cams[2][2], cams[2][1], EB)]))
            planted.append((int(line_off[-1]) + k, dec, dl, sgn))
        v0 = len(kvec)
        ids = [v0 + j for j in range(3)]
        for q, t, _ in cams:
            kvec.append(K); qvec.append(q); tvec.append(t)
        for s in (ls, la, lb):
            segs.append(np.asarray(s))
            line_off.append(line_off[-1] + len(s))
        n = len(rows)
        pairs = np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32)
        matches[ids[0]] = {ids[1]: pairs.copy(), ids[2]: pairs.copy()}
        matches[ids[1]], matches[ids[2]] = {}, {}
    V = len(kvec)
    img_ids = np.arange(V, dtype=np.int32)
    neighbors = {int(i): [] for i in img_ids}
    for i, m in matches.items():
        neighbors[i] = sorted(m)
    segs = np.ascontiguousarray(np.concatenate(segs), np.float64)
    sc = Scene(img_ids=img_ids, model_ids=np.zeros(V, np.int32), kvec=np.ascontiguousarray(kvec),
               qvec=np.ascontiguousarray(qvec), tvec=np.ascontiguousarray(tvec), line_off=np.asarray(line_off, np.int64),
               segs=segs, gt_id=-np.ones(len(segs), np.int32), neighbors=neighbors, matches=matches,
               ranges=(np.full(3, -1e7), np.full(3, 1e7)))
    return sc, planted


def planted_scores(t, sc, planted):
    """Score of candidate A (the first candidate: view a is the lower image id) of every planted node, with the number
    of candidates of the node."""
    out = []
    for node, *_ in planted:
        v = int(np.searchsorted(sc.line_off, node, "right") - 1)
        cl, cng = t.get_cands_node(int(sc.img_ids[v]), int(node - sc.line_off[v]))
        out.append((len(cng), float(cl[0, 9]) if cl is not None and len(cl) else np.nan))
    return out


def check_planted(t, sc, planted):
    """Every planted node has its two candidates; A scores 0 at +delta and >= score_th at -delta."""
    for (node, dec, dl, sgn), (n, s) in zip(planted, planted_scores(t, sc, planted)):
        assert n == 2, (node, dec, dl, sgn, n)
        assert (s == 0.0) if sgn > 0 else (s >= SCORE_TH), (node, dec, dl, sgn, s)


def checked_boundary_3d_scene(name):
    from oracle.oracle import OracleTri
    sc, planted = boundary_3d_scene(name)
    o = _feed(OracleTri(boundary_3d_cfg(name), threads=1), sc)
    check_planted(o, sc, planted)
    return sc, planted
