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


def _seg(cam, S, E):
    """The 2D segment of the 3D segment (S, E) in view cam = (q, t, R)."""
    return np.concatenate([_project(K_ALL, cam[2], cam[1], S), _project(K_ALL, cam[2], cam[1], E)])


def _angle(u, v):
    c = np.cross(u, v)
    return np.degrees(np.arctan2(np.linalg.norm(c), abs(float(u @ v))))


F = 692.82
K_ALL = np.array([F, F, 400.0, 300.0])


def _group(rng, depth, origin):
    """A source camera C0 and two neighbours a and b ~0.35 depth to either side, all looking at the point `depth` ahead
    of C0: (C0, forward direction, Ca, Cb, [(q, t, R)] of the three views)."""
    C0 = origin + rng.normal(size=3) * depth * 0.1
    fwd = rng.normal(size=3)
    fwd /= np.linalg.norm(fwd)
    focus = C0 + depth * fwd
    side = np.cross(fwd, rng.normal(size=3))
    side /= np.linalg.norm(side)
    Ca, Cb = C0 + 0.35 * depth * side, C0 - 0.3 * depth * side + 0.1 * depth * fwd
    return C0, fwd, Ca, Cb, [_look_at(C, focus, rng) for C in (C0, Ca, Cb)]


def _base_line(rng, C0, fwd, depth, others, accept=None, half=0.25):
    """A line at depth ~ `depth`, length 2 half depth, roughly across the view, with endpoints re-expressed on their rays:
    (S, E, start ray, end ray, |S - C0|, |E - C0|). `accept(S, E)` may reject it (drawn again)."""
    while True:
        M = C0 + depth * (fwd + 0.15 * rng.normal(size=3))
        while True:  # not near an epipolar plane of view a or b (the ray-plane angle test of phase A)
            u = np.cross(M - C0, rng.normal(size=3))
            u /= np.linalg.norm(u)
            if min(_angle(u, C - C0) for C in others) > 40.0:
                break
        S, E = M - u * depth * half, M + u * depth * half
        rs, re_ = (S - C0) / np.linalg.norm(S - C0), (E - C0) / np.linalg.norm(E - C0)
        lam_s, lam_e = float(np.linalg.norm(S - C0)), float(np.linalg.norm(E - C0))
        S, E = C0 + lam_s * rs, C0 + lam_e * re_
        if accept is None or accept(S, E):
            return S, E, rs, re_, lam_s, lam_e


def boundary_3d_scene(name, seed=601):
    """(scene, planted) with planted = [(node index, decision, delta, sign)], sign +1: A must score 0, -1: >= score_th."""
    th_angle, th_si, decisions = BOUNDARY_3D[name]
    rng = np.random.default_rng(seed)
    kvec, qvec, tvec, segs, line_off, planted, matches = [], [], [], [], [0], [], {}
    for depth, origin in GEOMETRIES:
        C0, fwd, Ca, Cb, cams = _group(rng, depth, origin)
        R0, t0 = cams[0][2], cams[0][1]
        rows = [(d, dl, s) for d in decisions for dl in DELTAS for s in (1, -1)]
        ls, la, lb = [], [], []
        for k, (dec, dl, sgn) in enumerate(rows):
            S, E, rs, re_, lam_s, lam_e = _base_line(rng, C0, fwd, depth, (Ca, Cb))
            zs, ze = float((R0 @ S + t0)[2]), float((R0 @ E + t0)[2])
            SB, EB = S, E
            if dec == "angle":
                EB = _end_at_angle(C0, S, E, re_, lam_e, th_angle * (1 + sgn * dl))
            elif dec == "scaleinv_start":
                SB = C0 + (lam_s + th_si * (zs + EPS) * (1 + sgn * dl)) * rs
            else:
                EB = C0 + (lam_e + th_si * (ze + EPS) * (1 + sgn * dl)) * re_
            ls.append(_seg(cams[0], S, E))
            la.append(_seg(cams[1], S, E))
            lb.append(_seg(cams[2], SB, EB))
            planted.append((int(line_off[-1]) + k, dec, dl, sgn))
        _add_group(K_ALL, cams, (ls, la, lb), kvec, qvec, tvec, segs, line_off, matches)
    return _assemble(kvec, qvec, tvec, segs, line_off, matches, (np.full(3, -1e7), np.full(3, 1e7))), planted


def _end_at_angle(C0, S, E, re_, lam_e, target):
    """The point of the end ray at which the segment from S makes `target` degrees with E - S (bisection: the angle
    grows with the distance along the ray)."""
    lo, hi = lam_e, lam_e * 4
    for _ in range(200):
        mu = 0.5 * (lo + hi)
        if _angle(E - S, C0 + mu * re_ - S) < target:
            lo = mu
        else:
            hi = mu
    return C0 + 0.5 * (lo + hi) * re_


def _add_group(K, cams, lines, kvec, qvec, tvec, segs, line_off, matches):
    """Appends the three views of a group and their segments; source segment k matches segment k of views a and b."""
    ls, la, lb = lines
    v0 = len(kvec)
    ids = [v0 + j for j in range(3)]
    for q, t, _ in cams:
        kvec.append(K); qvec.append(q); tvec.append(t)
    for s in (ls, la, lb):
        segs.append(np.asarray(s))
        line_off.append(line_off[-1] + len(s))
    n = len(ls)
    pairs = np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32)
    matches[ids[0]] = {ids[1]: pairs.copy(), ids[2]: pairs.copy()}
    matches[ids[1]], matches[ids[2]] = {}, {}


def _assemble(kvec, qvec, tvec, segs, line_off, matches, ranges):
    from limap_b200.synth import Scene
    V = len(kvec)
    img_ids = np.arange(V, dtype=np.int32)
    neighbors = {int(i): [] for i in img_ids}
    for i, m in matches.items():
        neighbors[i] = sorted(m)
    segs = np.ascontiguousarray(np.concatenate(segs), np.float64)
    sc = Scene(img_ids=img_ids, model_ids=np.zeros(V, np.int32), kvec=np.ascontiguousarray(kvec),
               qvec=np.ascontiguousarray(qvec), tvec=np.ascontiguousarray(tvec), line_off=np.asarray(line_off, np.int64),
               segs=segs, gt_id=-np.ones(len(segs), np.int32), neighbors=neighbors, matches=matches, ranges=ranges)
    return sc


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


# ---- phase A gates, 2D linker sub-tests and phase C: decisions planted at threshold * (1 -+ delta) -------------------
# Same node shape as above: a source segment with one match row into view a and one into view b. Three kinds of outcome:
#   "cand"  (phase A): the gate of the row into view a is planted; the outcome is whether that row yields a candidate.
#           The row into view b is ordinary and always does.
#   "score" (2D linker): a sub-test of LineLinker2d between candidate A projected into view b and the segment of view b
#           is planted; A scores 0 or >= score_th, as in check_planted. The 3D linker is held clear (th_angle 90,
#           th_scaleinv 1), every other 2D sub-test is off or clear.
#   "valid" (phase C): the one pair score of the node is planted at fullscore_th through the 3D angle; the outcome is
#           whether the node has valid connections.
# Every builder asserts its planted outcomes through the oracle (checked_planted_scene), so a family whose geometry does
# not land the decision as intended fails instead of turning into an ordinary scene.
#
# Tiers. The ray-plane angle adds 4e-10: 1e-9 on the angle is ~2e-9 on the squared form the kernel compares, just outside
# its 1e-9 band (cmp_margin), 4e-10 lies inside it. The epipolar IoU is planted at an absolute offset, because the band in
# which the kernel recomputes the reference's normalised form is absolute (1e-7): 1e-5 and 1.5e-7 lie outside it, 5e-8
# and 1e-11 inside. In iou_grazing the epipolar lines meet the segment at 1e-1, 1e-2 and 1e-3 deg, where every form of
# the intersection loses ~1e-16 / sin(angle) relative (~3e-11 in the IoU at 1e-3 deg, the reference's own rounding), so
# that family stops at 5e-8.
TRI_ANGLE_DELTAS = DELTAS + (4e-10,)
IOU_TH = 0.1
IOU_DELTAS = (1e-5, 1.5e-7, 5e-8, 1e-11)
GRAZING_DELTAS = (1e-5, 1.5e-7, 5e-8)
GRAZING_ANGLES = (1e-1, 1e-2, 1e-3)
SENSITIVITY_TH = 70.0
L2D = DEFAULT_YAML_TRIANGULATION["linker2d_config"]  # score_th 0.5, th_angle 5, th_perp 2, th_overlap 0.05
SMART_OVERLAP, SMART_ANGLE = 0.2, 1.0                 # LineLinker2dConfig defaults (the yaml keeps them)
SMART_BIO = (0.06, 0.08, 0.1)                         # smart sigma 1.27, 1.8, 2.33 deg: the plain angle test is 2x clear
FULLSCORE_TH = 0.75


def _seg_px(cam, S, E):
    """The 2D segment of (S, E) in view cam, projected without the EPS of dehomogeneous(): the back-projected rays of
    these pixels pass through S and E to rounding, so the triangulated lines are (S, E) themselves."""
    out = []
    for X in (S, E):
        h = cam[2] @ X + cam[1]
        out += [h[0] / h[2] * K_ALL[0] + K_ALL[2], h[1] / h[2] * K_ALL[1] + K_ALL[3]]
    return np.asarray(out)


def _seg_ref(cam, S, E):
    """CameraView::projection of (S, E) as the reference evaluates it: dehomogeneous(K (R X + T)), EPS included."""
    Km = np.array([[K_ALL[0], 0.0, K_ALL[2]], [0.0, K_ALL[1], K_ALL[3]], [0.0, 0.0, 1.0]])
    out = []
    for X in (S, E):
        h = Km @ (cam[2] @ X + cam[1])
        out += [h[0] / (h[2] + EPS), h[1] / (h[2] + EPS)]
    return np.asarray(out)


def _epipolar_iou(l1, cam1, l2, cam2):
    """compute_epipolar_IoU (triangulation/functions.cc) through the oracle, whose restatement is pinned to the
    reference's compiled function."""
    from oracle import oracle as orc
    c1, c2 = (orc.cam_array(0, K_ALL, c[0], c[1]) for c in (cam1, cam2))
    f = orc.lib().orc_compute_epipolar_IoU
    return f(orc._p(np.ascontiguousarray(l1)), orc._p(c1), orc._p(np.ascontiguousarray(l2)), orc._p(c2))


def _slide_to_iou(l1, cam1, seg, cam2, iou):
    """The segment slid along its own line (its back-projection plane is unchanged) until the epipolar IoU of l1 in it
    is `iou`: bisection on the slide, which lowers the IoU from 1 at no slide."""
    v = seg[2:] - seg[:2]
    lo, hi = 0.0, 1.0
    for _ in range(200):
        s = 0.5 * (lo + hi)
        if _epipolar_iou(l1, cam1, np.concatenate([seg[:2] + s * v, seg[2:] + s * v]), cam2) > iou:
            lo = s
        else:
            hi = s
    s = 0.5 * (lo + hi)
    return np.concatenate([seg[:2] + s * v, seg[2:] + s * v])


def _unit(v):
    return v / np.linalg.norm(v)


def _phase_a_cfg(**kw):
    # fullscore_th 0.25 rather than the yaml's 1: where both rows triangulate the same line, the pair score is 1 up to the
    # rounding of acos near 0, and a threshold of 1 would turn that rounding into the valid connections
    return dict(DEFAULT_YAML_TRIANGULATION, debug_mode=True, fullscore_th=0.25, **kw)


def _l2d_cfg(iou=IOU_TH, **l2d):
    return dict(DEFAULT_YAML_TRIANGULATION, debug_mode=True, fullscore_th=0.25, IoU_threshold=iou,
                linker2d_config=dict(L2D, **l2d),
                linker3d_config=dict(DEFAULT_YAML_TRIANGULATION["linker3d_config"], th_angle=90.0, th_scaleinv=1.0))


def _rows(decisions, deltas):
    return [(d, dl, s) for d in decisions for dl in deltas for s in (1, -1)]


def _tri_angle_row(g, dec, dl, sgn, th):
    """The plane of the segment in view a makes th * (1 + sgn dl) deg with the start (or end) ray of the source segment
    and ~20 deg more with the other ray: the plane through Ca whose normal n has n . r = sin(angle) and which meets r at
    the source line's own point. Lines are drawn with their source plane far from the epipolar plane of view a, so that
    such a plane exists with the other ray well above the threshold. Below the threshold the row is rejected."""
    def accept(S, E):
        return abs(_unit(np.cross(S - g.C0, E - g.C0)) @ _unit(g.Ca - g.C0)) > 0.7
    S, E, rs, re_, lam_s, lam_e = _base_line(g.rng, g.C0, g.fwd, g.depth, (g.Ca, g.Cb), accept)
    rp, ro, lam_p = (rs, re_, lam_s) if dec == "start" else (re_, rs, lam_e)
    a = np.radians(th * (1 + sgn * dl))
    w1 = _unit(ro - (ro @ rp) * rp)
    w2 = np.cross(rp, w1)
    B = g.Ca - g.C0
    b1, b2 = w1 @ B, w2 @ B
    # n = sin(a) rp + cos(a) (cos(phi) w1 + sin(phi) w2) with n . B = lam_p sin(a): the plane meets rp at lam_p
    phi0, dphi = np.arctan2(b2, b1), np.arccos(np.tan(a) * (lam_p - rp @ B) / np.hypot(b1, b2))
    phi = max((phi0 + dphi, phi0 - dphi), key=np.cos)  # the other ray at ~angle + 20 deg
    n = np.sin(a) * rp + np.cos(a) * (np.cos(phi) * w1 + np.sin(phi) * w2)
    Pp, Po = g.C0 + (n @ B) / (n @ rp) * rp, g.C0 + (n @ B) / (n @ ro) * ro
    Sa, Ea = (Pp, Po) if dec == "start" else (Po, Pp)
    return _seg_px(g.cams[0], S, E), _seg_px(g.cams[1], Sa, Ea), _seg_px(g.cams[2], S, E), sgn < 0


def _other_row(g, S, E):
    """The segment of view b of a phase-A row: the projection of the line turned by 3 deg about its midpoint within the
    source segment's back-projection plane, so that candidate B is a different line than A (two identical candidates
    tie on their scores, and rounding would pick the best one) that still triangulates exactly."""
    n, M = _unit(np.cross(S - g.C0, E - g.C0)), (S + E) / 2
    c, s = np.cos(np.radians(3.0)), np.sin(np.radians(3.0))
    turn = lambda v: c * v + s * np.cross(n, v) + (1 - c) * (n @ v) * n
    return _seg_px(g.cams[2], M + turn(S - M), M + turn(E - M))


def _iou_row(g, dec, dl, sgn):
    S, E, *_ = _base_line(g.rng, g.C0, g.fwd, g.depth, (g.Ca, g.Cb))
    ls = _seg_px(g.cams[0], S, E)
    la = _slide_to_iou(ls, g.cams[0], _seg_px(g.cams[1], S, E), g.cams[1], IOU_TH + sgn * dl)
    return ls, la, _other_row(g, S, E), sgn < 0


def _grazing_row(g, alpha, dl, sgn):
    """A line turned by ~alpha deg out of the epipolar plane of view a through its midpoint, across the ray: in view a
    the epipolar lines of the source endpoints meet its segment at ~alpha deg."""
    M = g.C0 + g.depth * (g.fwd + 0.15 * g.rng.normal(size=3))
    ne = _unit(np.cross(M - g.C0, g.Ca - g.C0))
    u0 = _unit(np.cross(ne, M - g.C0))
    epipole = _project(K_ALL, g.cams[1][2], g.cams[1][1], g.C0)

    def line(beta):
        u = np.cos(beta) * u0 + np.sin(beta) * ne
        return M - u * g.depth * 0.25, M + u * g.depth * 0.25

    def image_angle(beta):
        la = _seg_px(g.cams[1], *line(beta))
        return _angle(np.append(la[2:] - la[:2], 0.0), np.append(la[:2] - epipole, 0.0))
    beta = np.radians(alpha)
    for _ in range(3):  # the image angle is proportional to beta at these angles
        beta *= alpha / image_angle(beta)
    S, E = line(beta)
    ls = _seg_px(g.cams[0], S, E)
    la = _slide_to_iou(ls, g.cams[0], _seg_px(g.cams[1], S, E), g.cams[1], IOU_TH + sgn * dl)
    return ls, la, _other_row(g, S, E), sgn < 0


def _sensitivity(cam, S, E):
    """Line3d::sensitivity(view): 90 deg minus the angle between the line and the ray through its projection's middle."""
    R = cam[2]
    l = _seg_ref(cam, S, E)
    mid = (l[:2] + l[2:]) / 2
    ray = _unit(R.T @ np.array([(mid[0] - K_ALL[2]) / K_ALL[0], (mid[1] - K_ALL[3]) / K_ALL[1], 1.0]))
    return 90.0 - np.degrees(np.arccos(abs(_unit(E - S) @ ray)))


def _sensitivity_row(g, dec, dl, sgn):
    """A line ~20 deg from view 0's ray through its middle and ~10 deg from view a's: both sensitivities are near or
    above 70 deg, view 0's is planted (bisection on the line's angle to the ray), view a's is clearly above. Above the
    threshold in both views the row is rejected."""
    M = g.C0 + g.depth * (g.fwd + 0.15 * g.rng.normal(size=3))
    m, ma = _unit(M - g.C0), _unit(M - g.Ca)
    psi = np.arccos(m @ ma)
    qa = _unit(ma - (ma @ m) * m)
    r20, r10 = np.radians(20.0), np.radians(10.0)
    om = np.arccos(np.clip((np.cos(r10) - np.cos(r20) * np.cos(psi)) / (np.sin(r20) * np.sin(psi)), -1.0, 1.0))
    q = np.cos(om) * qa + np.sin(om) * np.cross(m, qa)

    def line(rho):
        u = np.cos(rho) * m + np.sin(rho) * q
        return M - u * g.depth * 0.25, M + u * g.depth * 0.25
    target = SENSITIVITY_TH * (1 + sgn * dl)
    lo, hi = np.radians(5.0), np.radians(40.0)
    for _ in range(200):  # the sensitivity falls as the line turns away from the ray
        rho = 0.5 * (lo + hi)
        if _sensitivity(g.cams[0], *line(rho)) > target:
            lo = rho
        else:
            hi = rho
    S, E = line(0.5 * (lo + hi))
    assert _sensitivity(g.cams[1], S, E) > SENSITIVITY_TH + 2.0
    return _seg_px(g.cams[0], S, E), _seg_px(g.cams[1], S, E), _other_row(g, S, E), sgn > 0


def _overlap(l1, l2):
    """compute_overlap (line_dists.h): l1 projected onto l2, in units of l2's length, intersected with [0, 1]."""
    v = l2[2:] - l2[:2]
    ln = np.linalg.norm(v)
    p = sorted(((l1[:2] - l2[:2]) @ v / ln / ln, (l1[2:] - l2[:2]) @ v / ln / ln))
    return min(p[1], 1.0) - max(p[0], 0.0)


def _bioverlap(l1, l2):
    return max(_overlap(l1, l2), _overlap(l2, l1))


def _rotated(seg, deg):
    """The segment turned by deg about its midpoint."""
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    mid, h = (seg[:2] + seg[2:]) / 2, (seg[2:] - seg[:2]) / 2
    h = np.array([c * h[0] - s * h[1], s * h[0] + c * h[1]])
    return np.concatenate([mid - h, mid + h])


def _slid(seg, s):
    v = seg[2:] - seg[:2]
    return np.concatenate([seg[:2] + s * v, seg[2:] + s * v])


def _shifted(seg, d):
    """The segment moved by d pixels along its normal (a parallel line at distance d)."""
    n = _unit(seg[2:] - seg[:2])[::-1] * np.array([-1.0, 1.0])
    return np.concatenate([seg[:2] + d * n, seg[2:] + d * n])


def _smart_angle(bio):
    """The angle threshold of LineLinker2d::compute_score_smartangle at bi-overlap `bio` < th_smartoverlap."""
    ratio = min((SMART_OVERLAP - bio) / (SMART_OVERLAP - L2D["th_overlap"]), 1.0)
    return L2D["th_angle"] - ratio * (L2D["th_angle"] - SMART_ANGLE)


def _l2d_row(g, dec, dl, sgn, kind):
    """Candidate A is the source line itself; the segment of view b is its projection, moved so that one 2D sub-test
    between the two lands on its threshold: turned about its midpoint (angle), slid along its line (overlap), moved
    parallel (perpendicular distance), slid to a bi-overlap below th_smartoverlap and turned (smart angle)."""
    # short segments where view b's segment is turned: its triangulated line B stays close to A
    S, E, *_ = _base_line(g.rng, g.C0, g.fwd, g.depth, (g.Ca, g.Cb), half=0.05 if kind in ("angle", "smart") else 0.25)
    a = _seg_ref(g.cams[2], S, E)  # what the reference computes from A
    f = 1 + sgn * dl
    if kind == "angle":
        b, fails = _rotated(a, dec * f), sgn > 0
    elif kind == "overlap":
        b, fails = _slid(a, 1.0 - L2D["th_overlap"] * f), sgn < 0  # bi-overlap 1 - s, accepted when > th_overlap
    elif kind == "perp":
        b, fails = _shifted(a, L2D["th_perp"] * f), sgn > 0
    else:  # smart angle at bi-overlap ~dec: the angle at which angle == smart threshold(bio(angle)) * f
        b0 = _slid(a, 1.0 - dec)
        lo, hi = 0.0, L2D["th_angle"]
        for _ in range(200):
            phi = 0.5 * (lo + hi)
            if phi < _smart_angle(_bioverlap(a, _rotated(b0, phi))) * f:
                lo = phi
            else:
                hi = phi
        b, fails = _rotated(b0, 0.5 * (lo + hi)), sgn > 0
        assert L2D["th_overlap"] < _bioverlap(a, b) < SMART_OVERLAP
    return _seg_px(g.cams[0], S, E), _seg_px(g.cams[1], S, E), b, fails


def _fullscore_row(g, dec, dl, sgn):
    """The 3D angle at which the pair score exp(-(angle / (th_angle mult))^2 / 2) = 0.5^((angle / th_angle)^2) equals
    fullscore_th * (1 + sgn dl). Below fullscore_th the node has no valid connection."""
    th_angle = 10.0
    S, E, rs, re_, lam_s, lam_e = _base_line(g.rng, g.C0, g.fwd, g.depth, (g.Ca, g.Cb))
    angle = th_angle * np.sqrt(np.log(FULLSCORE_TH * (1 + sgn * dl)) / np.log(0.5))
    EB = _end_at_angle(g.C0, S, E, re_, lam_e, angle)
    return _seg_px(g.cams[0], S, E), _seg_px(g.cams[1], S, E), _seg_px(g.cams[2], S, EB), sgn < 0


# name -> (outcome kind, configuration, rows, row builder)
PLANTED = {
    "tri_angle_1": ("cand", _phase_a_cfg(line_tri_angle_threshold=1.0, sensitivity_threshold=90.0),
                    _rows(("start", "end"), TRI_ANGLE_DELTAS), lambda g, *r: _tri_angle_row(g, *r, th=1.0)),
    "tri_angle_5": ("cand", _phase_a_cfg(line_tri_angle_threshold=5.0, sensitivity_threshold=90.0),
                    _rows(("start", "end"), TRI_ANGLE_DELTAS), lambda g, *r: _tri_angle_row(g, *r, th=5.0)),
    "iou": ("cand", _phase_a_cfg(IoU_threshold=IOU_TH), _rows(("iou",), IOU_DELTAS), _iou_row),
    "iou_grazing": ("cand", _phase_a_cfg(IoU_threshold=IOU_TH, line_tri_angle_threshold=0.0),
                    _rows(GRAZING_ANGLES, GRAZING_DELTAS), _grazing_row),
    "sensitivity": ("cand", _phase_a_cfg(sensitivity_threshold=SENSITIVITY_TH, line_tri_angle_threshold=0.0),
                    _rows(("sensitivity",), DELTAS), _sensitivity_row),
    # the 2D angle with the bi-overlap ~1 >= th_smartoverlap; th_angle 20 is above the 14.4775 deg switch of angle2_deg
    "l2d_angle_5": ("score", _l2d_cfg(use_perp=False), _rows((5.0,), DELTAS), lambda g, *r: _l2d_row(g, *r, "angle")),
    "l2d_angle_20": ("score", _l2d_cfg(use_perp=False, th_angle=20.0), _rows((20.0,), DELTAS),
                     lambda g, *r: _l2d_row(g, *r, "angle")),
    # IoU <= bi-overlap for a collinear pair: IoU_threshold 0.01 lets the rows through phase A
    "l2d_overlap": ("score", _l2d_cfg(iou=0.01, use_angle=False, use_perp=False), _rows(("overlap",), DELTAS),
                    lambda g, *r: _l2d_row(g, *r, "overlap")),
    "l2d_smartangle": ("score", _l2d_cfg(iou=0.01, use_perp=False), _rows(SMART_BIO, DELTAS),
                       lambda g, *r: _l2d_row(g, *r, "smart")),
    "l2d_perp": ("score", _l2d_cfg(use_angle=False, use_overlap=False), _rows(("perp",), DELTAS),
                 lambda g, *r: _l2d_row(g, *r, "perp")),
    "l2d_perp_all": ("score", _l2d_cfg(), _rows(("perp",), DELTAS), lambda g, *r: _l2d_row(g, *r, "perp")),
    "fullscore": ("valid", dict(boundary_3d_cfg("angle_10"), fullscore_th=FULLSCORE_TH), _rows(("fullscore",), DELTAS),
                  _fullscore_row),
}


def planted_score_tol(name):
    """Bar on the scores against the reference's stored outputs: 1e-9, and 1e-8 for iou_grazing, whose rows are
    triangulated from planes ~1e-3 deg apart; rounding there moves the endpoints by ~1e-11 and the scores by ~1e-9."""
    return 1e-8 if name == "iou_grazing" else 1e-9


def planted_golden(name):
    """File name (tests/golden/ref) of the reference's outputs on family `name`."""
    kind = PLANTED[name][0]
    return {"cand": "boundary_phase_a_", "score": "boundary_2d_", "valid": "boundary_phase_c_"}[kind] + name


def planted_cfg(name, **kw):
    return dict(PLANTED[name][1], **kw)


def planted_scene(name, seed=701):
    """(scene, planted) with planted = [(node index, decision, delta, sign, whether the planted test must fail)]."""
    from types import SimpleNamespace
    _, _, rows, build = PLANTED[name]
    rng = np.random.default_rng(seed)
    kvec, qvec, tvec, segs, line_off, planted, matches = [], [], [], [], [0], [], {}
    for depth, origin in GEOMETRIES:
        C0, fwd, Ca, Cb, cams = _group(rng, depth, origin)
        g = SimpleNamespace(rng=rng, depth=depth, C0=C0, fwd=fwd, Ca=Ca, Cb=Cb, cams=cams)
        ls, la, lb = [], [], []
        for k, (dec, dl, sgn) in enumerate(rows):
            s0, sa, sb, fails = build(g, dec, dl, sgn)
            ls.append(s0); la.append(sa); lb.append(sb)
            planted.append((int(line_off[-1]) + k, dec, dl, sgn, bool(fails)))
        _add_group(K_ALL, cams, (ls, la, lb), kvec, qvec, tvec, segs, line_off, matches)
    return _assemble(kvec, qvec, tvec, segs, line_off, matches, (np.full(3, -1e7), np.full(3, 1e7))), planted


def check_planted_family(name, t, sc, planted):
    """Every planted decision of family `name` as intended in triangulator `t` (see the kinds above)."""
    kind = PLANTED[name][0]
    for node, dec, dl, sgn, fails in planted:
        v = int(np.searchsorted(sc.line_off, node, "right") - 1)
        img, l = int(sc.img_ids[v]), int(node - sc.line_off[v])
        cl, cng = t.get_cands_node(img, l)
        views = np.asarray(cng).reshape(-1, 2)[:, 0]
        row = (node, dec, dl, sgn, fails)
        if kind == "cand":  # the row into view b always yields its candidate; the row into view a only if it passes
            assert (views == sc.img_ids[v + 2]).sum() == 1, row
            assert (views == sc.img_ids[v + 1]).sum() == (0 if fails else 1), row
            continue
        assert len(views) == 2, row
        if kind == "score":
            s = float(cl[0, 9])
            assert (s == 0.0) if fails else (s >= SCORE_TH), (row, s)
        else:
            off, _ = t.get_valid_edges(img)
            assert (off[l + 1] == off[l]) == fails, (row, off[l + 1] - off[l])


def checked_planted_scene(name):
    """planted_scene, with every planted decision asserted through the oracle."""
    from oracle.oracle import OracleTri
    sc, planted = planted_scene(name)
    check_planted_family(name, _feed(OracleTri(planted_cfg(name), threads=1), sc), sc, planted)
    return sc, planted


def unlabelled_vps(sc, seed=5):
    """VP results in which every line is unlabelled (-1): the VP instantiations of the node kernel run the same rows
    without adding a proposal."""
    from limap_b200.vplib import VPResult
    rng = np.random.default_rng(seed)
    out = {}
    for v, i in enumerate(sc.img_ids):
        vps = rng.normal(size=(3, 3))
        labels = -np.ones(int(sc.line_off[v + 1] - sc.line_off[v]), np.int32)
        out[int(i)] = VPResult(labels, vps / np.linalg.norm(vps, axis=1, keepdims=True))
    return out
