"""Seeded inputs of the localization line-matching tests (tests/test_loc_matching_*.py, tests/golden/make_locmatch_golden.py).

A case is a small localization set: database images and query images (SIMPLE_PINHOLE and PINHOLE cameras around a box
of 3D map lines), the database lines with their track ids (line2track, -1 untracked), the map's track lines, the
retrieval lists and learned-matcher style 2D-2D pairs (duplicates, unsorted). Query poses are the true ones turned by
2 degrees and shifted by 5 cm. Special lines: a zero-length database line, a query line starting one pixel from the
epipole of a database camera, a query image and a database image without lines, a database image without tracked lines. The
"planted" case adds database lines whose epipolar IoU with a query line lies at th -/+ 1e-5, 1.5e-7, 5e-8, 1e-11,
1e-13 and 2e-15 for each threshold of THRESHOLDS, slid into place along their own line by bisection on boundary_scenes'
epipolar IoU (its planting helper, over slides up to twice the segment's length so that IoU 0 - delta is reachable). The
last three offsets lie inside the band in which the kernel switches to the reference's normalised form, the last two
below the fast form's own error."""
import numpy as np

import boundary_scenes as bs

THRESHOLDS = (0.0, 0.1, 0.2, 0.5)
PLANT_DELTAS = (1e-5, 1.5e-7, 5e-8, 1e-11, 1e-13, 2e-15)
PLANT_THRESHOLDS = THRESHOLDS
REPROJ_FUNCS = ("Perpendicular", "Midpoint", "Midpoint_Perpendicular")


def _turn(q, t, rng, deg=2.0, trans=0.05):
    from limap_b200.synth import _quat_mul
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    h = np.deg2rad(deg) / 2
    dq = np.r_[np.cos(h), axis * np.sin(h)]
    return _quat_mul(dq[None], np.asarray(q)[None])[0], np.asarray(t) + rng.normal(size=3) * trans


def _proj(kvec, R, t, X):
    h = R @ X + t
    return np.array([kvec[0] * h[0] / h[2] + kvec[2], kvec[1] * h[1] / h[2] + kvec[3]])


def _cam(model, kvec, q, t):
    return np.r_[model, kvec, q, t].astype(np.float64)


def make_case(seed=0, n_db=6, n_q=3, n_tracks=40, clutter=8, planted=False, empty_images=True):
    rng = np.random.default_rng(seed)
    S = rng.uniform(-1, 1, (n_tracks, 3))
    E = S + rng.normal(size=(n_tracks, 3)) * 0.6
    tracks = np.concatenate([S, E], 1)
    cams, lines, line2track, names = {}, {}, {}, {}
    db_ids = list(range(n_db))
    q_ids = list(range(100, 100 + n_q))
    true_pose = {}
    for k, img in enumerate(db_ids + q_ids):
        ang = 2 * np.pi * k / (n_db + n_q)
        C = np.array([4 * np.cos(ang), 4 * np.sin(ang), rng.uniform(-0.5, 0.5)])
        q, t, R = bs._look_at(C, rng.normal(size=3) * 0.2, rng)
        model = k % 2
        kvec = bs.K_ALL.copy() if model == 0 else np.array([bs.K_ALL[0] * 1.05, bs.K_ALL[0] * 0.97, 410.0, 290.0])
        true_pose[img] = (q, t, R)
        segs, trk = [], []
        for tid in range(n_tracks):
            if rng.random() < 0.25:
                continue
            a, b = rng.uniform(0, 0.15), rng.uniform(0.85, 1.0)
            X0, X1 = S[tid] + a * (E[tid] - S[tid]), S[tid] + b * (E[tid] - S[tid])
            segs.append(np.r_[_proj(kvec, R, t, X0), _proj(kvec, R, t, X1)] + rng.normal(size=4) * 0.5)
            trk.append(tid if rng.random() < 0.6 else -1)
        for _ in range(clutter):
            segs.append(rng.uniform([0, 0, 0, 0], [800, 600, 800, 600]))
            trk.append(-1)
        if img in q_ids:
            q, t = _turn(q, t, rng)
        cams[img] = _cam(model, kvec, q, t)
        lines[img] = np.array(segs, np.float64).reshape(-1, 4)
        line2track[img] = np.array(trk, np.int64)
        names[img] = f"img_{img:04d}.png"
    # special lines
    lines[db_ids[0]][0, 2:] = lines[db_ids[0]][0, :2]                       # zero length: IoU NaN, never matches
    Cdb = -true_pose[db_ids[1]][2].T @ true_pose[db_ids[1]][1]
    qk = cams[q_ids[0]]
    from limap_b200.base import _quat_to_R
    Rq = _quat_to_R(qk[5:9])
    # a query endpoint one pixel from the epipole of db_ids[1]: at the epipole itself F x is rounding noise in every form
    lines[q_ids[0]][0, :2] = _proj(qk[1:5], Rq, qk[9:12], Cdb) + np.array([0.6, 0.8])
    line2track[db_ids[2]][:] = -1                                          # a target without tracked lines
    if empty_images:
        lines[db_ids[3]] = np.zeros((0, 4))                                # a target without lines
        line2track[db_ids[3]] = np.zeros(0, np.int64)
        if n_q > 2:
            lines[q_ids[2]] = np.zeros((0, 4))                             # a query without lines
    if planted:
        _plant(cams, lines, line2track, tracks, q_ids[1], db_ids[4], true_pose, rng)
    retrieval = {q: list(rng.permutation([d for d in db_ids])[: max(2, n_db - 1)]) for q in q_ids}
    retrieval[q_ids[0]] = [db_ids[0], db_ids[1], db_ids[2], db_ids[3]] + retrieval[q_ids[0]][:1]
    retrieval[q_ids[1]] = [db_ids[4]] + [d for d in retrieval[q_ids[1]] if d != db_ids[4]]
    pairs = {}
    for q in q_ids:
        pairs[q] = {}
        for d in retrieval[q]:
            nq, nd = len(lines[q]), len(lines[d])
            m = rng.integers(0, 3 * max(nq, 1)) if nq and nd else 0
            p = np.stack([rng.integers(0, max(nq, 1), m), rng.integers(0, max(nd, 1), m)], 1) if m else np.zeros((0, 2))
            if m > 3:
                p = np.concatenate([p, p[:3]])                             # duplicates
            pairs[q][d] = [tuple(map(int, x)) for x in p]
    return dict(cams=cams, lines=lines, line2track=line2track, tracks=tracks, retrieval=retrieval, pairs=pairs,
                db_ids=db_ids, q_ids=q_ids, names=names)


def _slide_to_iou(l1, cam1, seg, cam2, iou):
    """boundary_scenes._slide_to_iou over slides in [0, 2]: the IoU falls from 1 at no slide below 0 past one length."""
    v = seg[2:] - seg[:2]
    lo, hi = 0.0, 2.0
    for _ in range(200):
        s = 0.5 * (lo + hi)
        if bs._epipolar_iou(l1, cam1, np.concatenate([seg[:2] + s * v, seg[2:] + s * v]), cam2) > iou:
            lo = s
        else:
            hi = s
    s = 0.5 * (lo + hi)
    return np.concatenate([seg[:2] + s * v, seg[2:] + s * v])


def _plant(cams, lines, line2track, tracks, qid, did, true_pose, rng):
    """Database lines of did whose epipolar IoU with query line 1 of qid is th -/+ delta, tracked. The two views are
    rebuilt on K_ALL (SIMPLE_PINHOLE), as the planting helper evaluates them."""
    qk = cams[qid]
    cams[qid] = _cam(0, bs.K_ALL, qk[5:9], qk[9:12])
    dk = cams[did]
    cams[did] = _cam(0, bs.K_ALL, dk[5:9], dk[9:12])
    from limap_b200.base import _quat_to_R
    cq = (cams[qid][5:9], cams[qid][9:12], _quat_to_R(cams[qid][5:9]))
    cd = (cams[did][5:9], cams[did][9:12], _quat_to_R(cams[did][5:9]))
    tid = 0
    S, E = tracks[tid, :3], tracks[tid, 3:]
    l1 = bs._seg_ref(cq, S, E)
    lines[qid][1] = l1
    seg = bs._seg_px(cd, S, E)
    new, trk = [], []
    for th in PLANT_THRESHOLDS:
        for dl in PLANT_DELTAS:
            for sgn in (-1, 1):
                new.append(_slide_to_iou(l1, cq, seg, cd, th + sgn * dl))
                trk.append(tid)
    lines[did] = np.concatenate([lines[did], np.array(new)])
    line2track[did] = np.concatenate([line2track[did], np.array(trk, np.int64)])

