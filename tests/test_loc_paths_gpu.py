"""The query pose refinement (loc_refine_kernel) step by step against the oracle (oracle/orc_loc.cpp): the initial cost
of every cost x weight x loss, single-block queries on the block edges of tests/test_loc_block_host.py, the trajectory
after 1..10 iterations against a share and a spread calibrated on the oracle itself, the solver's exits (zero gradient,
too many invalid steps, a failed first evaluation) and the usability bit they decide, non-unit start quaternions,
empty groups and the lane stride of the block loop.

The trajectory bar is calibrated in each test: the oracle is run against itself with the start tvec moved by one ulp.
The share of queries whose (iterations, successful, flags) then agree, and the largest difference in x among them,
measure how far the last-bit decisions of these queries reach; the device, which differs from the oracle in FMA
contraction, summation order and L D L^T against L L^T, must agree as often up to a binomial slack and as closely up
to SPREAD_FACTOR."""
import os
import sys

import numpy as np
import pytest

from limap_b200 import synth
from limap_b200 import hybrid_localization as hl
from oracle import localization as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_loc_block_host as hb  # noqa: E402

pytestmark = pytest.mark.gpu

CF = range(6)
WF = range(5)
KS = (1, 2, 3, 5, 10)
DBL_MAX = np.finfo(np.float64).max
# Initial cost: a sum of non-negative terms, each the same expression on both sides up to FMA contraction, so the
# summation order bounds the relative error by about n u (n <= 100 blocks here). Measured on an H100 (700 W power
# limit): <= 7.9e-13. The point-to-ray residual sqrt(|d|^2 - (d . dir)^2 + 1e-8) cancels |d|^2 ~ 25 m^2 down to a
# squared distance ~1e-4 m^2, so its terms carry ~u |d|^2 / s ~ 1e-11 relative each: measured <= 1.3e-12 in the sum.
COST0_TOL = 1e-12
COST0_TOL_POINT_TO_RAY = 1e-11
# Single-block costs, relative to max(cost, 1). The blocks differ by FMA contraction only, but a single block has no
# sum to average its rounding: measured on an H100 <= 2.5e-11 over the stored reference evaluations.
BLOCK_COST_TOL = 1e-10
# ... except exp(10 acos(cos)) at cos = 1 - 5e-13: acos there is ~1e-6, and a rounding of 1e-16 in cos moves it by
# 1e-10, so the weight carries ~1e-9 relative (measured 8.9e-9).
BLOCK_COST_TOL_ACOS_EDGE = 1e-7
# The device's share of queries on the oracle's path may fall short of the oracle's own one-ulp share p by three
# binomial standard deviations sqrt(p (1 - p) / Q) plus one query. After 10 iterations these small queries have
# converged and stop on last-bit exits, so p is 0.4-0.95 there: measured on an H100, the device fell short by at most
# 0.16 (p = 0.47, Q = 64; the slack is 0.20 there) and by at most one query where p = 1. Its spread in x may exceed the
# oracle's own by SPREAD_FACTOR, above a floor of 1e-15: measured at most 34x up to 5 iterations and 8e2x after 10.
SPREAD_FACTOR = 1e4
SPREAD_FLOOR = 1e-15


def _share_slack(p, Q):
    return 3.0 * np.sqrt(p * (1.0 - p) / Q) + 1.0 / Q


def _cfg(cf=2, wf=0, loss=0, scale=1.0, p3=None, iters=100, wp=1.0, wl=1.0, invalid=10):
    p3 = cf in (4, 5) if p3 is None else p3
    return dict(cost_function=cf, weight_function=wf, loss_kind=loss, loss_scale=scale, points_3d_dist=p3,
                max_num_iterations=iters, weight_point=wp, weight_line=wl, max_num_consecutive_invalid_steps=invalid)


KEYS = ("kvec", "qvec", "tvec", "pt_off", "p3d", "p2d", "grp_off", "l3d", "l2d_off", "l2d")


def _gpu(arrs, c):
    cfg = hl._cabi.LocConfig(c["cost_function"], c["weight_function"], c["loss_kind"], int(c["points_3d_dist"]),
                             c["loss_scale"], c["weight_point"], c["weight_line"], c["max_num_iterations"],
                             c["max_num_consecutive_invalid_steps"])
    return hl.loc_solve_arrays({k: arrs[k] for k in KEYS}, cfg)


def _orc(arrs, c):
    return orc.solve({k: arrs[k] for k in KEYS}, **c)


def _small(seed, **kw):
    base_kw = dict(Q=64, P=40, G=12, seed=seed, noise_px=1.0, outlier_frac=0.1)
    base_kw.update(kw)
    return synth.make_loc_queries(**base_kw)


# ---- per-query lists <-> lm_loc_solve arrays --------------------------------------------------------------------------
def _unpack(a):
    """Per-query dicts: kvec, qvec, tvec, groups [(l3d[6], l2d[n][4])], p3d, p2d."""
    out = []
    for q in range(len(a["kvec"])):
        g0, g1 = a["grp_off"][q], a["grp_off"][q + 1]
        groups = [(a["l3d"][g], a["l2d"][a["l2d_off"][g]:a["l2d_off"][g + 1]]) for g in range(g0, g1)]
        p0, p1 = a["pt_off"][q], a["pt_off"][q + 1]
        out.append(dict(kvec=a["kvec"][q], qvec=a["qvec"][q], tvec=a["tvec"][q], groups=groups, p3d=a["p3d"][p0:p1],
                        p2d=a["p2d"][p0:p1]))
    return out


def _pack(queries):
    groups = [g for q in queries for g in q["groups"]]
    cat = lambda k, w: np.concatenate([np.reshape(q[k], (-1, w)) for q in queries]) if queries else np.zeros((0, w))
    return dict(kvec=cat("kvec", 4), qvec=cat("qvec", 4), tvec=cat("tvec", 3),
                pt_off=np.r_[0, np.cumsum([np.size(q["p3d"]) // 3 for q in queries])].astype(np.int64),
                p3d=cat("p3d", 3), p2d=cat("p2d", 2),
                grp_off=np.r_[0, np.cumsum([len(q["groups"]) for q in queries])].astype(np.int64),
                l3d=np.reshape([g[0] for g in groups], (-1, 6)),
                l2d_off=np.r_[0, np.cumsum([np.size(g[1]) // 4 for g in groups])].astype(np.int64),
                l2d=np.concatenate([np.reshape(g[1], (-1, 4)) for g in groups]) if groups else np.zeros((0, 4)))


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("qvec", "tvec", "iters", "cost", "flags"))


# ---- initial cost -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cf", CF)
def test_initial_cost_every_weight_and_loss(cf):
    """max_num_iterations = 0: cost[:, 0] is one evaluation of every block at the start; the solve ends on the
    iteration limit (usable), with x bit-unchanged."""
    a = _small(200 + cf)
    worst = 0.0
    for wf in WF:
        for loss, scale in ((0, 1.0), (1, 2.0), (2, 1.5), (3, 1.0)):
            for p3 in (False, True):
                c = _cfg(cf, wf, loss, scale, p3=p3, iters=0)
                g, o = _gpu(a, c), _orc(a, c)
                assert (o["term"] == 1).all()
                assert (g["flags"] == 3).all() and (g["iters"] == 0).all()
                assert np.array_equal(g["qvec"], a["qvec"]) and np.array_equal(g["tvec"], a["tvec"])
                assert np.array_equal(g["cost"][:, 0], g["cost"][:, 1])
                err = np.abs(g["cost"][:, 0] - o["cost"][:, 0]) / o["cost"][:, 0]
                worst = max(worst, err.max())
                assert err.max() <= (COST0_TOL_POINT_TO_RAY if p3 else COST0_TOL), (wf, loss, p3, err.max())
    print(f"cf={cf}: initial cost, largest relative difference {worst:.2e}")


# ---- single-block queries ---------------------------------------------------------------------------------------------
def _line_queries(data, kvec, q, t):
    """One query per line block: one 3D line with one 2D line (ScaledLoss factor a = 1), no points."""
    return _pack([dict(kvec=kvec[i], qvec=q[i], tvec=t[i], groups=[(data[i, :6], data[i, 6:10])], p3d=np.zeros((0, 3)),
                       p2d=np.zeros((0, 2))) for i in range(len(data))])


def _point_queries(data, kvec, q, t):
    return _pack([dict(kvec=kvec[i], qvec=q[i], tvec=t[i], groups=[], p3d=data[i, :3], p2d=data[i, 3:5])
                  for i in range(len(data))])


def _block_cost(arrs, c, res_ref, tol=BLOCK_COST_TOL):
    """The device's cost[:, 0] of single-block queries against 1/2 |r|^2 of the reference's residuals and against the
    oracle."""
    g, o = _gpu(arrs, c), _orc(arrs, c)
    ref = 0.5 * (res_ref * res_ref).sum(1)
    fin = np.isfinite(ref)
    assert np.array_equal(g["cost"][~fin, 0], np.full((~fin).sum(), DBL_MAX))
    assert (o["term"][~fin] == 7).all() and (g["flags"][~fin] == 1).all()
    e1 = (np.abs(g["cost"][fin, 0] - ref[fin]) / np.maximum(ref[fin], 1.0)).max(initial=0)
    e2 = (np.abs(g["cost"][:, 0] - o["cost"][:, 0]) / np.maximum(o["cost"][:, 0], 1.0)).max(initial=0)
    print(f"single blocks cf={c['cost_function']} wf={c['weight_function']}: {e1:.2e} {e2:.2e}")
    assert e1 <= tol and e2 <= tol, (e1, e2)
    return g, o


def test_single_block_queries_reference_values():
    """Every stored reference evaluation as a query of its own (tests/golden/ref/localization.npz)."""
    G = hb.G
    for cf in CF:
        for wf in WF:
            idx = np.flatnonzero((G["kind"] == 0) & (G["cf"] == cf) & (G["wf"] == wf))
            arrs = _line_queries(G["data"][idx], G["kvec"][idx], G["qvec"][idx], G["tvec"][idx])
            _block_cost(arrs, _cfg(cf, wf, iters=0), G["res"][idx])
    for use3d in (0, 1):
        idx = np.flatnonzero((G["kind"] == 1) & (G["use3d"] == use3d))
        arrs = _point_queries(G["data"][idx], G["kvec"][idx], G["qvec"][idx], G["tvec"][idx])
        _block_cost(arrs, _cfg(2, 0, p3=bool(use3d), iters=0), G["res"][idx])


def test_single_block_queries_planted_edges():
    rng = np.random.default_rng(41)
    for rel in (1e-4, -1e-4):  # line_line_dist either side of n2 = 1e-8
        d = hb._line_along_ray(rng, 64, rel)
        _block_cost(_line_queries(*d), _cfg(4, 0, iters=0), hb.oracle_block(4, 0, False, 0, *d)[0])
    for perpendicular, cfs in ((False, ((0, 1), (0, 2))), (True, ((1, 0), (3, 0), (2, 1)))):  # sine / cosine near 1
        d = hb._on_projected_line(rng, 64, perpendicular)
        for cf, wf in cfs:
            _block_cost(_line_queries(*d), _cfg(cf, wf, iters=0), hb.oracle_block(cf, wf, False, 0, *d)[0],
                        BLOCK_COST_TOL_ACOS_EDGE if wf == 2 else BLOCK_COST_TOL)
    d = hb.random_lines(rng, 64)
    d[0][:, 3:6] = hb.backproject(d[1], d[2], d[3], rng.uniform(0, 640, 64), rng.uniform(0, 480, 64),
                                  -rng.uniform(1, 6, 64))  # ending behind the camera
    for cf in CF:
        _block_cost(_line_queries(*d), _cfg(cf, 1, iters=0), hb.oracle_block(cf, 1, False, 0, *d)[0])
    # a zero-length 2D line alone in its group: a = 0 / 0, the first evaluation fails (term 7) whatever the cost
    d = hb.random_lines(rng, 16)
    d[0][:, 8:10] = d[0][:, 6:8]
    for cf in CF:
        _block_cost(_line_queries(*d), _cfg(cf, 0, iters=0), np.full((16, 2), np.nan))
    # a point on the camera plane: non-finite reprojection (term 7), finite point-to-ray distance
    n = 16
    kvec, _, _ = hb.random_poses(rng, n)
    q, t = np.tile([1.0, 0, 0, 0], (n, 1)), np.zeros((n, 3))
    data = np.zeros((n, 10))
    data[:, :2], data[:, 3:5] = rng.normal(size=(n, 2)), rng.uniform(0, 480, (n, 2))
    for use3d in (False, True):
        _block_cost(_point_queries(data, kvec, q, t), _cfg(2, 0, p3=use3d, iters=0),
                    hb.oracle_block(2, 0, use3d, 1, data, kvec, q, t)[0])


# ---- trajectory -------------------------------------------------------------------------------------------------------
def _path(r):
    return np.concatenate([r["iters"], r["flags"][:, None].astype(np.int32)], 1)


def _spread(a, b, same):
    dq = np.minimum(np.abs(a["qvec"] - b["qvec"]).max(1), np.abs(a["qvec"] + b["qvec"]).max(1))
    return max(dq[same].max(initial=0), np.abs(a["tvec"] - b["tvec"]).max(1)[same].max(initial=0))


def _calibrated(arrs, c, label):
    """The device against the oracle, with the bars taken from the oracle against itself one ulp away."""
    o = _orc(arrs, c)
    moved = dict(arrs, tvec=np.nextafter(arrs["tvec"], np.inf))
    o1 = _orc(moved, c)
    same_self = (_path(o) == _path(o1)).all(1)
    share_self, spread_self = same_self.mean(), _spread(o, o1, same_self)
    g = _gpu(arrs, c)
    same = (_path(g) == _path(o)).all(1)
    share, spread = same.mean(), _spread(g, o, same)
    print(f"{label}: share {share:.3f} (oracle one ulp away {share_self:.3f}), spread {spread:.2e} "
          f"(oracle {spread_self:.2e})")
    assert share >= share_self - _share_slack(share_self, len(same)), (label, share, share_self)
    assert spread <= SPREAD_FACTOR * max(spread_self, SPREAD_FLOOR), (label, spread, spread_self)
    return g, o


@pytest.mark.parametrize("cf", CF)
def test_trajectory_every_cost_and_weight(cf):
    for wf in WF:
        a = _small(300 + 10 * cf + wf)
        for k in KS:
            _calibrated(a, _cfg(cf, wf, iters=k), f"cf={cf} wf={wf} k={k}")


@pytest.mark.parametrize("loss,scale", [(1, 2.0), (2, 1.5), (3, 1.0), (3, 0.1)])
def test_trajectory_robust_losses(loss, scale):
    a = _small(400 + loss)
    for cf in (0, 2, 4):
        for k in KS:
            _calibrated(a, _cfg(cf, 0, loss, scale, iters=k), f"loss={loss}({scale}) cf={cf} k={k}")


def test_trajectory_units_of_1000px_and_odd_batches():
    big = synth.make_loc_queries(Q=64, P=40, G=12, seed=41, noise_px=1.0, scale=1000.0)
    for cf in (2, 4, 5):
        for k in KS:
            _calibrated(big, _cfg(cf, 0, iters=k), f"1000 px cf={cf} k={k}")
    for Q in (1, 3, 67):  # not a multiple of the four warps per CTA
        a = _small(500 + Q, Q=Q)
        for k in (1, 3, 10):
            _calibrated(a, _cfg(2, 1, 3, 1.0, iters=k), f"Q={Q} k={k}")


# ---- exits and usability ----------------------------------------------------------------------------------------------
def _points_only(seed, Q=16):
    a = _small(seed, Q=Q)
    return synth.loc_subset(a, np.ones(len(a["p3d"]), bool), np.zeros(len(a["l2d"]), bool))


def test_exit_zero_gradient():
    """weight_point = 0: the ScaledLoss factor zeroes J and g, so the solve stops on the gradient test before its first
    iteration (term 3): usable, zero iterations, x unchanged."""
    a = _points_only(601)
    c = _cfg(2, 0, wp=0.0)
    g, o = _gpu(a, c), _orc(a, c)
    assert (o["term"] == 3).all() and (o["flags"] == 3).all()
    assert (g["flags"] == 3).all() and (g["iters"] == 0).all() and (g["cost"] == 0).all()
    assert np.array_equal(g["qvec"], a["qvec"]) and np.array_equal(g["tvec"], a["tvec"])


@pytest.mark.parametrize("invalid", [10, 1])
def test_exit_invalid_steps(invalid):
    """weight_point = 1e-200: g ~ 1e-198 and the step ~ 1e-188, so the model cost change step . g underflows to 0 and
    every step is invalid; after max_num_consecutive_invalid_steps of them the solve ends unusable (term 4)."""
    a = _points_only(602)
    c = _cfg(2, 0, wp=1e-200, invalid=invalid)
    g, o = _gpu(a, c), _orc(a, c)
    assert (o["term"] == 4).all() and (o["flags"] == 1).all()
    assert (g["flags"] == 1).all()
    assert (g["iters"][:, 0] == invalid).all() and (g["iters"][:, 1] == 0).all()
    assert np.array_equal(g["iters"], o["iters"])
    assert np.array_equal(g["qvec"], a["qvec"]) and np.array_equal(g["tvec"], a["tvec"])


def test_exit_failed_first_evaluation():
    """A point on the camera plane (z = 0, reprojection 1 / 0) among ordinary points, or a group whose 2D lines all
    have zero length (a = 0 / 0): the first evaluation is not finite (term 7), the result is unusable, cost[:, 0] is
    DBL_MAX and x is unchanged. Queries without such a block in the same batch are unaffected."""
    a = _small(603, Q=8)
    qs = _unpack(a)
    for i in (0, 2, 4):  # a camera-plane point: world = camera frame, bit for bit
        qs[i] = dict(qs[i], qvec=np.array([1.0, 0, 0, 0]), tvec=np.zeros(3))
        qs[i]["p3d"] = np.r_[qs[i]["p3d"][:5], [[0.3, -0.2, 0.0]], qs[i]["p3d"][5:]]
        qs[i]["p2d"] = np.r_[qs[i]["p2d"][:5], [[320.0, 240.0]], qs[i]["p2d"][5:]]
    for i in (1, 5):  # a group of two zero-length 2D lines
        l2 = qs[i]["groups"][3][1].copy()
        l2 = np.r_[l2[:1], l2[:1]]
        l2[:, 2:] = l2[:, :2]
        qs[i]["groups"] = qs[i]["groups"][:3] + [(qs[i]["groups"][3][0], l2)] + qs[i]["groups"][4:]
    arrs = _pack(qs)
    bad = np.array([0, 1, 2, 4, 5])
    for cf, p3 in ((2, False), (0, False), (4, False)):
        c = _cfg(cf, 0, 3, 1.0, p3=p3, iters=5)
        g, o = _gpu(arrs, c), _orc(arrs, c)
        assert (o["term"][bad] == 7).all() and (o["term"][[3, 6, 7]] != 7).all()
        assert (g["flags"][bad] == 1).all() and (g["flags"][[3, 6, 7]] == 3).all()
        assert (g["cost"][bad] == DBL_MAX).all() and (g["iters"][bad] == 0).all()
        assert np.array_equal(g["qvec"][bad], arrs["qvec"][bad]) and np.array_equal(g["tvec"][bad], arrs["tvec"][bad])
        alone = _gpu(_pack([qs[i] for i in (3, 6, 7)]), c)
        for k in ("qvec", "tvec", "iters", "cost", "flags"):
            assert np.array_equal(alone[k], g[k][[3, 6, 7]]), k


# ---- start poses and layouts ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("qnorm", [0.5, 2.0, 1.0 + 1e-8])
def test_non_unit_start_quaternions(qnorm):
    """WorldToPixel normalises q; PixelToWorld uses the unnormalised conjugate (CF 4, 5 and point-to-ray)."""
    a = _small(700)
    a = dict(a, qvec=a["qvec"] * qnorm)
    for cf in CF:
        for p3 in (False, True):
            for k in (1, 3):
                _calibrated(a, _cfg(cf, 0, p3=p3, iters=k), f"|q|={qnorm} cf={cf} p3={p3} k={k}")


def test_empty_groups():
    """3D lines with no 2D line before, between and after the others, and a query whose groups are all empty but which
    has points: the block order is that of the same queries without them, so the results are bit-identical."""
    a = _small(800, Q=8)
    qs = _unpack(a)
    rng = np.random.default_rng(8)
    empty = lambda: (rng.normal(size=6), np.zeros((0, 4)))
    with_empty = [dict(q) for q in qs]
    with_empty[0]["groups"] = [empty(), empty()] + qs[0]["groups"]
    with_empty[1]["groups"] = qs[1]["groups"][:4] + [empty()] + qs[1]["groups"][4:7] + [empty(), empty()] + \
        qs[1]["groups"][7:]
    with_empty[2]["groups"] = qs[2]["groups"] + [empty()]
    with_empty[3]["groups"] = [empty(), empty(), empty()]  # points only
    no_lines = [dict(q) for q in qs]
    no_lines[3]["groups"] = []
    with_empty[5]["groups"] = [empty()] + qs[5]["groups"][:1] + [empty()] + qs[5]["groups"][1:] + [empty()]
    A, B = _pack(with_empty), _pack(no_lines)
    assert len(A["l3d"]) == len(B["l3d"]) + 12 and np.array_equal(A["l2d"], B["l2d"])
    for cf in (2, 4):
        c = _cfg(cf, 1, 3, 1.0, iters=10)
        g, h = _gpu(A, c), _gpu(B, c)
        assert _same(g, h)
        assert (g["flags"] == 3).all()
    # all groups of every query empty, no points: nothing to solve
    z = _pack([dict(q, groups=[empty()], p3d=np.zeros((0, 3)), p2d=np.zeros((0, 2))) for q in qs[:3]])
    g = _gpu(z, _cfg())
    assert (g["flags"] == 0).all() and (g["iters"] == 0).all()


def test_lane_stride_block_counts():
    """Queries of exactly 1, 31, 32, 33, 64 and 65 blocks (lines and points mixed): lanes stride over blocks by 32, so
    these are the counts where a lane's share changes. Each is solved alone and inside a batch, bit-identically, and
    follows the oracle."""
    rng = np.random.default_rng(9)
    base = _unpack(synth.make_loc_queries(Q=12, P=80, G=40, seed=900, noise_px=1.0, outlier_frac=0.1))
    qs = []
    for i, n in enumerate((1, 31, 32, 33, 64, 65) * 2):
        q = base[i]
        n_pts = int(rng.integers(0, n + 1)) if i < 6 else (n if i % 2 else 0)
        groups, left = [], n - n_pts
        for l3, l2 in q["groups"]:
            if left == 0:
                break
            groups.append((l3, l2[:left]))
            left -= len(groups[-1][1])
        if left:  # not enough 2D lines: points make up the count
            n_pts += left
        qs.append(dict(q, groups=groups, p3d=q["p3d"][:n_pts], p2d=q["p2d"][:n_pts]))
        assert sum(len(g[1]) for g in groups) + n_pts == n
    arrs = _pack(qs)
    for cf, wf in ((2, 0), (3, 1), (5, 4)):
        c = _cfg(cf, wf, 3, 1.0, iters=10)
        g = _gpu(arrs, c)
        assert (g["flags"] & 1).all()
        for i, q in enumerate(qs):
            s = _gpu(_pack([q]), c)
            for k in ("qvec", "tvec", "iters", "cost", "flags"):
                assert np.array_equal(s[k][0], g[k][i]), (i, k)
        _calibrated(arrs, dict(c, max_num_iterations=3), f"block counts cf={cf}")
