"""The query pose refinement's residual blocks (limap_b200/csrc/loc_block.cuh) compiled for the host and checked, with
no GPU, against (a) the reference's own compiled ReprojectionLineFunctor / ReprojectionPointFunctor values stored in
tests/golden/ref/localization.npz and (b) the oracle's functors (oracle/orc_loc.cpp), both taken to the 6-dof tangent
through QuaternionPlusJacobian. Also the loss, Ceres' corrector and the 6x6 L D L^T step solve, and the branches of the
block math planted on their edges: line_line_dist either side of n2 = 1e-8, the sine / cosine clamps at 1, zero-length
2D lines, 3D lines ending behind the camera and points on the camera plane."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import localization as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "loc_block_host.cu")
G = np.load(os.path.join(ROOT, "tests", "golden", "ref", "localization.npz"))
_P = C.c_void_p
CF = range(6)
WF = range(5)
NRES = {0: 2, 1: 3, 2: 2, 3: 4, 4: 2, 5: 2}
# Bars. The block is the oracle's and the reference's expression operation for operation; they differ in FMA
# contraction only (the oracle and the reference are built with -march=x86-64-v3, this harness without FMA). Residuals:
# relative to max(|r|, 1), since the midpoint and perpendicular residuals are differences of pixel coordinates of
# some 100 px. Jacobian rows: relative to the row maximum.
RES_TOL = 1e-12
JAC_TOL = 1e-9


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("loc_block_host") / "libloc_block_host.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-o", so, HARNESS], check=True)
    L = C.CDLL(so)
    L.loch_block.argtypes = [C.c_int64, C.c_int, C.c_int, C.c_int] + [_P] * 6
    L.loch_loss.argtypes = [C.c_int64, C.c_int, C.c_double, _P, _P, _P]
    L.loch_corrector.argtypes = [C.c_int64, C.c_int, C.c_int, C.c_double] + [_P] * 6
    L.loch_ldlt.argtypes = [C.c_int64] + [_P] * 5
    return L


def _c(a, dt=np.float64):
    return np.ascontiguousarray(a, dt)


def _p(a):
    return a.ctypes.data_as(_P)


def block(hlib, cf, wf, use3d, kind, data, kvec, qvec, tvec):
    """The device block on the host: residuals [n][4] and tangent Jacobian [n][4][6]."""
    n = len(data)
    kind = _c(np.broadcast_to(kind, (n,)), np.int32)
    data, kvec, x = _c(data), _c(kvec), _c(np.concatenate([qvec, tvec], 1))
    res, jac = np.zeros((n, 4)), np.zeros((n, 4, 6))
    hlib.loch_block(n, cf, wf, int(use3d), _p(kind), _p(data), _p(kvec), _p(x), _p(res), _p(jac))
    return res, jac


def plus_jacobian(q):
    """QuaternionPlusJacobian (4x3) on qvec, identity on tvec: [n][7][6]."""
    P = np.zeros((len(q), 7, 6))
    x0, x1, x2, x3 = q.T
    P[:, :4, :3] = np.stack([np.stack([-x1, -x2, -x3], 1), np.stack([x0, x3, -x2], 1), np.stack([-x3, x0, x1], 1),
                             np.stack([x2, -x1, x0], 1)], 1)
    P[:, 4:, 3:] = np.eye(3)
    return P


def oracle_block(cf, wf, use3d, kind, data, kvec, qvec, tvec):
    n = len(data)
    res, jac = np.zeros((n, 4)), np.zeros((n, 4, 7))
    for i in range(n):
        res[i], jac[i] = orc.functor(int(np.broadcast_to(kind, (n,))[i]), data[i], kvec[i], qvec[i], tvec[i], cf, wf,
                                     use3d)
    return res, np.einsum("nrj,nji->nri", jac, plus_jacobian(qvec))


def _compare(res, jac, rref, jref, what):
    """max relative residual and Jacobian-row errors; NaN / inf must sit at the same places."""
    fin = np.isfinite(rref).all(1)
    assert np.array_equal(np.isfinite(res), np.isfinite(rref)), what
    er = (np.abs(res - rref)[fin] / np.maximum(np.abs(rref[fin]).max(1, keepdims=True), 1.0)).max(initial=0)
    assert er <= RES_TOL, (what, er)
    jf, jr = jac[fin], jref[fin]
    sc = np.maximum(np.abs(jr).max(2, keepdims=True), 1e-300)
    ej = (np.abs(jf - jr) / sc).max(initial=0)
    assert ej <= JAC_TOL, (what, ej)
    return er, ej


# ---- random blocks: every CF x wf, both point modes, unit and non-unit quaternions ---------------------------------
QNORMS = (1.0, 0.5, 2.0, 1.0 + 1e-8)


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _quat_R(q):
    """ceres::QuaternionToRotation (normalised by |q|^2)."""
    a, b, c, d = q.T
    n = 1.0 / (a * a + b * b + c * c + d * d)
    return np.stack([a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (a * c + b * d),
                     2 * (a * d + b * c), a * a - b * b + c * c - d * d, 2 * (c * d - a * b),
                     2 * (b * d - a * c), 2 * (a * b + c * d), a * a - b * b - c * c + d * d], 1).reshape(-1, 3, 3) * n[:, None, None]


def random_poses(rng, n):
    q = _unit(rng.normal(size=(n, 4))) * np.array(QNORMS)[np.arange(n) % len(QNORMS), None]
    t = rng.normal(size=(n, 3))
    fx = rng.uniform(300, 900, n)
    kvec = np.stack([fx, fx * rng.uniform(0.85, 1.15, n), rng.uniform(250, 400, n), rng.uniform(200, 300, n)], 1)
    return kvec, q, t


def backproject(kvec, q, t, u, v, z):
    """World point at pixel (u, v), camera depth z."""
    xc = np.stack([(u - kvec[:, 2]) / kvec[:, 0] * z, (v - kvec[:, 3]) / kvec[:, 1] * z, z], -1)
    return np.einsum("nji,nj->ni", _quat_R(q), xc - t)


def project(kvec, q, t, X):
    xc = np.einsum("nij,nj->ni", _quat_R(q), X) + t
    return np.stack([kvec[:, 0] * xc[:, 0] / xc[:, 2] + kvec[:, 2], kvec[:, 1] * xc[:, 1] / xc[:, 2] + kvec[:, 3]], 1)


def random_lines(rng, n):
    kvec, q, t = random_poses(rng, n)
    s3 = backproject(kvec, q, t, rng.uniform(0, 640, n), rng.uniform(0, 480, n), rng.uniform(1, 6, n))
    e3 = backproject(kvec, q, t, rng.uniform(0, 640, n), rng.uniform(0, 480, n), rng.uniform(1, 6, n))
    l2 = np.concatenate([project(kvec, q, t, s3), project(kvec, q, t, e3)], 1) + rng.normal(size=(n, 4)) * 2.0
    return np.concatenate([s3, e3, l2], 1), kvec, q, t


def random_points(rng, n):
    kvec, q, t = random_poses(rng, n)
    p3 = backproject(kvec, q, t, rng.uniform(0, 640, n), rng.uniform(0, 480, n), rng.uniform(1, 6, n))
    p2 = project(kvec, q, t, p3) + rng.normal(size=(n, 2)) * 2.0
    return np.concatenate([p3, p2, np.zeros((n, 5))], 1), kvec, q, t


@pytest.mark.parametrize("cf", CF)
def test_line_block_matches_reference_values(hlib, cf):
    """Every stored reference evaluation of ReprojectionLineFunctor, all five weights."""
    for wf in WF:
        idx = np.flatnonzero((G["kind"] == 0) & (G["cf"] == cf) & (G["wf"] == wf))
        assert len(idx) >= 40
        res, jac = block(hlib, cf, wf, 0, 0, G["data"][idx], G["kvec"][idx], G["qvec"][idx], G["tvec"][idx])
        jref = np.einsum("nrj,nji->nri", G["jac"][idx], plus_jacobian(G["qvec"][idx]))
        _compare(res, jac, G["res"][idx], jref, (cf, wf))
        assert not res[:, NRES[cf]:].any() and not jac[:, NRES[cf]:].any()
    nrm = np.linalg.norm(G["qvec"][G["kind"] == 0], axis=1)
    assert (np.abs(nrm - 1) < 1e-12).any() and (np.abs(nrm - 1) > 1e-6).any()  # unit and non-unit quaternions


@pytest.mark.parametrize("use3d", [0, 1])
def test_point_block_matches_reference_values(hlib, use3d):
    idx = np.flatnonzero((G["kind"] == 1) & (G["use3d"] == use3d))
    assert len(idx) >= 40
    res, jac = block(hlib, 2, 0, use3d, 1, G["data"][idx], G["kvec"][idx], G["qvec"][idx], G["tvec"][idx])
    jref = np.einsum("nrj,nji->nri", G["jac"][idx], plus_jacobian(G["qvec"][idx]))
    _compare(res, jac, G["res"][idx], jref, use3d)


@pytest.mark.parametrize("cf", CF)
def test_line_block_matches_oracle(hlib, cf):
    """Seeded blocks with quaternion norms 1, 0.5, 2 and 1 + 1e-8 (PixelToWorld uses the unnormalised conjugate)."""
    rng = np.random.default_rng(100 + cf)
    for wf in WF:
        data, kvec, q, t = random_lines(rng, 120)
        res, jac = block(hlib, cf, wf, 0, 0, data, kvec, q, t)
        rref, jref = oracle_block(cf, wf, False, 0, data, kvec, q, t)
        _compare(res, jac, rref, jref, (cf, wf))
        # the quaternion columns respond to the norm where PixelToWorld enters (CF 4, 5): the reference's own
        # behaviour, kept
        assert np.isfinite(res).all()


@pytest.mark.parametrize("use3d", [0, 1])
def test_point_block_matches_oracle(hlib, use3d):
    rng = np.random.default_rng(7 + use3d)
    data, kvec, q, t = random_points(rng, 400)
    res, jac = block(hlib, 2, 0, use3d, 1, data, kvec, q, t)
    rref, jref = oracle_block(2, 0, bool(use3d), 1, data, kvec, q, t)
    _compare(res, jac, rref, jref, use3d)
    if use3d:
        assert not res[:, 1].any() and not jac[:, 1].any()


# ---- planted branches -----------------------------------------------------------------------------------------------
def _unit_rotate(q, p):
    """ceres::UnitQuaternionRotatePoint, also for the non-unit q PixelToWorld passes it."""
    v = q[:, 1:]
    uv = 2 * np.cross(v, p)
    return p + q[:, :1] * uv + np.cross(v, uv)


def _pixel_to_world(kvec, q, t, p2, depth):
    l = np.stack([(p2[:, 0] - kvec[:, 2]) / kvec[:, 0], (p2[:, 1] - kvec[:, 3]) / kvec[:, 1], np.ones(len(p2))], 1)
    return _unit_rotate(q * [1, -1, -1, -1], l * depth[:, None] - t)


def _line_along_ray(rng, n, rel):
    """3D lines through the PixelToWorld ray of their 2D start point, turned off the ray so that n2 = |dir x dir3d|^2
    of Ceres_3DLineLineDist is 1e-8 (1 + rel)."""
    kvec, q, t = random_poses(rng, n)
    p2 = np.stack([rng.uniform(50, 590, n), rng.uniform(50, 430, n)], 1)
    s3 = _pixel_to_world(kvec, q, t, p2, rng.uniform(2, 5, n))
    d = _pixel_to_world(kvec, q, t, p2, np.full(n, 2.0)) - _pixel_to_world(kvec, q, t, p2, np.ones(n))
    nd = np.linalg.norm(d, axis=1)
    e = _unit(np.cross(d, rng.normal(size=(n, 3))))
    # dir3d = (e3 - s3) / sqrt(|e3 - s3|^2 + 1e-8) with |e3 - s3| = 1, so |dir3d|^2 = 1 / (1 + 1e-8)
    sin = np.sqrt(1e-8 * (1 + rel) * (1 + 1e-8)) / nd
    e3 = s3 + np.sqrt(1 - sin ** 2)[:, None] * d / nd[:, None] + sin[:, None] * e
    l2 = np.concatenate([p2, project(kvec, q, t, e3)], 1)
    return np.concatenate([s3, e3, l2], 1), kvec, q, t


def test_line_line_dist_parallel_branch_either_side(hlib):
    """A 3D line laid along the viewing ray of its 2D start point, n2 one part in 1e4 either side of 1e-8. The start
    residual of Ceres_3DLineLineDist is then ~0 on the general branch (the 3D point lies on the ray) and
    sqrt(|dir x d|^2 / |dir|^2 + 1e-8) = 1e-4 on the parallel branch (n2 <= 1e-8)."""
    rng = np.random.default_rng(3)
    for rel, parallel in ((1e-4, False), (-1e-4, True)):
        data, kvec, q, t = _line_along_ray(rng, 200, rel)
        res, jac = block(hlib, 4, 0, 0, 0, data, kvec, q, t)
        if parallel:
            assert (np.abs(res[:, 0] - 1e-4) < 1e-9).all(), np.abs(res[:, 0] - 1e-4).max()
        else:
            assert (np.abs(res[:, 0]) < 1e-8).all(), np.abs(res[:, 0]).max()
        rref, jref = oracle_block(4, 0, False, 0, data, kvec, q, t)
        # the general branch divides a rounding-level n . d by sqrt(n2): the residual is compared absolutely there
        assert np.abs(res[:, 0] - rref[:, 0]).max() <= 1e-12
        sc = np.maximum(np.abs(jref).max(2, keepdims=True), 1e-300)
        assert (np.abs(jac - jref) / sc)[:, 1].max() <= JAC_TOL
        if parallel:
            assert (np.abs(jac - jref) / sc)[:, 0].max() <= JAC_TOL


def _on_projected_line(rng, n, perpendicular):
    """2D segments on the projected 3D line (parallel to dir2d) or with both endpoints off the projected start point
    perpendicular to it."""
    data, kvec, q, t = random_lines(rng, n)
    sr, er = project(kvec, q, t, data[:, :3]), project(kvec, q, t, data[:, 3:6])
    d = _unit(er - sr)
    a, b = rng.uniform(-200, -20, (n, 1)), rng.uniform(20, 200, (n, 1))
    if perpendicular:
        d = np.stack([-d[:, 1], d[:, 0]], 1)
    data[:, 6:8], data[:, 8:10] = sr + a * d, sr + b * d
    return data, kvec, q, t


def test_sine_and_cosine_clamps_unreachable(hlib):
    """The clamps at 1 of CeresComputeDist2D_sine / _cosine cannot fire in double precision: their first argument is
    normalised with sqrt(|d|^2 + 1e-8) and then divided by sqrt(|.|^2 + EPS), so the ratio stays below 1 by about
    EPS / 2 = 5e-13, far above the rounding of the dot / cross product (~1e-16). Planted at the edge, the sine and cosine
    come within 1e-11 of 1 and stay <= 1. The clamp is kept because the reference has it."""
    rng = np.random.default_rng(5)
    # cosine2d(dir2d, direc): 2D segments along the projected line; w = exp(10 (1 - cos)) of wf 1
    data, kvec, q, t = _on_projected_line(rng, 300, False)
    r0, _ = block(hlib, 0, 0, 0, 0, data, kvec, q, t)
    r1, j1 = block(hlib, 0, 1, 0, 0, data, kvec, q, t)
    one_minus_cos = np.log(r1[:, :2] / r0[:, :2]).max(1) / 10.0
    assert (one_minus_cos >= 0).all() and (one_minus_cos < 1e-11).all(), one_minus_cos.max()
    # wf 2 (exp(10 acos(cos))) at the same edge: acos' derivative -1/sqrt(1 - c^2) is large but finite, as the oracle's
    r2, j2 = block(hlib, 0, 2, 0, 0, data, kvec, q, t)
    assert np.isfinite(j2).all()
    rref, jref = oracle_block(0, 2, False, 0, data, kvec, q, t)
    assert (np.abs(r2 - rref) <= 1e-9 * np.maximum(np.abs(rref), 1.0)).all()
    # sine2d(dir2d, s2d - sr) of the perpendicular distances: endpoints off the projected start point perpendicular to
    # the projected line; CF 3 writes (a sa, c sc), so sa = |res[0:2]| / |a|
    data, kvec, q, t = _on_projected_line(rng, 300, True)
    r3, _ = block(hlib, 3, 0, 0, 0, data, kvec, q, t)
    sr = project(kvec, q, t, data[:, :3])
    sa = np.hypot(r3[:, 0], r3[:, 1]) / np.linalg.norm(data[:, 6:8] - sr, axis=1)
    sc = np.hypot(r3[:, 2], r3[:, 3]) / np.linalg.norm(data[:, 8:10] - sr, axis=1)
    for s in (sa, sc):
        assert (s > 1 - 1e-11).all() and (s <= 1 + 1e-15).all(), (s.min(), s.max())
    # sine2d(d1, d2) of CF 1: the same segments are perpendicular to the projected line, res[2] = n1 sine
    r1, _ = block(hlib, 1, 0, 0, 0, data, kvec, q, t)
    n1 = np.sqrt(((project(kvec, q, t, data[:, 3:6]) - sr) ** 2).sum(1) + 1e-8)
    s1 = r1[:, 2] / n1
    assert (s1 > 1 - 1e-11).all() and (s1 <= 1 + 1e-15).all(), (s1.min(), s1.max())
    for cf in (1, 3):
        _compare(*block(hlib, cf, 1, 0, 0, data, kvec, q, t), *oracle_block(cf, 1, False, 0, data, kvec, q, t), cf)


def test_zero_length_2d_line(hlib):
    """direc = 0: wf 3 weighs by sqrt(1e-8) = 1e-4, wf 4 by 1e4, wf 1 by exp(10) (cosine 0 / EPS-normalised = 0) and
    wf 2 by exp(10 pi / 2); CF 1's angle term is 0; CF 5's plane through two equal rays has n = 0 and its residuals
    are 0 / 0 = NaN, as the oracle's (the solve then fails its first evaluation)."""
    rng = np.random.default_rng(9)
    data, kvec, q, t = random_lines(rng, 60)
    data[:, 8:10] = data[:, 6:8]
    r0, _ = block(hlib, 2, 0, 0, 0, data, kvec, q, t)
    for wf, w in ((1, np.exp(10.0)), (2, np.exp(10.0 * np.pi / 2)), (3, 1e-4), (4, 1e4)):
        r, _ = block(hlib, 2, wf, 0, 0, data, kvec, q, t)
        assert np.allclose(r[:, :2], r0[:, :2] * w, rtol=1e-13, atol=0), wf
    r1, _ = block(hlib, 1, 0, 0, 0, data, kvec, q, t)
    assert not r1[:, 2].any()
    r5, _ = block(hlib, 5, 0, 0, 0, data, kvec, q, t)
    assert np.isnan(r5[:, :2]).all()
    for cf in CF:
        for wf in WF:
            res, jac = block(hlib, cf, wf, 0, 0, data, kvec, q, t)
            _compare(res, jac, *oracle_block(cf, wf, False, 0, data, kvec, q, t), (cf, wf))


def test_line_ending_behind_the_camera(hlib):
    rng = np.random.default_rng(13)
    data, kvec, q, t = random_lines(rng, 60)
    data[:, 3:6] = backproject(kvec, q, t, rng.uniform(0, 640, 60), rng.uniform(0, 480, 60), -rng.uniform(1, 6, 60))
    zc = np.einsum("nij,nj->ni", _quat_R(q), data[:, 3:6]) + t
    assert (zc[:, 2] < 0).all()
    for cf in CF:
        for wf in WF:
            res, jac = block(hlib, cf, wf, 0, 0, data, kvec, q, t)
            assert np.isfinite(res).all()
            _compare(res, jac, *oracle_block(cf, wf, False, 0, data, kvec, q, t), (cf, wf))


def test_point_on_the_camera_plane(hlib):
    """z = 0 in the camera frame: the reprojection divides by zero (non-finite residuals, which fail an evaluation);
    the point-to-ray distance does not project and stays finite."""
    n = 40
    rng = np.random.default_rng(17)
    kvec, _, _ = random_poses(rng, n)
    q, t = np.tile([1.0, 0, 0, 0], (n, 1)), np.zeros((n, 3))  # world frame = camera frame, bit for bit
    data = np.zeros((n, 10))
    data[:, :2] = rng.normal(size=(n, 2))
    data[:, 3:5] = rng.uniform(0, 480, (n, 2))
    res, _ = block(hlib, 2, 0, 0, 1, data, kvec, q, t)
    assert not np.isfinite(res[:, :2]).any()
    rref, _ = oracle_block(2, 0, False, 1, data, kvec, q, t)
    assert not np.isfinite(rref[:, :2]).any()
    res, jac = block(hlib, 2, 0, 1, 1, data, kvec, q, t)
    assert np.isfinite(res).all() and np.isfinite(jac).all()
    _compare(res, jac, *oracle_block(2, 0, True, 1, data, kvec, q, t), "use3d")


# ---- loss and corrector ---------------------------------------------------------------------------------------------
LOSSES = [(0, 1.0), (1, 2.0), (1, 0.3), (2, 1.5), (3, 1.0), (3, 0.1)]


def _loss(hlib, kind, scale, a, s):
    s = _c(s)
    a = _c(np.broadcast_to(a, s.shape))
    rho = np.zeros((len(s), 3))
    hlib.loch_loss(len(s), kind, scale, _p(a), _p(s), _p(rho))
    return rho


@pytest.mark.parametrize("kind,scale", LOSSES)
def test_loss_matches_oracle(hlib, kind, scale):
    """The same expressions as the oracle's restatement of loss_function.cc: equal to the last bit up to FMA."""
    rng = np.random.default_rng(kind)
    s = np.r_[0.0, 10.0 ** rng.uniform(-12, 8, 2000), scale * scale]
    a = np.r_[1.0, rng.uniform(0.01, 3.0, 2000), 1.0]
    d, o = _loss(hlib, kind, scale, a, s), orc.loss(kind, scale, a, s)
    assert (np.abs(d - o) <= 4e-16 * np.abs(o)).all()
    assert (d[:, 1] > 0).all() and (d[:, 2] <= 0).all()


def test_huber_at_its_threshold(hlib):
    """Huber switches to the linear branch at s > b = scale^2 strictly: at s == b it is still quadratic (rho'' = 0),
    one ulp above it is linear (rho'' < 0), and rho and rho' are continuous across."""
    for scale in (2.0, 0.3, 1.7):
        b = scale * scale
        s = np.array([np.nextafter(b, 0), b, np.nextafter(b, np.inf)])
        d, o = _loss(hlib, 1, scale, 1.0, s), orc.loss(1, scale, 1.0, s)
        assert np.array_equal(d[:2, 2], [0.0, 0.0]) and d[2, 2] < 0
        assert np.array_equal(d[:2, :2], np.stack([s[:2], [1.0, 1.0]], 1))
        assert np.abs(d - o).max() <= 4e-16 * np.abs(o).max()
        assert abs(d[2, 0] - d[1, 0]) < 1e-14 * b and abs(d[2, 1] - 1.0) < 1e-14


def _corrector_ref(r, J, rho):
    """ceres corrector.cc in numpy: sqrt(rho') (J - alpha/|r|^2 r r^T J), residuals sqrt(rho') / (1 - alpha) r."""
    s = (r * r).sum(1)
    sq = np.sqrt(rho[:, 1])
    rs, al_s = sq.copy(), np.zeros(len(r))
    use = ~((s == 0) | (rho[:, 2] <= 0))
    al = 1 - np.sqrt(1 + 2 * s[use] * rho[use, 2] / rho[use, 1])
    rs[use] = sq[use] / (1 - al)
    al_s[use] = al / s[use]
    rtj = np.einsum("ni,nic->nc", r, J)
    Jc = sq[:, None, None] * (J - al_s[:, None, None] * r[:, :, None] * rtj[:, None, :])
    return r * rs[:, None], Jc


@pytest.mark.parametrize("kind,scale", LOSSES)
def test_corrector_rows(hlib, kind, scale):
    """The corrector's residual and Jacobian scaling, on blocks of 2, 3 and 4 residuals with norms across the loss
    scale, against the numpy restatement; also r = 0 (the rho'' branch is skipped)."""
    rng = np.random.default_rng(20 + kind)
    for m in (2, 3, 4):
        n = 600
        res = np.zeros((n, 4))
        res[:, :m] = rng.normal(size=(n, m)) * 10.0 ** rng.uniform(-3, 2, (n, 1))
        res[0] = 0.0
        jac = np.zeros((n, 4, 6))
        jac[:, :m] = rng.normal(size=(n, m, 6)) * 10.0 ** rng.uniform(-2, 3, (n, 1, 6))
        a = rng.uniform(0.1, 2.0, n)
        rho, rc, jc = np.zeros((n, 3)), np.zeros((n, 4)), np.zeros((n, 4, 6))
        hlib.loch_corrector(n, m, kind, scale, _p(_c(a)), _p(_c(res)), _p(_c(jac)), _p(rho), _p(rc), _p(jc))
        assert np.array_equal(rho, _loss(hlib, kind, scale, a, (res * res).sum(1)))
        rr, jr = _corrector_ref(res, jac, rho)
        assert (np.abs(rc - rr) <= 1e-14 * np.abs(rr).max(1, keepdims=True)).all()
        # the corrected Jacobian subtracts alpha r r^T J / |r|^2 from J: compared relative to |J| of the column
        sc = np.maximum(np.abs(jac).max(1, keepdims=True), 1e-300) * np.sqrt(rho[:, 1])[:, None, None]
        assert (np.abs(jc - jr) / sc).max() <= 1e-13
        assert not rc[:, m:].any() and not jc[:, m:].any()
        if kind == 0:  # trivial loss: the identity times sqrt(a)
            assert np.allclose(jc, jac * np.sqrt(a)[:, None, None], rtol=1e-15, atol=0)


# ---- the 6x6 step solve ---------------------------------------------------------------------------------------------
def _pack(A):
    iu = np.triu_indices(6)
    return _c(A[:, iu[0], iu[1]])


def _ldlt(hlib, A, dg, b):
    n = len(A)
    x, ok = np.zeros((n, 6)), np.zeros(n, np.int32)
    hlib.loch_ldlt(n, _p(_pack(A)), _p(_c(dg)), _p(_c(b)), _p(x), _p(ok))
    return x, ok.astype(bool)


def test_ldlt_solve6_well_and_ill_conditioned(hlib):
    """Against numpy's float64 solve of the damped system (A + diag(dg)) x = b. Well conditioned: forward error within
    1e-13. Condition numbers up to 1e12: the backward error |(A + D) x - b| / (|A + D| |x|) within 1e-15 (LDL^T
    without pivoting is backward stable on symmetric positive definite matrices), forward error within 4 cond u
    (measured: at most 0.42 cond u)."""
    rng = np.random.default_rng(31)
    n = 3000
    for cond_exp in (1, 6, 12):
        U = np.linalg.qr(rng.normal(size=(n, 6, 6)))[0]
        ev = 10.0 ** -np.sort(rng.uniform(0, cond_exp, (n, 6)), 1)[:, ::-1] * 10.0 ** rng.uniform(-6, 6, (n, 1))
        J = U * np.sqrt(ev)[:, None, :]
        A = J @ np.swapaxes(J, 1, 2)  # J J^T, symmetric positive semi-definite
        dg = np.abs(np.einsum("nii->ni", A)) * 10.0 ** rng.uniform(-16, -4, (n, 1))
        b = rng.normal(size=(n, 6))
        x, ok = _ldlt(hlib, A, dg, b)
        M = A + dg[:, :, None] * np.eye(6)
        # the packed upper triangle is all the solve reads: symmetric by construction up to rounding
        Ms = np.triu(M) + np.swapaxes(np.triu(M, 1), 1, 2)
        assert ok.all()
        ref = np.linalg.solve(Ms, b[..., None])[..., 0]
        bw = np.linalg.norm(np.einsum("nij,nj->ni", Ms, x) - b, axis=1) / (
            np.linalg.norm(Ms, axis=(1, 2)) * np.linalg.norm(x, axis=1))
        assert bw.max() <= 1e-15, bw.max()
        cond = np.linalg.cond(Ms)
        fw = np.linalg.norm(x - ref, axis=1) / np.linalg.norm(ref, axis=1)
        if cond_exp == 1:
            assert fw.max() <= 1e-13, fw.max()
        assert (fw <= 4 * cond * 2.2e-16 + 1e-13).all(), (fw / cond).max()


def test_ldlt_solve6_refuses_non_positive_pivots(hlib):
    """An indefinite or singular system returns false (the step is invalid), as the oracle's Cholesky does."""
    rng = np.random.default_rng(37)
    n = 500
    J = rng.normal(size=(n, 6, 6))
    A = J @ np.swapaxes(J, 1, 2)
    k = rng.integers(0, 6, n)
    A[np.arange(n), k, :] = 0.0
    A[np.arange(n), :, k] = 0.0  # a zero row and column: pivot k is 0
    A[: n // 2, k[: n // 2], k[: n // 2]] = -1.0  # or negative
    _, ok = _ldlt(hlib, A, np.zeros((n, 6)), rng.normal(size=(n, 6)))
    assert not ok.any()
    # with a damping diagonal the same systems are positive definite and solve
    x, ok = _ldlt(hlib, np.abs(A), np.full((n, 6), 1e-3) + np.abs(A).sum(2), rng.normal(size=(n, 6)))
    assert ok.all() and np.isfinite(x).all()
