"""ctypes wrapper of the query pose refinement oracle (JointLocEngine / LineLocEngine). TEST INFRASTRUCTURE ONLY:
imported by tests/ and scripts/, never by limap_b200/.

  orc_loc_solve      the fp64 restatement of the residuals, weights, losses and LM solve, oracle/orc_loc.cpp ->
                     oracle/_build/liblimap_orc_loc.so; queries run in parallel over the host's cores
  orc_loc_functor    one residual functor on 7-wide jets (values and ambient Jacobian)
  orc_loc_loss       the loss (Trivial, Huber, SoftLOne, Cauchy) and ScaledLoss factor of many blocks
  ref_loc_functor    the reference's own ReprojectionLineFunctor / ReprojectionPointFunctor (cost_functions.h, compiled
                     unchanged by oracle/ref_loc.cpp) on 7-wide jets -> oracle/_ref/liblimap_ref_loc.so; built only where
                     the reference source tree exists, used to write tests/golden/ref/localization.npz"""
import ctypes as C
import os
import sysconfig

import numpy as np

from . import evaluation as _ev
from . import ref as _ref

_HERE = os.path.dirname(os.path.abspath(__file__))
ORC_SRC = os.path.join(_HERE, "orc_loc.cpp")
ORC_LIB = os.path.join(_HERE, "_build", "liblimap_orc_loc.so")
REF_SRC = os.path.join(_HERE, "ref_loc.cpp")
REF_LIB = os.path.join(_HERE, "_ref", "liblimap_ref_loc.so")
_DEPS = [ORC_SRC, os.path.join(_HERE, "orc_lm.h"), os.path.join(_HERE, "orc_geom.h")]
_P = C.c_void_p
_lib = None
_ref_lib = None


class _Config(C.Structure):
    _fields_ = [("cost_function", C.c_int32), ("weight_function", C.c_int32), ("loss_kind", C.c_int32),
                ("points_3d_dist", C.c_int32), ("loss_scale", C.c_double), ("weight_point", C.c_double),
                ("weight_line", C.c_double), ("max_num_iterations", C.c_int32),
                ("max_num_consecutive_invalid_steps", C.c_int32)]


def build(force=False):
    if force or _ev._stale(ORC_LIB, _DEPS):
        os.makedirs(os.path.dirname(ORC_LIB), exist_ok=True)
        _ev._run([_ev._CXX] + _ev._ORC_FLAGS + ["-shared", "-o", ORC_LIB, ORC_SRC])
    shadow = os.path.join(_HERE, "ref_shim_loc", "limap", "optimize", "hybrid_localization",
                          "hybrid_localization_config.h")
    if _ref.can_build() and _ref.available() and (force or _ev._stale(REF_LIB, [REF_SRC, shadow, _ref.LIB_PATH])):
        import pybind11
        # REF_FLAGS of oracle/Makefile, with oracle/ref_shim_loc ahead of the reference tree
        _ev._run([_ev._CXX, "-O3", "-march=x86-64-v3", "-include", "immintrin.h", "-fopenmp", "-fPIC", "-std=c++17", "-w",
                  "-Iref_shim_loc", "-Iref_shim", "-I" + _ref.REFERENCE_SRC, "-I" + sysconfig.get_paths()["include"],
                  "-I" + pybind11.get_include(), "-shared", "-o", REF_LIB, REF_SRC,
                  "-L" + os.path.dirname(_ref.LIB_PATH), "-llimap_ref", "-Wl,-rpath,$ORIGIN"])
    return ORC_LIB


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(ORC_LIB)
        L.orc_loc_solve.restype = None
        L.orc_loc_solve.argtypes = [C.c_int64] + [_P] * 10 + [_P, C.c_int32] + [_P] * 6
        L.orc_loc_functor.restype = None
        L.orc_loc_functor.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int] + [_P] * 6
        L.orc_loc_loss.restype = None
        L.orc_loc_loss.argtypes = [C.c_int, C.c_double, C.c_int64, _P, _P, _P]
        _lib = L
    return _lib


def ref_lib():
    global _ref_lib
    if _ref_lib is None:
        build()
        if not os.path.exists(REF_LIB):
            raise RuntimeError(f"{REF_LIB} is missing (built only where the reference source tree exists)")
        L = C.CDLL(REF_LIB)
        L.ref_loc_functor.restype = None
        L.ref_loc_functor.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int] + [_P] * 6
        _ref_lib = L
    return _ref_lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


def solve(batch, cost_function=2, weight_function=0, loss_kind=0, loss_scale=1.0, weight_point=1.0, weight_line=1.0,
          points_3d_dist=None, max_num_iterations=100, max_num_consecutive_invalid_steps=10, stop_after=-1):
    """batch: a dict of the lm_loc_solve arrays (limap_b200.hybrid_localization.LocBatch.arrays()). Returns qvec, tvec,
    iters, cost, flags and term per query."""
    if points_3d_dist is None:
        points_3d_dist = cost_function in (4, 5)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    i64 = lambda a: np.ascontiguousarray(a, np.int64)
    kvec, qvec, tvec = f64(batch["kvec"]), f64(batch["qvec"]), f64(batch["tvec"])
    p3d, p2d, l3d, l2d = (f64(batch[k]).reshape(-1, n) for k, n in (("p3d", 3), ("p2d", 2), ("l3d", 6), ("l2d", 4)))
    pt_off, grp_off, l2d_off = i64(batch["pt_off"]), i64(batch["grp_off"]), i64(batch["l2d_off"])
    Q = len(kvec)
    cfg = _Config(cost_function, weight_function, loss_kind, int(bool(points_3d_dist)), loss_scale, weight_point,
                  weight_line, max_num_iterations, max_num_consecutive_invalid_steps)
    out = dict(qvec=np.zeros((Q, 4)), tvec=np.zeros((Q, 3)), iters=np.zeros((Q, 2), np.int32),
               cost=np.zeros((Q, 2)), flags=np.zeros(Q, np.uint8), term=np.zeros(Q, np.int32))
    lib().orc_loc_solve(Q, _ptr(kvec), _ptr(qvec), _ptr(tvec), _ptr(pt_off), _ptr(p3d), _ptr(p2d), _ptr(grp_off),
                        _ptr(l3d), _ptr(l2d_off), _ptr(l2d), C.byref(cfg), int(stop_after), _ptr(out["qvec"]),
                        _ptr(out["tvec"]), _ptr(out["iters"]), _ptr(out["cost"]), _ptr(out["flags"]),
                        _ptr(out["term"]))
    return out


def functor(kind, data, kvec, qvec, tvec, cost_function=2, weight_function=0, use3d=False, ref=False):
    """Residuals res[4] and ambient Jacobian jac[4][7] of one line (kind 0, data = l3d[6] + l2d[4]) or point (kind 1,
    data = p3d[3] + p2d[2]) functor; ref=True evaluates the reference's compiled functor instead."""
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    res, jac = np.zeros(4), np.zeros((4, 7))
    fn = ref_lib().ref_loc_functor if ref else lib().orc_loc_functor
    fn(kind, cost_function, weight_function, int(use3d), _ptr(f64(data)), _ptr(f64(kvec)), _ptr(f64(qvec)),
       _ptr(f64(tvec)), _ptr(res), _ptr(jac))
    return res, jac


def loss(kind, scale, a, s):
    """rho[n][3] of the loss (kind 0..3, scale) with ScaledLoss factors a[n] at squared residual norms s[n]."""
    s = np.ascontiguousarray(s, np.float64).ravel()
    a = np.ascontiguousarray(np.broadcast_to(a, s.shape), np.float64)
    rho = np.zeros((len(s), 3))
    lib().orc_loc_loss(kind, scale, len(s), _ptr(a), _ptr(s), _ptr(rho))
    return rho
