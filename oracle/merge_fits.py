"""ctypes wrappers of merging.merging (SetUncertaintySegs3d + MergeToLineTracks, merging.py:6-21 / merging.cc:347-511).
TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/, never by limap_b200/.

  merge_to_linetracks      the fp64 restatement, oracle/orc_merge_fits.cpp -> oracle/_build/liblimap_orc_merge.so
  ref_merge_to_linetracks  the reference's own compiled MergeToLineTracks (oracle/_ref/liblimap_ref.so) behind
                           oracle/ref_merge_fits.cpp -> oracle/_ref/liblimap_ref_merge.so; built only where the
                           reference source tree exists, used to write tests/golden/ref/merge_to_linetracks_*.npz

Both libraries are built with the flags of oracle/Makefile (the oracle's CXXFLAGS; the reference's REF_FLAGS with
-ffp-contract=off for the wrapper, as for ref_api.cpp)."""
import ctypes as C
import os
import subprocess
import sysconfig

import numpy as np

from . import oracle as _orc
from . import ref as _ref

_HERE = os.path.dirname(os.path.abspath(__file__))
ORC_SRC = os.path.join(_HERE, "orc_merge_fits.cpp")
REF_SRC = os.path.join(_HERE, "ref_merge_fits.cpp")
ORC_LIB = os.path.join(_HERE, "_build", "liblimap_orc_merge.so")
REF_LIB = os.path.join(_HERE, "_ref", "liblimap_ref_merge.so")
_CXX = "/usr/bin/g++"
_ORC_FLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-variable",
              "-Wno-sign-compare"]
_P = C.c_void_p
_libs = {}

LINKER2D_DEFAULTS = dict(score_th=0.5, th_angle=8.0, th_overlap=0.1, th_smartoverlap=0.2, th_smartangle=1.0, th_perp=5.0,
                         th_innerseg=5.0, th_scaleinv=0.0, use_angle=1, use_overlap=1, use_smartangle=1, use_perp=1,
                         use_innerseg=0, use_scaleinv=0)  # line_linker.h:23-45
LINKER3D_DEFAULTS = dict(score_th=0.5, th_angle=10.0, th_overlap=0.01, th_smartoverlap=0.1, th_smartangle=1.0,
                         th_perp=0.02, th_innerseg=0.02, th_scaleinv=0.01, use_angle=1, use_overlap=1, use_smartangle=1,
                         use_perp=0, use_innerseg=1, use_scaleinv=0)  # line_linker.h:85-111


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def _run(cmd):
    env = dict(os.environ)
    env.pop("CXX", None)
    subprocess.run(cmd, check=True, env=env, cwd=_HERE)


def build(force=False):
    """Compile the restatement (always possible) and, where the reference tree and oracle/_ref/liblimap_ref.so exist,
    the wrapper of the reference's MergeToLineTracks."""
    hdrs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith(".h")]
    if force or _stale(ORC_LIB, [ORC_SRC] + hdrs):
        os.makedirs(os.path.dirname(ORC_LIB), exist_ok=True)
        _run([_CXX] + _ORC_FLAGS + ["-shared", "-o", ORC_LIB, ORC_SRC])
    if _ref.can_build() and _ref.available() and (force or _stale(REF_LIB, [REF_SRC, _ref.LIB_PATH])):
        import pybind11
        flags = ["-O3", "-march=x86-64-v3", "-include", "immintrin.h", "-fopenmp", "-fPIC", "-std=c++17", "-w",
                 "-Iref_shim", "-I" + _ref.REFERENCE_SRC, "-I" + sysconfig.get_paths()["include"],
                 "-I" + pybind11.get_include(), "-ffp-contract=off"]
        _run([_CXX] + flags + ["-shared", "-o", REF_LIB, REF_SRC, "-L" + os.path.dirname(_ref.LIB_PATH), "-llimap_ref",
                               "-Wl,-rpath,$ORIGIN"])
    return ORC_LIB


def _lib(path):
    if path not in _libs:
        if path == ORC_LIB:
            build()
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing (the reference's wrapper is built only where its source tree exists)")
        _libs[path] = C.CDLL(path)
    return _libs[path]


def linker_struct(d, defaults):
    v = dict(defaults)
    v.update({k: x for k, x in (d or {}).items() if k in v})
    return _orc.OrcLinkerCfg(*[float(v[n]) if t is C.c_double else int(bool(v[n])) for n, t in _orc.OrcLinkerCfg._fields_])


def _call(L, prefix, fit, linker2d, linker3d, var2d):
    run, fetch = getattr(L, prefix + "merge_to_linetracks"), getattr(L, prefix + "merge_fetch")
    run.restype = C.c_int64
    run.argtypes = [C.c_int32] + [_P] * 10 + [C.c_double, _P, _P, _P]
    fetch.argtypes = [_P] * 7
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    i64 = lambda a: np.ascontiguousarray(a, np.int64)
    f64 = _orc._f64
    a = [i32(fit.img_ids), i32(fit.model_ids), f64(fit.kvec), f64(fit.qvec), f64(fit.tvec), i64(fit.line_off),
         f64(np.asarray(fit.segs)[:, :4]), f64(fit.lines3d).reshape(-1, 6), i64(fit.ng_off), i32(fit.ng_ids)]
    counts = np.zeros(4, np.int64)
    T = run(len(a[0]), *[_orc._p(x) for x in a], float(var2d), C.byref(linker_struct(linker2d, LINKER2D_DEFAULTS)),
            C.byref(linker_struct(linker3d, LINKER3D_DEFAULTS)), _orc._p(counts))
    if T < 0:
        L.ref_merge_last_error.restype = C.c_char_p
        raise RuntimeError(L.ref_merge_last_error().decode())
    nn, ne, ns, nl = (int(x) for x in counts)
    out = dict(unc=np.zeros(nl), node_line=np.zeros(nn, np.int64), edges=np.zeros((ne, 2), np.int32), sim=np.zeros(ne),
               track_off=np.zeros(T + 1, np.int64), track_nodes=np.zeros(ns, np.int32), track_line=np.zeros((T, 7)))
    fetch(*[_orc._p(out[k]) for k in ("unc", "node_line", "edges", "sim", "track_off", "track_nodes", "track_line")])
    return out


def merge_to_linetracks(fit, linker2d=None, linker3d=None, var2d=5.0, threads=None):
    """fp64 restatement of merging.merging on a synth.FitScene-like object (img_ids, model_ids, kvec, qvec, tvec,
    line_off, segs, lines3d, ng_off, ng_ids). Returns dict(unc, node_line, edges, sim, track_off, track_nodes,
    track_line)."""
    L = _lib(ORC_LIB)
    L.orc_merge_set_num_threads.argtypes = [C.c_int]
    L.orc_merge_set_num_threads(int(threads) if threads else min(8, _orc.usable_cpus()))
    return _call(L, "orc_", fit, linker2d, linker3d, var2d)


def ref_merge_to_linetracks(fit, linker2d=None, linker3d=None, var2d=5.0):
    """The reference's merging.merging: its compiled SetUncertaintySegs3d + MergeToLineTracks."""
    return _call(_lib(REF_LIB), "ref_", fit, linker2d, linker3d, var2d)
