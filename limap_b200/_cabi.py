"""ctypes binding of the C ABI in include/limap_b200.h. Fails loudly when the CUDA library is missing:
there is no CPU fallback on the product path."""
import ctypes as C
import os

import numpy as np

from .config import TriConfig

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LIMAP_B200_LIB") or os.path.join(_HERE, "lib", "liblimap_b200.so")  # (override: A/B builds)
_lib = None


class LimapB200Error(RuntimeError):
    pass


class TriStats(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_candidates", C.c_int64), ("n_valid_edges", C.c_int64),
                ("n_nodes", C.c_int64), ("n_kernel_launches", C.c_int64),
                ("n_pairs_gated", C.c_int64), ("n_pairs_exact", C.c_int64), ("max_rows_per_node", C.c_int64),
                ("last_run_ms", C.c_double), ("last_node_kernel_ms", C.c_double)]


class BAConfig(C.Structure):
    _fields_ = [("geometric_alpha", C.c_double), ("cauchy_scale", C.c_double),
                ("max_num_iterations", C.c_int32), ("min_num_images", C.c_int32),
                ("num_outliers", C.c_int32), ("max_num_consecutive_invalid_steps", C.c_int32),
                ("vp_multiplier", C.c_double)]


class VPConfig(C.Structure):
    _fields_ = [("min_length", C.c_double), ("inlier_threshold", C.c_double), ("th_perp_supports", C.c_double),
                ("min_num_supports", C.c_int32), ("n_models", C.c_int32), ("seed", C.c_uint64)]


class VPStats(C.Structure):
    _fields_ = [("n_images", C.c_int64), ("n_segments", C.c_int64), ("n_vps", C.c_int64), ("kernel_ms", C.c_double)]


class BAStats(C.Structure):
    _fields_ = [("n_tracks", C.c_int64), ("n_blocks", C.c_int64), ("total_iterations", C.c_int64),
                ("total_successful", C.c_int64), ("solve_ms", C.c_double), ("prepare_ms", C.c_double)]


class FilterConfig(C.Structure):
    _fields_ = [("th_angular_2d", C.c_double), ("th_perp_2d", C.c_double), ("th_sv_angular_3d", C.c_double),
                ("th_overlap", C.c_double)]


class MergeStats(C.Structure):
    _fields_ = [("n_supports", C.c_int64), ("n_tracks", C.c_int64), ("n_pairs_gated", C.c_int64),
                ("n_edges", C.c_int64), ("n_kernel_launches", C.c_int64), ("last_flags_ms", C.c_float),
                ("last_flags_kernel_ms", C.c_float), ("last_remerge_ms", C.c_float),
                ("last_remerge_kernel_ms", C.c_float)]


class FitMergeStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("n_lines", "n_nodes", "n_pairs_tested", "n_pairs_gated", "n_edges", "n_tracks",
                                         "n_retries")] + [("pair_kernel_ms", C.c_double), ("total_ms", C.c_double)]


NODE_RECORD_DTYPE = np.dtype([("line", np.float64, 9), ("score", np.float64), ("ng_view", np.int32),
                              ("ng_line", np.int32), ("n_cand", np.int32), ("n_valid", np.int32)])

_P = C.c_void_p
_SIGS = {
    "lm_last_error": (C.c_char_p, []),
    "lm_version": (C.c_char_p, []),
    "lm_ctx_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "lm_ctx_destroy": (None, [_P]),
    "lm_ctx_set_stream": (C.c_int, [_P, _P]),
    "lm_ctx_synchronize": (C.c_int, [_P]),
    "lm_scene_upload": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P]),
    "lm_tri_configure": (C.c_int, [_P, C.POINTER(TriConfig)]),
    "lm_tri_set_ranges": (C.c_int, [_P, _P, _P]),
    "lm_tri_unset_ranges": (C.c_int, [_P]),
    "lm_tri_set_vps": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P, _P]),
    "lm_tri_add_image_matches": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P]),
    "lm_tri_add_image_matches_device": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P]),
    "lm_tri_add_image_exhaustive": (C.c_int, [_P, C.c_int32, C.c_int32, _P]),
    "lm_tri_clear": (C.c_int, [_P]),
    "lm_tri_set_shard": (C.c_int, [_P, C.c_int32, C.c_int32]),
    "lm_tri_set_pipeline_groups": (C.c_int, [_P, C.c_int32]),
    "lm_tri_set_node_sink": (C.c_int, [_P, _P]),
    "lm_tri_run": (C.c_int, [_P]),
    "lm_tri_get_stats": (C.c_int, [_P, C.POINTER(TriStats)]),
    "lm_tri_get_best": (C.c_int, [_P, C.c_int32, _P, _P, _P]),
    "lm_tri_get_valid_edges": (C.c_int64, [_P, C.c_int32, _P, _P]),
    "lm_tri_get_cands_node": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "lm_tri_num_nodes": (C.c_int64, [_P]),
    "lm_tri_export_nodes": (C.c_int, [_P, C.c_int64, C.c_int64, _P]),
    "lm_tri_import_nodes": (C.c_int, [_P, C.c_int64, C.c_int64, _P]),
    "lm_tri_num_valid_edges": (C.c_int64, [_P]),
    "lm_tri_export_edges": (C.c_int, [_P, _P]),
    "lm_tri_import_edges": (C.c_int, [_P, C.c_int64, _P, C.c_int32]),
    "lm_scene_node_offset": (C.c_int64, [_P, C.c_int32]),
    "lm_tri_gather_message_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "lm_tri_pack_message": (C.c_int, [_P, C.c_int64, C.c_int64, _P]),
    "lm_tri_unpack_messages": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int64, _P]),
    "lm_tri_gather_status": (C.c_int64, [_P, C.POINTER(C.c_int64)]),
    "lm_tri_build_tracks": (C.c_int64, [_P, C.POINTER(C.c_int64)]),
    "lm_tri_get_tracks": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "lm_tri_add_matches_bulk": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P]),
    "lm_tri_get_nodes": (C.c_int, [_P, _P]),
    "lm_tri_get_all_valid_edges": (C.c_int64, [_P, _P, _P]),
    "lm_ba_solve": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "lm_ba_get_stats": (C.c_int, [_P, _P]),
    "lm_vp_detect": (C.c_int64, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, C.c_int64]),
    "lm_vp_detect_indexed": (C.c_int64, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_int64]),
    "lm_vp_get_stats": (C.c_int, [_P, _P]),
    "lm_sfm_rank_neighbors": (C.c_int, [_P, C.c_int32, _P, C.c_int64, _P, _P, _P, C.c_int32, C.c_double, C.c_int32, _P, _P]),
    "lm_sfm_robust_ranges": (C.c_int, [_P, C.c_int64, _P, C.c_double, C.c_double, C.c_double, _P]),
    "lm_tracks_support_flags": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P, _P, _P]),
    "lm_aggregate_lines": (C.c_int, [C.c_int64, _P, _P, _P, C.c_int32, _P]),
    "lm_remerge_labels": (C.c_int64, [_P, C.c_int64, _P, _P, _P, _P, _P]),
    "lm_merge_get_stats": (C.c_int, [_P, _P]),
    "lm_merge_fits_build": (C.c_int64, [_P, C.c_int32] + [_P] * 10 + [C.c_double, _P, _P, _P]),
    "lm_merge_fits_get": (C.c_int, [_P] * 9),
    "lm_merge_fits_get_stats": (C.c_int, [_P, _P]),
}
EXPORTED_SYMBOLS = tuple(_SIGS)


def lib():
    """Load liblimap_b200.so (built in-tree by __graft_entry__.build / limap_b200._build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LimapB200Error(
                f"{LIB_PATH} is missing: build the CUDA engine first (python -c 'import "
                "__graft_entry__ as g; g.build()'). limap_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc is not None and rc < 0:
        raise LimapB200Error(lib().lm_last_error().decode("utf-8", "replace"))
    return rc


def ptr(a):
    """Pointer of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return a.ctypes.data_as(C.c_void_p)


class Context:
    """Owns one lm_ctx (one CUDA device, one stream)."""

    def __init__(self, device=0):
        self._h = _P()
        check(lib().lm_ctx_create(int(device), C.byref(self._h)))
        self.device = device
        self._keep = []  # host arrays whose async copies may still be in flight

    def close(self):
        if self._h:
            lib().lm_ctx_destroy(self._h)
            self._h = _P()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_stream(self, cuda_stream):
        check(lib().lm_ctx_set_stream(self._h, C.c_void_p(int(cuda_stream))))

    def synchronize(self):
        check(lib().lm_ctx_synchronize(self._h))
        self._keep.clear()

    def stats(self):
        s = TriStats()
        check(lib().lm_tri_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in TriStats._fields_}
