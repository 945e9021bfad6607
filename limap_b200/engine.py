"""Array-level Python face of the CUDA engine (one lm_ctx). The limap-style classes in
limap_b200.triangulation wrap this; bench.py and the parity tests call it directly."""
import ctypes as C

import numpy as np

from . import _cabi
from .config import make_tri_config
from ._cabi import Context, check, lib, ptr


class TriEngine:
    """GlobalLineTriangulator on flat arrays (src/limap/triangulation/global_line_triangulator.h:27-93)."""

    def __init__(self, cfg=None, device=0):
        self.ctx = Context(device)
        self.cfg = make_tri_config(cfg) if not hasattr(cfg, "_fields_") else cfg
        check(lib().lm_tri_configure(self.ctx.handle, C.byref(self.cfg)))
        self.img_ids = None
        self.line_off = None

    # ---- scene ---------------------------------------------------------------------------------
    def upload_scene(self, img_ids, model_ids, kvec, qvec, tvec, line_off, segs):
        img_ids = np.ascontiguousarray(img_ids, np.int32)
        model_ids = np.ascontiguousarray(model_ids, np.int32)
        kvec = np.ascontiguousarray(kvec, np.float64)
        qvec = np.ascontiguousarray(qvec, np.float64)
        tvec = np.ascontiguousarray(tvec, np.float64)
        line_off = np.ascontiguousarray(line_off, np.int64)
        segs = np.ascontiguousarray(segs, np.float64)
        check(lib().lm_scene_upload(self.ctx.handle, len(img_ids), ptr(img_ids), ptr(model_ids),
                                    ptr(kvec), ptr(qvec), ptr(tvec), ptr(line_off), ptr(segs)))
        self.img_ids = img_ids
        self.line_off = line_off
        self._segs_ref = segs  # a pinned buffer is copied asynchronously: keep it alive until the next upload
        self._view = {int(i): v for v, i in enumerate(img_ids)}

    def upload(self, scene):
        self.upload_scene(scene.img_ids, scene.model_ids, scene.kvec, scene.qvec, scene.tvec,
                          scene.line_off, scene.segs)

    def n_lines(self, img_id):
        v = self._view[int(img_id)]
        return int(self.line_off[v + 1] - self.line_off[v])

    def set_ranges(self, lo, hi):
        lo = np.ascontiguousarray(lo, np.float64)
        hi = np.ascontiguousarray(hi, np.float64)
        check(lib().lm_tri_set_ranges(self.ctx.handle, ptr(lo), ptr(hi)))

    def unset_ranges(self):
        check(lib().lm_tri_unset_ranges(self.ctx.handle))

    def set_vps(self, vpresults, img_ids, line_off):
        """InitVPResults: {img_id: VPResult-like with .labels and .vps}."""
        ids = [int(i) for i in img_ids if int(i) in vpresults]
        label_off, vp_off, labels, vps = [0], [0], [], []
        for i in ids:
            r = vpresults[i]
            lab = np.asarray(r.labels, np.int32).reshape(-1)
            v = np.asarray(r.vps, np.float64).reshape(-1, 3)
            labels.append(lab)
            vps.append(v)
            label_off.append(label_off[-1] + len(lab))
            vp_off.append(vp_off[-1] + len(v))
        labels = np.concatenate(labels) if labels else np.zeros(0, np.int32)
        vps = np.concatenate(vps) if vps else np.zeros((0, 3))
        ids_a = np.asarray(ids, np.int32)
        lo, vo = np.asarray(label_off, np.int64), np.asarray(vp_off, np.int64)
        check(lib().lm_tri_set_vps(self.ctx.handle, len(ids), ptr(ids_a), ptr(lo), ptr(np.ascontiguousarray(labels)),
                                   ptr(vo), ptr(np.ascontiguousarray(vps))))

    # ---- TriangulateImage ----------------------------------------------------------------------
    def add_image_matches(self, img_id, ng_ids, row_off, pairs):
        ng_ids = np.ascontiguousarray(ng_ids, np.int32)
        row_off = np.ascontiguousarray(row_off, np.int64)
        pairs = np.ascontiguousarray(pairs, np.int32)
        self.ctx._keep.append(pairs)  # the H2D copy is asynchronous when `pairs` is pinned
        check(lib().lm_tri_add_image_matches(self.ctx.handle, int(img_id), len(ng_ids), ptr(ng_ids),
                                             ptr(row_off), ptr(pairs)))

    def add_image_matches_device(self, img_id, ng_ids, row_off, d_pairs_ptr):
        ng_ids = np.ascontiguousarray(ng_ids, np.int32)
        row_off = np.ascontiguousarray(row_off, np.int64)
        check(lib().lm_tri_add_image_matches_device(self.ctx.handle, int(img_id), len(ng_ids),
                                                    ptr(ng_ids), ptr(row_off), C.c_void_p(int(d_pairs_ptr))))

    def add_image_matches_torch(self, img_id, matches):
        """matches: {ng_img_id: (M,2) integer torch tensor on this engine's CUDA device} -- the top-k output of a GPU
        matcher (line2d/endpoints/matcher.py:87-103) goes into the match store device-to-device, no host hop."""
        import torch
        ngs = sorted(matches.keys())
        row_off = np.zeros(len(ngs) + 1, np.int64)
        parts = []
        for i, g in enumerate(ngs):
            m = matches[g]
            if m.numel() and (m.dim() != 2 or m.shape[1] != 2):
                raise RuntimeError("match_info.cols() must be 2")
            if not m.is_cuda or m.device.index != self.ctx.device:
                raise RuntimeError(f"matches must live on cuda:{self.ctx.device}")
            parts.append(m.reshape(-1, 2).to(torch.int32))
            row_off[i + 1] = row_off[i] + parts[-1].shape[0]
        if parts:
            pairs = torch.cat(parts, 0).contiguous()
        else:
            pairs = torch.zeros((0, 2), dtype=torch.int32, device=f"cuda:{self.ctx.device}")
        torch.cuda.current_stream(pairs.device).synchronize()  # the engine copies on its own stream
        self.ctx._keep.append(pairs)
        self.add_image_matches_device(img_id, np.asarray(ngs, np.int32), row_off, pairs.data_ptr())

    def add_image_matches_dict(self, img_id, matches):
        """matches: {ng_img_id: (M,2) int array}; neighbours are visited in ascending id order
        (std::map iteration, base_line_triangulator.cc:74)."""
        ngs = sorted(matches.keys())
        row_off = np.zeros(len(ngs) + 1, np.int64)
        parts = []
        for i, g in enumerate(ngs):
            m = np.asarray(matches[g])
            if m.size and (m.ndim != 2 or m.shape[1] != 2):
                raise RuntimeError("match_info.cols() must be 2")  # THROW_CHECK_EQ(cols, 2)
            m = m.reshape(-1, 2)
            parts.append(m.astype(np.int32, copy=False))
            row_off[i + 1] = row_off[i] + len(m)
        pairs = np.concatenate(parts, 0) if parts else np.zeros((0, 2), np.int32)
        self.add_image_matches(img_id, np.asarray(ngs, np.int32), row_off, pairs)

    def add_matches_bulk(self, src_ids, ng_ids, row_off, pairs):
        """Many (image, neighbour) match tables in one call (lm_tri_add_matches_bulk)."""
        src_ids = np.ascontiguousarray(src_ids, np.int32)
        ng_ids = np.ascontiguousarray(ng_ids, np.int32)
        row_off = np.ascontiguousarray(row_off, np.int64)
        pairs = np.ascontiguousarray(pairs, np.int32)
        self.ctx._keep.append(pairs)
        check(lib().lm_tri_add_matches_bulk(self.ctx.handle, len(src_ids), ptr(src_ids), ptr(ng_ids), ptr(row_off),
                                            ptr(pairs)))

    def get_nodes(self, out=None):
        """All node records as a structured array (NODE_RECORD_DTYPE)."""
        n = int(self.line_off[-1])
        if out is None:
            out = np.zeros(n, _cabi.NODE_RECORD_DTYPE)
        check(lib().lm_tri_get_nodes(self.ctx.handle, ptr(out)))
        return out

    def get_all_valid_edges(self, off=None, edges=None):
        """(node_off[n_nodes+1], edges[n,2] = (ng_img_id, ng_line_id)); pass preallocated (pinned) arrays to
        avoid staging copies."""
        n = int(self.line_off[-1])
        # the count call runs the pending work first (ensure_ran), so `ne` is never stale
        ne = int(check(lib().lm_tri_get_all_valid_edges(self.ctx.handle, None, None)))
        if edges is not None and len(edges) < ne:
            raise ValueError(f"edges buffer holds {len(edges)} rows, {ne} valid connections to return")
        if off is not None and len(off) < n + 1:
            raise ValueError(f"off buffer holds {len(off)} entries, {n + 1} needed")
        if off is None:
            off = np.zeros(n + 1, np.int64)
        if edges is None:
            edges = np.zeros((max(ne, 1), 2), np.int32)
        check(lib().lm_tri_get_all_valid_edges(self.ctx.handle, ptr(off), ptr(edges)))
        return off, edges[:ne]

    def add_image_exhaustive(self, img_id, neighbors):
        ng = np.ascontiguousarray(neighbors, np.int32)
        check(lib().lm_tri_add_image_exhaustive(self.ctx.handle, int(img_id), len(ng), ptr(ng)))

    def clear(self):
        check(lib().lm_tri_clear(self.ctx.handle))
        self.ctx._keep.clear()

    def set_shard(self, view_begin, view_end):
        check(lib().lm_tri_set_shard(self.ctx.handle, int(view_begin), int(view_end)))

    def set_pipeline_groups(self, n_groups):
        check(lib().lm_tri_set_pipeline_groups(self.ctx.handle, int(n_groups)))

    def run(self, nodes_out=None):
        """Run the enqueued work. `nodes_out` (a NODE_RECORD_DTYPE array over all 2D lines of the scene, ideally pinned)
        receives the node records of this run's shard while the run is still going (lm_tri_set_node_sink)."""
        if nodes_out is not None:
            if nodes_out.dtype != _cabi.NODE_RECORD_DTYPE or len(nodes_out) != int(self.line_off[-1]) or \
                    not nodes_out.flags.c_contiguous:
                raise ValueError("nodes_out must be a contiguous NODE_RECORD_DTYPE array with one record per 2D line")
            check(lib().lm_tri_set_node_sink(self.ctx.handle, ptr(nodes_out)))
        try:
            check(lib().lm_tri_run(self.ctx.handle))
        finally:
            if nodes_out is not None:
                check(lib().lm_tri_set_node_sink(self.ctx.handle, None))
        self.ctx._keep.clear()
        return self.ctx.stats()

    # ---- results -------------------------------------------------------------------------------
    def get_best(self, img_id):
        L = self.n_lines(img_id)
        line = np.zeros((L, 10), np.float64)
        ng = np.zeros((L, 2), np.int32)
        ncand = np.zeros(L, np.int32)
        check(lib().lm_tri_get_best(self.ctx.handle, int(img_id), ptr(line), ptr(ng), ptr(ncand)))
        return line, ng, ncand

    def get_valid_edges(self, img_id):
        L = self.n_lines(img_id)
        off = np.zeros(L + 1, np.int64)
        n = check(lib().lm_tri_get_valid_edges(self.ctx.handle, int(img_id), ptr(off), None))
        edges = np.zeros((max(n, 1), 2), np.int32)
        check(lib().lm_tri_get_valid_edges(self.ctx.handle, int(img_id), ptr(off), ptr(edges)))
        return off, edges[:n]

    def get_cands_node(self, img_id, line_id, cap=4096):
        line = np.zeros((cap, 10), np.float64)
        ng = np.zeros((cap, 2), np.int32)
        n = check(lib().lm_tri_get_cands_node(self.ctx.handle, int(img_id), int(line_id), cap,
                                              ptr(line), ptr(ng)))
        if n > cap:
            return self.get_cands_node(img_id, line_id, cap=n)
        return line[:n], ng[:n]

    def build_tracks(self):
        tot = C.c_int64(0)
        T = check(lib().lm_tri_build_tracks(self.ctx.handle, C.byref(tot)))
        n = tot.value
        track_off = np.zeros(T + 1, np.int64)
        img = np.zeros(max(n, 1), np.int32)
        line = np.zeros(max(n, 1), np.int32)
        node = np.zeros(max(n, 1), np.int32)
        l3d = np.zeros((max(n, 1), 10), np.float64)
        tl = np.zeros((max(T, 1), 7), np.float64)
        check(lib().lm_tri_get_tracks(self.ctx.handle, ptr(track_off), ptr(img), ptr(line), ptr(node),
                                      ptr(l3d), ptr(tl)))
        return dict(track_off=track_off, img_ids=img[:n], line_ids=line[:n], node_ids=node[:n],
                    line3d=l3d[:n], track_line=tl[:T])

    def stats(self):
        return self.ctx.stats()

    def close(self):
        self.ctx.close()


class BAEngine:
    """Batched line refinement / line bundle adjustment with constant cameras on flat arrays
    (HybridBAEngine / RefinementEngine, see include/limap_b200.h lm_ba_solve)."""

    def __init__(self, device=0, ctx=None):
        self.ctx = ctx if ctx is not None else Context(device)

    def solve(self, kvec, qvec, tvec, sup_off, sup_view, segs, line3d, line_init, max_num_iterations=100,
              min_num_images=4, num_outliers=2, geometric_alpha=10.0, cauchy_scale=0.25,
              max_num_consecutive_invalid_steps=10, sup_vp=None, vp_multiplier=1.0):
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        kvec, qvec, tvec, segs, line3d, line_init = map(f64, (kvec, qvec, tvec, segs, line3d, line_init))
        sup_off = np.ascontiguousarray(sup_off, np.int64)
        sup_view = np.ascontiguousarray(sup_view, np.int32)
        T = len(sup_off) - 1
        cfg = _cabi.BAConfig(geometric_alpha, cauchy_scale, max_num_iterations, min_num_images, num_outliers,
                             max_num_consecutive_invalid_steps, float(vp_multiplier))
        sup_vp = None if sup_vp is None else f64(sup_vp)
        out_line = np.zeros((T, 6))
        out_min = np.zeros((T, 6))
        iters = np.zeros((T, 2), np.int32)
        cost = np.zeros((T, 2))
        check(lib().lm_ba_solve(self.ctx.handle, len(kvec), ptr(kvec), ptr(qvec), ptr(tvec), T, ptr(sup_off),
                                ptr(sup_view), ptr(segs), ptr(line3d), ptr(line_init), ptr(sup_vp), C.byref(cfg),
                                ptr(out_line), ptr(out_min), ptr(iters), ptr(cost)))
        st = _cabi.BAStats()
        check(lib().lm_ba_get_stats(self.ctx.handle, C.byref(st)))
        stats = {k: getattr(st, k) for k, _ in _cabi.BAStats._fields_}
        return dict(line=out_line, minimal=out_min, iters=iters, cost=cost, stats=stats)

    def solve_trackset(self, ts, **kw):
        """TrackSet (limap_b200.synth.make_tracks) carries per-support cameras; dedupe them into a view table."""
        views, first_idx = np.unique(ts.img_ids, return_index=True)
        remap = np.zeros(int(views.max()) + 1, np.int32)
        remap[views] = np.arange(len(views), dtype=np.int32)
        return self.solve(ts.kvec[first_idx], ts.qvec[first_idx], ts.tvec[first_idx], ts.sup_off,
                          remap[ts.img_ids], ts.segs, ts.line3d, ts.line_init, **kw)


class MergeEngine:
    """Track filters, remerge and the fit-and-merge track build on flat arrays (include/limap_b200.h:
    lm_tracks_support_flags, lm_remerge_labels, lm_aggregate_lines, lm_merge_fits_build)."""

    def __init__(self, device=0, ctx=None):
        self.ctx = ctx if ctx is not None else Context(device)

    def support_flags(self, model_ids, kvec, qvec, tvec, sup_off, sup_view, segs, track_line, th_angular_2d=8.0,
                      th_perp_2d=5.0, th_sv_angular_3d=75.0, th_overlap=0.5):
        """uint8 per support: bit0 reprojection ok, bit1 sensitivity ok, bit2 overlap ok."""
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        kvec, qvec, tvec, segs, track_line = map(f64, (kvec, qvec, tvec, segs, track_line))
        model_ids = None if model_ids is None else np.ascontiguousarray(model_ids, np.int32)
        sup_off = np.ascontiguousarray(sup_off, np.int64)
        sup_view = np.ascontiguousarray(sup_view, np.int32)
        T = len(sup_off) - 1
        flags = np.zeros(int(sup_off[-1]), np.uint8)
        cfg = _cabi.FilterConfig(th_angular_2d, th_perp_2d, th_sv_angular_3d, th_overlap)
        check(lib().lm_tracks_support_flags(self.ctx.handle, len(kvec), ptr(model_ids), ptr(kvec), ptr(qvec), ptr(tvec),
                                            T, ptr(sup_off), ptr(sup_view), ptr(segs), ptr(track_line), C.byref(cfg),
                                            ptr(flags)))
        return flags

    def remerge_labels(self, track_line, active, linker3d):
        """(labels[T], n_groups, n_edges) of one RemergeLineTracks pass; linker3d: config.LinkerConfig."""
        track_line = np.ascontiguousarray(track_line, np.float64)
        active = np.ascontiguousarray(active, np.uint8)
        T = len(track_line)
        labels = np.zeros(T, np.int32)
        ne = C.c_int64(0)
        ng = check(lib().lm_remerge_labels(self.ctx.handle, T, ptr(track_line), ptr(active), C.byref(linker3d),
                                           ptr(labels), C.byref(ne)))
        return labels, int(ng), int(ne.value)

    def merge_fits(self, img_ids, model_ids, kvec, qvec, tvec, line_off, segs, lines3d, ng_off, ng_ids, var2d,
                   linker2d, linker3d):
        """MergeToLineTracks on flat arrays (lm_merge_fits_build); linker2d / linker3d: config.LinkerConfig. Returns
        dict(unc, length, node_line, edges, sim, track_off, track_nodes, track_line)."""
        i32 = lambda a: np.ascontiguousarray(a, np.int32)
        i64 = lambda a: np.ascontiguousarray(a, np.int64)
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        segs = np.asarray(segs, np.float64).reshape(-1, np.shape(segs)[-1] if np.size(segs) else 4)[:, :4]
        a = [i32(img_ids), i32(model_ids), f64(kvec), f64(qvec), f64(tvec), i64(line_off), f64(segs),
             f64(lines3d).reshape(-1, 6), i64(ng_off), i32(ng_ids)]
        counts = np.zeros(3, np.int64)
        T = check(lib().lm_merge_fits_build(self.ctx.handle, len(a[0]), *[ptr(x) for x in a], float(var2d),
                                            C.byref(linker2d), C.byref(linker3d), ptr(counts)))
        nn, ne, ns = (int(x) for x in counts)
        out = dict(unc=np.zeros(int(a[5][-1])), length=np.zeros(int(a[5][-1])), node_line=np.zeros(nn, np.int64), edges=np.zeros((ne, 2), np.int32),
                   sim=np.zeros(ne), track_off=np.zeros(T + 1, np.int64), track_nodes=np.zeros(ns, np.int32),
                   track_line=np.zeros((T, 7)))
        check(lib().lm_merge_fits_get(self.ctx.handle, *[ptr(out[k]) for k in (
            "unc", "length", "node_line", "edges", "sim", "track_off", "track_nodes", "track_line")]))
        return out

    def fit_merge_stats(self):
        st = _cabi.FitMergeStats()
        check(lib().lm_merge_fits_get_stats(self.ctx.handle, C.byref(st)))
        return {k: getattr(st, k) for k, _ in _cabi.FitMergeStats._fields_}

    @staticmethod
    def aggregate(off, lines, scores, num_outliers):
        off = np.ascontiguousarray(off, np.int64)
        lines = np.ascontiguousarray(lines, np.float64)
        scores = np.ascontiguousarray(scores, np.float64)
        out = np.zeros((len(off) - 1, 7))
        check(lib().lm_aggregate_lines(len(off) - 1, ptr(off), ptr(lines), ptr(scores), int(num_outliers), ptr(out)))
        return out

    def stats(self):
        st = _cabi.MergeStats()
        check(lib().lm_merge_get_stats(self.ctx.handle, C.byref(st)))
        return {k: getattr(st, k) for k, _ in _cabi.MergeStats._fields_}
