"""limap.merging — the post-triangulation part of the reference's merging module on the CUDA engine.

Mirrors src/limap/merging/merging.py:24-83 (remerge, check_track_by_reprojection,
filter_tracks_by_reprojection, check_sensitivity, filter_tracks_by_sensitivity, filter_tracks_by_overlap) over
merging/merging_utils.cc:27-155 and merging/merging.cc:513-645. The per-support geometry and the O(T^2)
pair test run on the GPU (include/limap_b200.h); list surgery on LineTrack objects stays in Python like the
reference's std::vector code. `merging()` (MergeToLineTracks from per-image 3D segments, merging.py:6-21,
merging.cc:347-511), the merge step of the fit-and-merge pipeline, runs its O(lines^2 x neighbours) pair tests,
edge sorts and uncertainties on the GPU (lm_merge_fits_build); the union-find and the aggregation run on the host.
"""
import numpy as np

from . import base
from .config import LINKER2D_DEFAULTS, LINKER3D_DEFAULTS, make_linker
from .engine import MergeEngine

_engine = None


def _eng():
    global _engine
    if _engine is None:
        _engine = MergeEngine()
    return _engine


def _SetUncertaintySegs3d(lines, view, var2d):
    """merging_utils.cc:15-25: copies of the 3D lines with uncertainty = Line3d::computeUncertainty(view, var2d)."""
    out = []
    for l in lines:
        n = base.Line3d(l.start, l.end, l.score, l.depths[0], l.depths[1], l.uncertainty)
        n.set_uncertainty(n.computeUncertainty(view, var2d))
        out.append(n)
    return out


def _linker_cfg(cfg, defaults):
    d = cfg.as_dict() if hasattr(cfg, "as_dict") else dict(cfg or {})
    return make_linker(defaults, d)


def merging(linker, all_2d_segs, imagecols, seg3d_list, neighbors, var2d=5.0):
    """merging.py:6-21: SetUncertaintySegs3d per image, then MergeToLineTracks (merging.cc:347-511) on the GPU.
    linker: base.LineLinker; all_2d_segs[img_id]: (N, 4|5) segments; seg3d_list[img_id]: N (2, 3) fits, zeros where the
    fit failed; neighbors: {img_id: [img_id, ...]}. Returns (base.Graph, list of base.LineTrack)."""
    ids = imagecols.get_img_ids()
    if len(neighbors) != len(ids):  # THROW_CHECK_EQ(all_lines_2d.size(), neighbors.size())
        raise RuntimeError(f"Check failed: all_lines_2d.size() == neighbors.size() ({len(ids)} vs. {len(neighbors)})")
    segs, fits, line_off = [], [], [0]
    for img_id in ids:
        s2 = np.asarray(all_2d_segs[img_id], np.float64)
        if s2.ndim != 2 or (s2.shape[0] != 0 and s2.shape[1] < 4):
            raise RuntimeError("THROW_CHECK_GE(segs2d.cols(), 4)")
        f3 = np.asarray(seg3d_list[img_id], np.float64).reshape(-1, 2, 3)
        if len(f3) != len(s2):  # THROW_CHECK_EQ(all_lines_2d.at(image_id).size(), all_lines_3d.at(image_id).size())
            raise RuntimeError(f"Check failed: 2D lines ({len(s2)}) and 3D lines ({len(f3)}) of image {img_id} differ")
        segs.append(s2[:, :4].reshape(-1, 4))
        fits.append(f3)
        line_off.append(line_off[-1] + len(s2))
    ng_off, ng_ids = [0], []
    for img_id in ids:
        if img_id not in neighbors:
            raise IndexError("map::at")  # neighbors.at(image_id)
        for j in neighbors[img_id]:
            if not imagecols.exist_image(int(j)):
                raise IndexError("map::at")  # all_lines_2d.at(ng_image_id)
            ng_ids.append(int(j))
        ng_off.append(len(ng_ids))
    l2 = _linker_cfg(linker.linker_2d.config, LINKER2D_DEFAULTS)
    l3 = _linker_cfg(linker.linker_3d.config, LINKER3D_DEFAULTS)
    img_ids, model, kvec, qvec, tvec = imagecols.arrays()
    r = _eng().merge_fits(img_ids, model, kvec, qvec, tvec, np.asarray(line_off, np.int64),
                          np.concatenate(segs) if segs else np.zeros((0, 4)),
                          np.concatenate(fits) if fits else np.zeros((0, 2, 3)),
                          np.asarray(ng_off, np.int64), np.asarray(ng_ids, np.int32), var2d, l2, l3)
    line_off = np.asarray(line_off, np.int64)
    view = np.searchsorted(line_off, r["node_line"], side="right") - 1
    node_img = np.asarray(ids, np.int64)[view] if len(view) else np.zeros(0, np.int64)
    node_lid = r["node_line"] - line_off[view] if len(view) else np.zeros(0, np.int64)
    graph = base.Graph(node_img, node_lid, r["edges"][:, 0], r["edges"][:, 1], r["sim"])
    flat_segs = np.concatenate(segs) if segs else np.zeros((0, 4))
    flat_fits = np.concatenate(fits) if fits else np.zeros((0, 2, 3))
    tracks = []
    for t in range(len(r["track_off"]) - 1):
        tr = base.LineTrack()
        for k in r["track_nodes"][r["track_off"][t]:r["track_off"][t + 1]].tolist():
            g = int(r["node_line"][k])
            l3d = base.Line3d(flat_fits[g, 0], flat_fits[g, 1], uncertainty=r["unc"][g])
            tr.node_id_list.append(k)
            tr.image_id_list.append(int(node_img[k]))
            tr.line_id_list.append(int(node_lid[k]))
            tr.line2d_list.append(base.Line2d(flat_segs[g, :2], flat_segs[g, 2:4]))
            tr.line3d_list.append(l3d)
            tr.score_list.append(float(r["length"][g]))  # Line3d::length() (merging.cc:493)
        tl = r["track_line"][t]
        tr.line = base.Line3d(tl[:3], tl[3:6], uncertainty=tl[6])
        tracks.append(tr)
    return graph, tracks


def _flatten(linetracks, imagecols):
    ids, model, kvec, qvec, tvec = imagecols.arrays()
    view_of = {int(i): v for v, i in enumerate(ids)}
    T = len(linetracks)
    sup_off = np.zeros(T + 1, np.int64)
    for t, tr in enumerate(linetracks):
        sup_off[t + 1] = sup_off[t] + tr.count_lines()
    S = int(sup_off[-1])
    sup_view = np.zeros(S, np.int32)
    segs = np.zeros((S, 4))
    track_line = np.zeros((T, 6))
    k = 0
    for t, tr in enumerate(linetracks):
        track_line[t, :3], track_line[t, 3:] = tr.line.start, tr.line.end
        for img_id, l2d in zip(tr.image_id_list, tr.line2d_list):
            sup_view[k] = view_of[int(img_id)]
            segs[k, :2], segs[k, 2:] = l2d.start, l2d.end
            k += 1
    return model, kvec, qvec, tvec, sup_off, sup_view, segs, track_line


def _flags(linetracks, imagecols, **th):
    if len(linetracks) == 0:
        return np.zeros(0, np.uint8), np.zeros(1, np.int64)
    arr = _flatten(linetracks, imagecols)
    return _eng().support_flags(*arr, **th), arr[4]


def _aggregate(tracks, num_outliers):
    """Aggregator::aggregate_line3d_list of every track's (line3d_list, score_list) -> track.line."""
    off = np.zeros(len(tracks) + 1, np.int64)
    for t, tr in enumerate(tracks):
        off[t + 1] = off[t] + len(tr.line3d_list)
    lines = np.zeros((int(off[-1]), 7))
    scores = np.zeros(int(off[-1]))
    k = 0
    for tr in tracks:
        for l3, sc in zip(tr.line3d_list, tr.score_list):
            lines[k, :3], lines[k, 3:6], lines[k, 6] = l3.start, l3.end, l3.uncertainty
            scores[k] = sc
            k += 1
    out = MergeEngine.aggregate(off, lines, scores, num_outliers)
    for t, tr in enumerate(tracks):
        tr.line = base.Line3d(out[t, :3], out[t, 3:6], uncertainty=out[t, 6])


def check_track_by_reprojection(track, imagecols, th_angular2d, th_perp2d):
    """merging.py:45-47 / CheckReprojection (merging_utils.cc:27-50): list of bool per supporting line."""
    f, _ = _flags([track], imagecols, th_angular_2d=th_angular2d, th_perp_2d=th_perp2d)
    return [bool(x & 1) for x in f]


def filter_tracks_by_reprojection(linetracks, imagecols, th_angular2d, th_perp2d, num_outliers=2):
    """merging.py:50-61 / FilterSupportingLines (merging_utils.cc:52-87)."""
    f, off = _flags(linetracks, imagecols, th_angular_2d=th_angular2d, th_perp_2d=th_perp2d)
    out = []
    for t, tr in enumerate(linetracks):
        keep = [k for k in range(tr.count_lines()) if f[off[t] + k] & 1]
        if not keep:
            continue
        nt = base.LineTrack()
        nt.node_id_list = [tr.node_id_list[k] for k in keep]
        nt.image_id_list = [tr.image_id_list[k] for k in keep]
        nt.line_id_list = [tr.line_id_list[k] for k in keep]
        nt.line2d_list = [tr.line2d_list[k] for k in keep]
        nt.line3d_list = [tr.line3d_list[k] for k in keep]
        nt.score_list = [tr.score_list[k] for k in keep]
        out.append(nt)
    _aggregate(out, num_outliers)
    return out


def check_sensitivity(linetrack, imagecols, th_angular3d):
    """merging.py:64-66 / CheckSensitivity (merging_utils.cc:89-109)."""
    f, _ = _flags([linetrack], imagecols, th_sv_angular_3d=th_angular3d)
    return [bool(x & 2) for x in f]


def _filter_by_count(linetracks, f, off, bit, min_num_supports):
    out = []
    for t, tr in enumerate(linetracks):
        imgs = {tr.image_id_list[k] for k in range(tr.count_lines()) if f[off[t] + k] & bit}
        if len(imgs) >= min_num_supports:
            out.append(tr)
    return out


def filter_tracks_by_sensitivity(linetracks, imagecols, th_angular3d, min_num_supports):
    """merging.py:69-75 / FilterTracksBySensitivity (merging_utils.cc:111-131)."""
    f, off = _flags(linetracks, imagecols, th_sv_angular_3d=th_angular3d)
    return _filter_by_count(linetracks, f, off, 2, min_num_supports)


def filter_tracks_by_overlap(linetracks, imagecols, th_overlap, min_num_supports):
    """merging.py:78-83 / FilterTracksByOverlap (merging_utils.cc:133-155)."""
    f, off = _flags(linetracks, imagecols, th_overlap=th_overlap)
    return _filter_by_count(linetracks, f, off, 4, min_num_supports)


def _remerge_once(linetracks, linker_cfg, num_outliers):
    """RemergeLineTracks (merging.cc:513-645)."""
    T = len(linetracks)
    track_line = np.zeros((T, 7))
    active = np.zeros(T, np.uint8)
    for t, tr in enumerate(linetracks):
        track_line[t, :3], track_line[t, 3:6], track_line[t, 6] = tr.line.start, tr.line.end, tr.line.uncertainty
        active[t] = 1 if tr.active else 0
    labels, n_groups, _ = _eng().remerge_labels(track_line, active, linker_cfg)
    new = [base.LineTrack() for _ in range(n_groups)]
    counter = [0] * n_groups
    for t, tr in enumerate(linetracks):
        g = int(labels[t])
        counter[g] += 1
        new[g].node_id_list += list(tr.node_id_list)
        new[g].image_id_list += list(tr.image_id_list)
        new[g].line_id_list += list(tr.line_id_list)
        new[g].line2d_list += list(tr.line2d_list)
        new[g].line3d_list += list(tr.line3d_list)
        new[g].score_list += list(tr.score_list)
    _aggregate(new, num_outliers)
    for g in range(n_groups):
        if counter[g] == 1:
            new[g].active = False
    return new


def remerge(linker3d, linetracks, num_outliers=2):
    """merging.py:24-42: iterate RemergeLineTracks until the number of tracks stops changing."""
    if len(linetracks) == 0:
        return linetracks
    cfg = linker3d.config if hasattr(linker3d, "config") else linker3d
    d = cfg.as_dict() if hasattr(cfg, "as_dict") else dict(cfg)
    linker_cfg = make_linker(LINKER3D_DEFAULTS, d)
    new_linetracks = linetracks
    num_tracks = len(new_linetracks)
    while True:
        new_linetracks = _remerge_once(new_linetracks, linker_cfg, num_outliers)
        if num_tracks == len(new_linetracks):
            break
        num_tracks = len(new_linetracks)
    return new_linetracks
