"""limap.runners as far as the triangulation and localization paths need it: `setup`, the LOAD branches of `compute_2d_segs` /
`compute_matches` (detections and matches come from disk or from a GPU matcher; the learned front end is out of scope)
and `line_triangulation` -- the steps of src/limap/runners/line_triangulation.py:18-245 ([A] metainfos, [B] segments,
[C] matches, [D] triangulation + track filters + remerge, [E] line bundle adjustment, [F] output + track report) driven
through this package's operator surface, and `hybrid_localization` (src/limap/runners/hybrid_localization.py:94-398) with
the epipolar matcher or loaded learned matches and the ransac.method None estimator. tests/test_runner_dropin.py additionally executes the reference's own runner
file, unmodified and loaded by path, against the same surface."""
import logging
import os

import numpy as np

from . import base, estimators, merging, optimize, triangulation, visualize, vplib
from . import hybrid_localization_functions as _locfn
from .util import io as limapio

_log = logging.getLogger("limap_b200")


def setup(cfg):  # runners/functions.py:11-28
    folder_save = cfg["output_dir"] or "tmp"
    limapio.check_makedirs(folder_save)
    folder_load = "tmp" if cfg.get("use_tmp") else cfg.get("load_dir")
    cfg["dir_save"] = folder_save
    cfg["dir_load"] = folder_load if folder_load is not None else folder_save
    return cfg


def _out_of_scope(what):
    def f(*a, **k):
        raise NotImplementedError(f"{what} is outside the hot path (SURVEY.md §2); provide the artefacts and set "
                                  "load_det / load_match, or pass neighbors and ranges")
    return f


undistort_images = _out_of_scope("image undistortion")
compute_sfminfos = _out_of_scope("COLMAP neighbours / ranges")
compute_2d_bipartites_from_colmap = _out_of_scope("point-line bipartites from a COLMAP model")
compute_exhaustive_matches = _out_of_scope("descriptor matching")
get_hloc_keypoints = _out_of_scope("hloc keypoint correspondences")
get_hloc_keypoints_from_log = _out_of_scope("hloc localization logs")


def segments_folder(cfg, root):
    """<root>/line_detections/<detector>/segments (runners/functions.py:232-235, line2d/base_detector.py:155-164)."""
    return os.path.join(root, "line_detections", cfg["line2d"]["detector"]["method"], "segments")


def matches_folder(cfg, root):
    """<root>/line_matchings/<detector>/feats_<extractor>/<matcher>_n<neighbours>_top<k>
    (runners/functions.py:316-320, line2d/base_matcher.py:60-72)."""
    m = cfg["line2d"]["matcher"]
    return os.path.join(root, "line_matchings", cfg["line2d"]["detector"]["method"],
                        "feats_{}".format(cfg["line2d"]["extractor"]["method"]),
                        "{}_n{}_top{}".format(m["method"], cfg["n_neighbors"], m.get("topk", 10)))


def compute_2d_segs(cfg, imagecols, compute_descinfo=True):  # runners/functions.py:197-290, load branch
    if not cfg["load_det"]:
        return _out_of_scope("2D line detection")()
    segs = limapio.read_all_segments_from_folder(segments_folder(cfg, cfg["dir_load"]))
    return {i: segs[i] for i in imagecols.get_img_ids()}, None


def compute_matches(cfg, descinfo_folder, image_ids, neighbors):  # runners/functions.py:293-345, load branch
    if not cfg["load_match"]:
        return _out_of_scope("2D line matching")()
    return matches_folder(cfg, cfg["dir_load"])


def line_triangulation(cfg, imagecols, neighbors=None, ranges=None):
    """Main interface of line triangulation over multi-view images (runners/line_triangulation.py:18-245)."""
    cfg = setup(cfg)
    tcfg = cfg["triangulation"]
    if tcfg["var2d"] == -1:
        tcfg["var2d"] = cfg["var2d"][cfg["line2d"]["detector"]["method"]]
    if not imagecols.IsUndistorted():
        imagecols = undistort_images(imagecols)
    if cfg.get("max_image_dim") not in (-1, None):
        imagecols.set_max_image_dim(cfg["max_image_dim"])
    save = cfg["dir_save"]
    limapio.save_txt_imname_dict(os.path.join(save, "image_list.txt"), imagecols.get_image_name_dict())
    limapio.save_npy(os.path.join(save, "imagecols.npy"), imagecols.as_dict())
    # [A] neighbours and ranges
    if neighbors is None:
        _, neighbors, ranges = compute_sfminfos(cfg, imagecols)
    else:
        neighbors = imagecols.update_neighbors(neighbors)
        neighbors = {i: list(n)[: cfg["n_neighbors"]] for i, n in neighbors.items()}
    limapio.save_txt_metainfos(os.path.join(save, "metainfos.txt"), neighbors, ranges)
    # [B] segments, [C] matches
    all_2d_segs, descinfo_folder = compute_2d_segs(cfg, imagecols, compute_descinfo=False)
    exhaustive = tcfg["use_exhaustive_matcher"]
    matches_dir = None if exhaustive else compute_matches(cfg, descinfo_folder, imagecols.get_img_ids(), neighbors)
    # [D] triangulation
    tri = triangulation.GlobalLineTriangulator(tcfg)
    tri.SetRanges(ranges)
    all_2d_lines = base.get_all_lines_2d(all_2d_segs)
    tri.Init(all_2d_lines, imagecols)
    if tcfg["use_vp"]:
        det = vplib.get_vp_detector(tcfg["vpdet_config"], n_jobs=tcfg["vpdet_config"]["n_jobs"])
        tri.InitVPResults(det.detect_vp_all_images(all_2d_lines, imagecols.get_map_camviews()))
    if tcfg["use_pointsfm"]["enable"]:
        compute_2d_bipartites_from_colmap()
    for img_id in imagecols.get_img_ids():
        if exhaustive:
            tri.TriangulateImageExhaustiveMatch(img_id, neighbors[img_id])
        else:
            tri.TriangulateImage(img_id, limapio.read_npy(os.path.join(matches_dir, f"matches_{img_id}.npy")).item())
    linetracks = tri.ComputeLineTracks()
    f2d = tcfg["filtering2d"]
    linetracks = merging.filter_tracks_by_reprojection(linetracks, imagecols, f2d["th_angular_2d"], f2d["th_perp_2d"])
    if not tcfg["remerging"]["disable"]:
        linetracks = merging.remerge(base.LineLinker3d(tcfg["remerging"]["linker3d"]), linetracks)
        linetracks = merging.filter_tracks_by_reprojection(linetracks, imagecols, f2d["th_angular_2d"], f2d["th_perp_2d"])
    linetracks = merging.filter_tracks_by_sensitivity(linetracks, imagecols, f2d["th_sv_angular_3d"], f2d["th_sv_num_supports"])
    linetracks = merging.filter_tracks_by_overlap(linetracks, imagecols, f2d["th_overlap"], f2d["th_overlap_num_supports"])
    # [E] line bundle adjustment (cameras constant)
    if not cfg["refinement"]["disable"]:
        ba = optimize.solve_line_bundle_adjustment(cfg["refinement"], imagecols, linetracks, max_num_iterations=200)
        tracks_map = ba.GetOutputLineTracks(num_outliers=cfg["refinement"]["num_outliers_aggregator"])
        linetracks = [t for _, t in tracks_map.items()]
    # [F] output + track report
    limapio.save_txt_linetracks(os.path.join(save, "alltracks.txt"), linetracks, n_visible_views=4)
    limapio.save_folder_linetracks_with_info(os.path.join(save, cfg["output_folder"]), linetracks, config=cfg,
                                             imagecols=imagecols, all_2d_segs=all_2d_segs)
    vis = visualize.Open3DTrackVisualizer(linetracks)
    vis.report()
    limapio.save_obj(os.path.join(save, "triangulated_lines_nv{}.obj".format(cfg["n_visible_views"])),
                     vis.get_lines_np(n_visible_views=cfg["n_visible_views"]))
    return linetracks


_LOC_MATCHERS = ("epipolar", "sold2", "superglue_endpoints", "gluestick", "linetr", "lbd", "l2d2")


def _pose_line(name, pose):  # the results / pose cache line of runners/hybrid_localization.py:366-395
    return " ".join([name] + [str(x) for x in pose.qvec] + [str(x) for x in pose.tvec]) + "\n"


def hybrid_localization(cfg, imagecols_db, imagecols_query, point_corresp, linemap_db, retrieval, results_path,
                        img_name_dict=None, logger=None):
    """Visual localization of the query images of imagecols_query (runners/hybrid_localization.py:94-398): 2D-2D line
    matches to the retrieved database images (the epipolar matcher, or a learned matcher's saved matches), 2D-3D matches
    through the line tracks, the optional reprojection filter, then pl_estimate_absolute_pose from the coarse query pose.
    All queries are matched in one pass over the device and solved in one lm_loc_solve launch. Writes results_path in
    the reference's text format and returns {query id: CameraPose}. Only ransac.method None is supported."""
    lcfg = cfg["localization"]
    if lcfg["2d_matcher"] not in _LOC_MATCHERS:
        raise ValueError("Unknown 2d line matcher: {}".format(lcfg["2d_matcher"]))
    if lcfg["ransac"]["method"] is not None:  # the estimator's own error, before any work
        estimators.pl_estimate_absolute_pose(lcfg, [], [], [], [], [], None)
    train_ids = imagecols_db.get_img_ids()
    query_ids = imagecols_query.get_img_ids()
    if img_name_dict is None:
        img_name_dict = {img_id: imagecols_db.image_name(img_id) for img_id in train_ids}
        img_name_dict.update({img_id: imagecols_query.image_name(img_id) for img_id in query_ids})
    id_to_name = img_name_dict
    name_to_id = {img_name_dict[img_id]: img_id for img_id in train_ids + query_ids}

    all_db_segs, _ = compute_2d_segs(cfg, imagecols_db, compute_descinfo=False)
    all_query_segs, _ = compute_2d_segs(cfg, imagecols_query, compute_descinfo=False)
    all_db_lines = base.get_all_lines_2d(all_db_segs)
    all_query_lines = base.get_all_lines_2d(all_query_segs)
    line2track = base.get_invert_idmap_from_linetracks(all_db_lines, linemap_db)

    pose_dir = results_path.parent / "poses_{}".format(lcfg["2d_matcher"])
    final_poses, todo = {}, []
    for qid in query_ids:
        if lcfg["skip_exists"]:
            limapio.check_makedirs(str(pose_dir))
            fname = os.path.join(pose_dir, f"{qid}.txt")
            if os.path.exists(fname):
                with open(fname) as f:
                    data = f.read().rstrip().split("\n")[0].split()
                    q, t = np.split(np.array(data[1:], float), [4])
                    final_poses[qid] = base.CameraPose(q, t)
                    continue
        todo.append(qid)

    retrieved = {qid: [name_to_id[n] for n in retrieval[id_to_name[qid]]] for qid in todo}
    pairs_2to2 = None
    if lcfg["2d_matcher"] != "epipolar":
        # the learned matcher's saved matches (line2d/base_matcher.py:60-72); extraction and matching are out of scope
        m = lcfg["2d_matcher"]
        folder = os.path.join(cfg["dir_save"], "line_matchings", cfg["line2d"]["detector"]["method"], f"feats_{m}",
                              "{}_n{}_top0".format(m, cfg["n_neighbors_loc"]))
        pairs_2to2 = {}
        for qid in todo:
            fname = os.path.join(folder, f"matches_{qid}.npy")
            if not os.path.exists(fname):
                return _out_of_scope(f"2D line matching ({m}; {fname} is missing)")()
            pairs_2to2[qid] = limapio.read_npy(fname).item()
    query_views = {qid: imagecols_query.camview(qid) for qid in todo}
    db_views = {t: imagecols_db.camview(t) for qid in todo for t in retrieved[qid]}
    matches = _locfn.match_queries_to_linemap(
        query_views, {qid: all_query_lines[qid] for qid in todo}, db_views, all_db_lines, retrieved, linemap_db,
        line2track, IoU_threshold=lcfg["IoU_threshold"], line_pairs_2to2=pairs_2to2,
        epipolar_filter=bool(lcfg.get("epipolar_filter")), reprojection_filter=lcfg["reprojection_filter"],
        dist_thres=2)

    # pl_estimate_absolute_pose's ransac.method None path for every query in one launch
    jointloc_cfg = {}
    if lcfg.get("optimize"):
        jointloc_cfg = lcfg["optimize"].copy()
        args = jointloc_cfg.pop("loss_func_args", None) or []
        name = jointloc_cfg.pop("loss_func")
        if name == "TrivialLoss":
            args = []
        elif name == "HuberLoss":
            assert len(args) == 1, "HuberLoss requires one argument"
        jointloc_cfg["loss_function"] = getattr(optimize, name)(*args)
    if "line_weight" in lcfg:
        jointloc_cfg["weight_point"] = 1.0
        jointloc_cfg["weight_line"] = lcfg["line_weight"]
    l3ds = [track.line for track in linemap_db]
    queries = []
    for qid in todo:
        pairs = matches[qid]
        if logger:
            logger.info(f"{len(pairs)} line matches found for {len(all_query_lines[qid])} 2D lines")
        p3ds, p2ds = point_corresp[qid]["p3ds"], point_corresp[qid]["p2ds"]
        inl = point_corresp[qid].get("inliers")
        if inl is not None:
            p2ds, p3ds = np.array(p2ds)[inl], np.array(p3ds)[inl]
        pose = imagecols_query.campose(qid)
        queries.append(dict(l3ds=l3ds, l3d_ids=[p[1] for p in pairs], l2ds=[all_query_lines[qid][p[0]] for p in pairs],
                            p3ds=p3ds, p2ds=p2ds, K=imagecols_query.cam(imagecols_query.camimage(qid).cam_id).K(),
                            R=pose.R(), T=pose.T()))
    poses, _ = optimize.solve_jointloc_batch(queries, lcfg["line_cost_func"], jointloc_cfg) if queries else ([], [])
    for qid, pose in zip(todo, poses):
        final_poses[qid] = pose
        if lcfg["skip_exists"]:
            with open(os.path.join(pose_dir, f"{qid}.txt"), "w") as f:
                f.writelines([_pose_line(id_to_name[qid], pose)])
    with open(results_path, "w") as f:
        f.writelines([_pose_line(id_to_name[qid], final_poses[qid]) for qid in query_ids])
    return final_poses
