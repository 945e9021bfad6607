"""merging.merging on the GPU (lm_merge_fits_build) against the fp64 oracle and the stored outputs of the reference's
compiled MergeToLineTracks: graph nodes, edges in insertion order with bit-exact weights, greedy tracks and their lines."""
import numpy as np
import pytest

import merge_fit_cases as mc
from test_merge_to_linetracks_oracle import assert_same_merge, check_precondition, golden

pytestmark = pytest.mark.gpu


def cuda_merge(fit, l2, l3, var2d, engine=None):
    from limap_b200.config import LINKER2D_DEFAULTS, LINKER3D_DEFAULTS, make_linker
    from limap_b200.engine import MergeEngine
    eng = engine or MergeEngine()
    r = eng.merge_fits(fit.img_ids, fit.model_ids, fit.kvec, fit.qvec, fit.tvec, fit.line_off, fit.segs, fit.lines3d,
                       fit.ng_off, fit.ng_ids, var2d, make_linker(LINKER2D_DEFAULTS, l2), make_linker(LINKER3D_DEFAULTS, l3))
    return r, eng.fit_merge_stats()


def edge_multiset(r):
    return sorted(map(tuple, r["edges"].tolist()))


@pytest.mark.parametrize("name", mc.CASES)
def test_cuda_matches_oracle(name):
    from oracle import merge_fits as orc
    fit, l2, l3, var2d = mc.case(name)
    want = orc.merge_to_linetracks(fit, l2, l3, var2d)
    got, st = cuda_merge(fit, l2, l3, var2d)
    check_precondition(name, got, fit)
    assert_same_merge(got, want)
    if name != "neighbor_lists":  # no self-loops: the whole edge list is exact
        assert edge_multiset(got) == edge_multiset(want)
        assert_same_merge(got, want, exact_self_loops=True)
    assert st["n_edges"] == len(got["sim"]) and st["n_nodes"] == len(got["node_line"])
    assert st["n_pairs_gated"] <= st["n_pairs_tested"]


@pytest.mark.parametrize("name", mc.CASES)
def test_cuda_matches_reference_outputs(name):
    fit, l2, l3, var2d = mc.case(name)
    got, _ = cuda_merge(fit, l2, l3, var2d)
    assert_same_merge(got, golden(name))


def test_many_tiles():
    """V=40, L=600, N=39: three 256-line tiles per image, every image a neighbour of every other."""
    from oracle import merge_fits as orc
    fit, l2, l3, var2d = mc._fit(V=40, L=600, N=39, seed=51), mc.YAML_L2, mc.YAML_L3, mc.YAML_VAR2D
    assert np.diff(fit.line_off).max() > 512
    want = orc.merge_to_linetracks(fit, l2, l3, var2d)
    got, st = cuda_merge(fit, l2, l3, var2d)
    assert len(want["sim"]) > 10000
    assert_same_merge(got, want, exact_self_loops=True)
    assert st["n_retries"] == 0


def test_edge_capacity_retry(monkeypatch):
    fit, l2, l3, var2d = mc.case("yaml")
    base, st0 = cuda_merge(fit, l2, l3, var2d)
    monkeypatch.setenv("LIMAP_B200_FIT_EDGE_CAPACITY", "16")
    got, st = cuda_merge(fit, l2, l3, var2d)
    assert st0["n_retries"] == 0 and st["n_retries"] == 1 and len(got["sim"]) > 16
    for k in base:
        assert got[k].tobytes() == base[k].tobytes(), k


@pytest.mark.parametrize("kind", ["angle", "innerseg"])
@pytest.mark.parametrize("depth", [1.0, 1e3])
@pytest.mark.parametrize("delta", [1e-6, 1e-9])
def test_gates_keep_boundary_pairs(kind, depth, delta):
    """Pairs at th * (1 -+ delta) of the 3D angle and inner-segment tests: the fp32 gates drop none the oracle passes."""
    from oracle import merge_fits as orc
    fit, expect = mc.planted_fit(kind, depth, delta)
    l2, l3 = mc.planted_linkers(kind)
    want = orc.merge_to_linetracks(fit, l2, l3, 5.0)
    pairs = set(map(tuple, want["edges"].tolist()))
    for k, ok in enumerate(expect):  # precondition: the self pair (l1_k, l2_k) of view 0 sits on the boundary
        assert ((2 * k, 2 * k + 1) in pairs) == ok
    got, st = cuda_merge(fit, l2, l3, 5.0)
    if kind == "innerseg":  # the ball gate drops the pairs of different planted pairs (the angle gate cannot here)
        assert st["n_pairs_gated"] < st["n_pairs_tested"]
    assert_same_merge(got, want)
    assert edge_multiset(got) == edge_multiset(want)


def test_merging_filter_remerge_chain():
    """limap.merging.merging -> filter_tracks_by_reprojection -> remerge equals the same chain on the oracle's tracks."""
    import limap.base as base
    import limap.merging as merging
    from oracle import merge_fits as orc
    fit, l2, l3, var2d = mc.case("yaml")
    ids = [int(i) for i in fit.img_ids]
    cams = {v: base.Camera("SIMPLE_PINHOLE" if fit.model_ids[v] == 0 else "PINHOLE",
                           [fit.kvec[v, 0], fit.kvec[v, 2], fit.kvec[v, 3]] if fit.model_ids[v] == 0 else list(fit.kvec[v]),
                           cam_id=v) for v in range(len(ids))}
    imgs = {i: base.CameraImage(v, base.CameraPose(fit.qvec[v], fit.tvec[v])) for v, i in enumerate(ids)}
    imagecols = base.ImageCollection(cams, imgs)
    all_2d = {i: fit.segs_of(v) for v, i in enumerate(ids)}
    fits = {i: list(fit.fits_of(v)) for v, i in enumerate(ids)}
    linker = base.LineLinker(l2, l3)
    graph, tracks = merging.merging(linker, all_2d, imagecols, fits, fit.neighbors, var2d=var2d)
    want = orc.merge_to_linetracks(fit, l2, l3, var2d)
    assert len(graph.nodes) == len(want["node_line"]) and len(graph.undirected_edges) == len(want["sim"])
    assert sum(graph.input_degrees) == 2 * len(want["sim"])
    # the oracle's tracks as LineTracks, built the way merging() builds them
    segs, lines = np.asarray(fit.segs), np.asarray(fit.lines3d)
    otracks = []
    for t in range(len(want["track_off"]) - 1):
        tr = base.LineTrack()
        for k in want["track_nodes"][want["track_off"][t]:want["track_off"][t + 1]].tolist():
            g = int(want["node_line"][k])
            v = int(np.searchsorted(fit.line_off, g, side="right") - 1)
            l3d = base.Line3d(lines[g, 0], lines[g, 1], uncertainty=want["unc"][g])
            tr.node_id_list.append(k)
            tr.image_id_list.append(ids[v])
            tr.line_id_list.append(g - int(fit.line_off[v]))
            tr.line2d_list.append(base.Line2d(segs[g, :2], segs[g, 2:4]))
            tr.line3d_list.append(l3d)
            tr.score_list.append(l3d.length())
        tl = want["track_line"][t]
        tr.line = base.Line3d(tl[:3], tl[3:6], uncertainty=tl[6])
        otracks.append(tr)
    assert len(tracks) == len(otracks) > 0
    for a, b in zip(tracks, otracks):
        assert a.node_id_list == b.node_id_list and a.image_id_list == b.image_id_list
        np.testing.assert_allclose(a.score_list, b.score_list, rtol=1e-15)

    def chain(ts):
        ts = merging.filter_tracks_by_reprojection(ts, imagecols, 8.0, 5.0, num_outliers=0)
        return merging.remerge(base.LineLinker3d(dict(score_th=0.5, th_angle=5.0, th_overlap=0.001,
                                                      th_innerseg=1.0)), ts, num_outliers=0)
    ra, rb = chain(tracks), chain(otracks)
    assert len(ra) == len(rb) > 0
    for a, b in zip(ra, rb):
        assert a.node_id_list == b.node_id_list and a.line_id_list == b.line_id_list
        np.testing.assert_allclose(np.concatenate([a.line.start, a.line.end]),
                                   np.concatenate([b.line.start, b.line.end]), rtol=0, atol=1e-9)
