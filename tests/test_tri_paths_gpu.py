"""GPU parity of every tri_node_kernel instantiation and of the configuration branches of its scorers, against the fp64
CPU oracle (which tests/test_ref_pinning.py pins to the reference's compiled code).

launch_tri_vf picks tri_node_kernel<SLAB, VP, FAST>:
  * FAST (reduced-form scorer, plane-pair triangulation) unless LIMAP_B200_REFERENCE_FORMS is set, the 2D linker uses
    innerseg or endpoint triangulation is on; the engine reads the variable on every run;
  * VP with use_vp (three proposal slots per match row);
  * SLAB when the staging of the largest node (rows x proposal slots) exceeds the shared-memory opt-in limit: persistent
    CTAs then stage each node in a global slab.
Every test asserts the precondition of the path it is meant to reach, so that it cannot silently turn into an ordinary
scene."""
import numpy as np
import pytest

from limap_b200.config import DEFAULT_YAML_TRIANGULATION
from limap_b200.synth import make_scene

from parity_utils import compare_nodes, compare_tracks, fake_vpresults, run_both

pytestmark = pytest.mark.gpu


def _cfg(**kw):
    c = dict(DEFAULT_YAML_TRIANGULATION)
    c.update(kw)
    return c


def _l2d(**kw):
    return dict(linker2d_config=dict(DEFAULT_YAML_TRIANGULATION["linker2d_config"], **kw))


def _l3d(**kw):
    return dict(linker3d_config=dict(DEFAULT_YAML_TRIANGULATION["linker3d_config"], **kw))


@pytest.fixture(params=["fast_forms", "reference_forms"])
def forms(request, monkeypatch):
    if request.param == "reference_forms":
        monkeypatch.setenv("LIMAP_B200_REFERENCE_FORMS", "1")
    else:
        monkeypatch.delenv("LIMAP_B200_REFERENCE_FORMS", raising=False)
    return request.param


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# name -> (configuration overrides, whether the scene keeps candidates). A threshold of 90 on the ray-plane angle or 0 on
# the sensitivity rejects every algebraic candidate (the engine must then agree on an empty result); the VP-constrained
# proposals do not go through these two tests and remain.
CONFIGS = {
    "l2d_innerseg": (_l2d(use_innerseg=True, th_innerseg=3.0), True),
    "l2d_no_perp": (_l2d(use_perp=False), True),
    "l2d_no_overlap": (_l2d(use_overlap=False), True),
    "l2d_no_smartangle": (_l2d(use_smartangle=False), True),
    "l2d_no_angle": (_l2d(use_angle=False), True),
    "l2d_score_th_0.3": (_l2d(score_th=0.3), True),
    "l2d_score_th_0.8": (_l2d(score_th=0.8), True),
    "l2d_th_angle_20": (_l2d(th_angle=20.0), True),       # above 14.4775 deg: the acos branch of angle2_deg
    "l3d_th_angle_20": (_l3d(th_angle=20.0), True),
    "l3d_th_angle_90": (_l3d(th_angle=90.0), True),       # the fp32 cosine gate off
    "l3d_th_scaleinv_0.002": (_l3d(th_scaleinv=0.002), True),
    "l3d_th_scaleinv_0.05": (_l3d(th_scaleinv=0.05), True),
    "l3d_score_th_0.3": (_l3d(score_th=0.3), True),
    "l3d_score_th_0.8": (_l3d(score_th=0.8), True),
    "tri_angle_0": (dict(line_tri_angle_threshold=0.0), True),   # polynomial gates of phase A off
    "tri_angle_90": (dict(line_tri_angle_threshold=90.0), False),
    "sensitivity_0": (dict(sensitivity_threshold=0.0), False),
    "sensitivity_90": (dict(sensitivity_threshold=90.0), True),
    "iou_0": (dict(IoU_threshold=0.0), True),
    "min_length_-1": (dict(min_length_2d=-1.0), True),          # the 2D length test skipped
    "min_length_20": (dict(min_length_2d=20.0), True),
    "rank_path": (dict(fullscore_th=0.0, max_valid_conns=2), True),  # every candidate valid: the rank decides
}


@pytest.mark.parametrize("use_vp", [False, True], ids=["novp", "vp"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_configuration_matrix(name, use_vp, forms):
    over, has_cands = CONFIGS[name]
    sc = make_scene(V=7, L=80, N=4, K=4, seed=401)
    vp = fake_vpresults(sc, 7) if use_vp else None
    eng, orc = run_both(sc, _cfg(debug_mode=True, use_vp=use_vp, **over), vpresults=vp)
    st = compare_nodes(sc, eng, orc, debug=True)
    assert eng.stats()["n_candidates"] == st["candidates"]
    if has_cands:
        assert st["candidates"] > 2000 and st["valid_edges"] > 200
    elif use_vp:
        assert st["candidates"] > 0
    else:
        assert st["candidates"] == 0
    compare_tracks(eng, orc)


# ---- staging and phase-B stress ----------------------------------------------------------------------------------
def _slab_scene(K, keep=3, every=25, seed=31):
    """V=8, L=300, N=7. Every 25th line of a view (a different residue per view) keeps all K matches per neighbour
    (7 K rows), the others keep `keep`, and every 11th line keeps none: large and small (and empty) nodes alternate in
    the persistent CTAs' node order."""
    sc = make_scene(V=8, L=300, N=7, K=K, seed=seed)
    for v, i in enumerate(sc.img_ids):
        for g, m in list(sc.matches[int(i)].items()):
            rank = np.tile(np.arange(K), len(m) // K)
            big = (m[:, 0] % every) == (v % every)
            keep_row = big | ((rank < keep) & (m[:, 0] % 11 != 5))
            sc.matches[int(i)][g] = np.ascontiguousarray(m[keep_row])
    return sc


def _rows_per_node(sc):
    out = []
    for v, i in enumerate(sc.img_ids):
        n = np.zeros(int(sc.line_off[v + 1] - sc.line_off[v]), np.int64)
        for m in sc.matches[int(i)].values():
            np.add.at(n, m[:, 0], 1)
        out.append(n)
    return np.concatenate(out)


@pytest.mark.parametrize("use_vp", [False, True], ids=["novp", "vp"])
def test_slab_path(use_vp, forms):
    """tri_node_kernel<true, VP, FAST>: nodes of >= 2000 candidate slots, twice the opt-in limit of either staging layout
    (246 B/slot fast, ~232 B/slot generic, 227 KB on an H100), more nodes than 4 CTAs per SM, small nodes after large
    ones in the same CTA's slab. The first run starts from the default staging size, overflows and is repeated."""
    ns = 3 if use_vp else 1
    sc = _slab_scene(K=100 if use_vp else 300)
    rows = _rows_per_node(sc)
    assert rows.max() * ns >= 2000 and (rows == 0).any() and (rows[rows > 0] < 30).sum() > 1000
    vp = fake_vpresults(sc, 9) if use_vp else None
    eng, orc = run_both(sc, _cfg(debug_mode=True, use_vp=use_vp), vpresults=vp, node_parallel=True)
    st = eng.stats()
    assert st["max_rows_per_node"] == rows.max() and st["max_rows_per_node"] * ns >= 2000
    assert st["n_nodes"] == len(rows) > 4 * _sm_count()
    cs = compare_nodes(sc, eng, orc, debug=True)
    assert cs["candidates"] > 20000 and cs["valid_edges"] > 1000
    compare_tracks(eng, orc)


def test_vp_view_staging_fallback(monkeypatch):
    """VP + fast forms stage the neighbour views of a node in shared memory (TMA bulk copies) up to
    stage_cap = min(255, (4 cap 8 - 4 cap) / 208) views; nodes with more distinct neighbour views read the rest from
    global memory. 48 neighbours x 2 rows x 3 slots = 288 slots: the default staging size (224) overflows, the run is
    repeated at 288, where stage_cap is 38 < 48. (Only tri_node_kernel<false, true, true> stages views: the generic
    scorer would not reach the fallback, so the test runs the fast forms only.)"""
    monkeypatch.delenv("LIMAP_B200_REFERENCE_FORMS", raising=False)
    sc = make_scene(V=49, L=30, N=48, K=2, seed=33)
    views_per_node = np.zeros(int(sc.line_off[-1]), np.int64)
    for v, i in enumerate(sc.img_ids):
        for m in sc.matches[int(i)].values():
            np.add.at(views_per_node, int(sc.line_off[v]) + np.unique(m[:, 0]), 1)
    vp = fake_vpresults(sc, 11)
    eng, orc = run_both(sc, _cfg(debug_mode=True, use_vp=True), vpresults=vp, node_parallel=True)
    st = eng.stats()
    slots = st["max_rows_per_node"] * 3
    assert slots > 224  # overflow of the default staging size, repeated run
    cap = (slots + 31) // 32 * 32
    assert views_per_node.max() > (4 * cap * 8 - 4 * cap) // 208
    cs = compare_nodes(sc, eng, orc, debug=True)
    assert cs["candidates"] > 20000
    compare_tracks(eng, orc)


def _camera_centres(sc):
    from limap_b200.base import CameraPose
    return np.stack([CameraPose(sc.qvec[v], sc.tvec[v]).center() for v in range(sc.n_views)])


def _widest_window(sc, orc, th_scaleinv):
    """Largest number of candidates of one node inside a row's scale-invariance window on the source start ray
    (|lam_s(j) - lam_s(i)| <= th_scaleinv * z_s(i), lam = distance from the source camera centre), from the oracle's
    debug candidates: columns 0-2 are the start point, column 6 its depth."""
    centres = _camera_centres(sc)
    widest = 0
    for v, i in enumerate(sc.img_ids):
        for l in range(int(sc.line_off[v + 1] - sc.line_off[v])):
            cl, _ = orc.get_cands_node(int(i), l)
            if len(cl) <= widest:
                continue
            lam = np.linalg.norm(cl[:, :3] - centres[v], axis=1)
            lim = th_scaleinv * cl[:, 6]
            srt = np.sort(lam)
            w = np.searchsorted(srt, lam + lim, "right") - np.searchsorted(srt, lam - lim, "left")
            widest = max(widest, int(w.max()))
    return widest


def test_dense_windows(forms):
    """64 views that all see the same 30 lines, every view a neighbour of every other: the partners of a row in phase B
    span windows far wider than 32 (the fast scorer's multi-pass wide branch, pair lists that end a chunk because the
    next row does not fit, segmented (row, image) maxima of the generic scorer that carry across 32-lane batches)."""
    sc = make_scene(V=64, L=30, N=63, K=4, seed=35)
    cfg = _cfg(debug_mode=True)
    eng, orc = run_both(sc, cfg, node_parallel=True)
    assert _widest_window(sc, orc, cfg["linker3d_config"]["th_scaleinv"]) > 64
    cs = compare_nodes(sc, eng, orc, debug=True)
    assert cs["valid_edges"] > 10000
    compare_tracks(eng, orc)


def _feed(eng, sc):
    eng.upload(sc)
    eng.set_ranges(*sc.ranges)
    for i in sc.img_ids:
        eng.add_image_matches(int(i), *sc.flat_matches(int(i)))
    eng.run()
    off, edges = eng.get_all_valid_edges()
    return eng.get_nodes().tobytes(), off.copy(), edges.copy()


def test_stale_staging_hint_across_scenes():
    """The staging size of the node kernel comes from the previous run of the context and survives a new scene: a small
    scene after the slab scene runs with a slab-sized hint, the slab scene after a small scene overflows the hint and is
    repeated. Node records and valid connections are those of a fresh context, byte for byte."""
    from limap_b200.engine import TriEngine
    big, small = _slab_scene(K=300), make_scene(V=6, L=80, N=4, K=4, seed=37)
    cfg = _cfg()
    fresh = {k: _feed(TriEngine(cfg), s) for k, s in (("big", big), ("small", small))}
    for order in (("big", "small"), ("small", "big")):
        eng = TriEngine(cfg)
        for k in order:
            nodes, off, edges = _feed(eng, big if k == "big" else small)
            assert (eng.stats()["max_rows_per_node"] >= 2000) == (k == "big")
            f_nodes, f_off, f_edges = fresh[k]
            assert nodes == f_nodes, (order, k)
            assert np.array_equal(off, f_off) and np.array_equal(edges, f_edges), (order, k)


# ---- decisions planted on a threshold, arbitrated by the reference's stored outputs -------------------------------
def test_boundary_min_length_against_compiled_reference(forms):
    """Segments of length exactly min_length_2d (tests/boundary_scenes.py) as source and as matched lines: CUDA
    reproduces the reference's compiled outputs (stored under tests/golden/ref) and the oracle -- candidate ids, counts
    and valid connections bit-exact, scores within 1e-9."""
    from boundary_scenes import min_length_cfg, min_length_scene
    from test_ref_pinning import _StoredTri, _gold, compare_stored
    sc, planted = min_length_scene(check=False)
    eng, orc = run_both(sc, min_length_cfg())
    r = _StoredTri(_gold("boundary_min_length"), sc, every=1)
    st = compare_stored(sc, r, eng, 1e-7)
    assert st["candidates"] > 1000
    nodes = eng.get_nodes()
    assert (nodes["n_cand"][planted] == 0).all()
    compare_nodes(sc, eng, orc, debug=True)


@pytest.mark.parametrize("name", ["angle_10", "angle_14.4775", "angle_20", "scaleinv"])
def test_boundary_3d_against_compiled_reference(name, forms):
    """3D angle (th_angle 10, 14.4775 -- the switch of the asin^2 series -- and 20) and scale-invariant distance at the
    start and at the end point, planted at threshold * (1 -+ delta) for delta 1e-6, 1e-9 and 1e-11, at depths ~1 and
    ~1e3 and at asset-unit coordinates (tests/boundary_scenes.py). The 1e-6 tier sits inside the fp32 gates' margins,
    the 1e-11 tier inside the 1e-9 band where pair_score_fast decides by two exponentials. CUDA must score every +delta
    pair 0 and every -delta pair >= score_th, and reproduce the reference's stored outputs and the oracle."""
    from boundary_scenes import boundary_3d_cfg, boundary_3d_scene, check_planted
    from test_ref_pinning import _StoredTri, _gold, compare_stored
    sc, planted = boundary_3d_scene(name)
    eng, orc = run_both(sc, boundary_3d_cfg(name))
    check_planted(eng, sc, planted)
    compare_stored(sc, _StoredTri(_gold("boundary_3d_" + name), sc, every=1), eng, 1e-7)
    compare_nodes(sc, eng, orc, debug=True)
