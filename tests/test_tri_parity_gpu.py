"""GPU parity: CUDA engine through the C ABI vs the fp64 CPU oracle on the same seeded scenes."""
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


def test_small_scene_debug_candidates():
    sc = make_scene(V=6, L=80, N=4, K=4, seed=11)
    eng, orc = run_both(sc, _cfg(debug_mode=True))
    st = compare_nodes(sc, eng, orc, debug=True)
    assert st["candidates"] > 500 and st["valid_edges"] > 100
    assert eng.stats()["n_candidates"] == st["candidates"]
    assert eng.stats()["n_rows"] == sc.n_rows()
    tr = compare_tracks(eng, orc)
    assert tr["tracks"] > 20


def test_medium_scene_default_yaml():
    sc = make_scene(V=12, L=300, N=8, K=10, seed=12)
    eng, orc = run_both(sc, _cfg())
    st = compare_nodes(sc, eng, orc)
    assert st["valid_edges"] > 1000
    tr = compare_tracks(eng, orc)
    assert tr["tracks"] > 100


@pytest.mark.parametrize("min_outer", [1, 2, 3])
def test_cpp_defaults_and_outer_edge_filter(min_outer):
    # C++ defaults differ from the yaml (min_length_2d 20, angle 5, min_num_outer_edges 1, linker thresholds); 2 and 3
    # make filterNodeByNumOuterEdges peel further, as dropped nodes cost their parents outer edges
    sc = make_scene(V=8, L=120, N=5, K=5, seed=13)
    eng, orc = run_both(sc, {"min_num_outer_edges": min_outer})
    unfiltered, _ = run_both(sc, {"min_num_outer_edges": 0})
    support = lambda e: int(e.build_tracks()["track_off"][-1])
    assert support(eng) < support(unfiltered)  # the filter removes nodes from the track graph of this scene
    compare_nodes(sc, eng, orc)
    compare_tracks(eng, orc)


def test_asset_unit_scale_non_contiguous_ids_shuffled_rows():
    # Hypersim asset units (|X| ~ 1e3), image ids with gaps, match rows not sorted by line id
    sc = make_scene(V=8, L=100, N=5, K=4, seed=14, scale=100.0, id_stride=7, shuffle_rows=True)
    eng, orc = run_both(sc, _cfg(debug_mode=True))
    compare_nodes(sc, eng, orc, debug=True)
    compare_tracks(eng, orc)


def test_endpoints_triangulation_and_halfpix_no_ranges():
    sc = make_scene(V=6, L=80, N=4, K=4, seed=15)
    eng, orc = run_both(sc, _cfg(use_endpoints_triangulation=True, add_halfpix=True), use_ranges=False)
    compare_nodes(sc, eng, orc)
    compare_tracks(eng, orc)


def test_max_valid_conns_cap():
    sc = make_scene(V=6, L=60, N=5, K=8, seed=16)
    eng, orc = run_both(sc, _cfg(max_valid_conns=3))
    compare_nodes(sc, eng, orc)
    compare_tracks(eng, orc)


def test_vp_proposals():
    # use_vp: up to three proposals per match row, [vp1, vp2, algebraic] (base_line_triangulator.cc:258-326)
    sc = make_scene(V=6, L=60, N=4, K=3, seed=21)
    vp = fake_vpresults(sc, 5)
    eng, orc = run_both(sc, _cfg(use_vp=True, debug_mode=True), vpresults=vp)
    st = compare_nodes(sc, eng, orc, debug=True)
    assert st["candidates"] > 1.2 * run_both(sc, _cfg())[0].stats()["n_candidates"]
    compare_tracks(eng, orc)
    # disable_vp_triangulation falls back to the algebraic proposal only
    eng2, orc2 = run_both(sc, _cfg(use_vp=True, disable_vp_triangulation=True), vpresults=vp)
    compare_nodes(sc, eng2, orc2)


def test_exhaustive_matcher():
    # TriangulateImageExhaustiveMatch: every line of every neighbour (CI E2E mode of the reference)
    sc = make_scene(V=5, L=40, N=3, K=2, seed=17)
    eng, orc = run_both(sc, _cfg(), exhaustive=True)
    compare_nodes(sc, eng, orc)
    compare_tracks(eng, orc)


def test_empty_and_ragged_inputs():
    sc = make_scene(V=5, L=30, N=3, K=3, seed=18)
    # image 0 has no matches at all, image 1 has an empty table for one neighbour
    i0, i1 = int(sc.img_ids[0]), int(sc.img_ids[1])
    sc.matches[i0] = {}
    g = sorted(sc.matches[i1].keys())[0]
    sc.matches[i1][g] = np.zeros((0, 2), np.int32)
    eng, orc = run_both(sc, _cfg())
    compare_nodes(sc, eng, orc)
    compare_tracks(eng, orc)


def test_out_of_range_match_raises():
    from limap_b200._cabi import LimapB200Error
    from limap_b200.engine import TriEngine
    sc = make_scene(V=4, L=20, N=2, K=2, seed=19)
    eng = TriEngine(_cfg())
    eng.upload(sc)
    i = int(sc.img_ids[0])
    ng, off, pairs = sc.flat_matches(i)
    pairs = pairs.copy()
    pairs[0, 0] = 10_000
    eng.add_image_matches(i, ng, off, pairs)
    with pytest.raises(LimapB200Error, match="IndexError"):
        eng.run()


def test_full_size_properties_hypersim100_shape():
    """BASELINE.json configs[1] shape (V=100 scaled down in L to keep the test short): size-independent
    properties -- every valid connection's candidate exists, scores are >= fullscore_th, best is the
    arg-max, rerun is idempotent, sharded runs agree with the full run."""
    sc = make_scene(V=40, L=400, N=10, K=10, seed=20)
    from limap_b200.engine import TriEngine
    eng = TriEngine(_cfg())
    eng.upload(sc)
    eng.set_ranges(*sc.ranges)
    for i in sc.img_ids:
        eng.add_image_matches(int(i), *sc.flat_matches(int(i)))
    s1 = eng.run()
    best1 = [eng.get_best(int(i)) for i in sc.img_ids]
    s2 = eng.run()
    assert s1["n_candidates"] == s2["n_candidates"] and s1["n_valid_edges"] == s2["n_valid_edges"]
    for (a, b, c), i in zip(best1, sc.img_ids):
        a2, b2, c2 = eng.get_best(int(i))
        assert np.array_equal(a, a2) and np.array_equal(b, b2) and np.array_equal(c, c2)
    assert s1["n_rows"] == sc.n_rows()
    # shard [0,20) + [20,40) == full
    tot = 0
    for lo, hi in ((0, 20), (20, 40)):
        eng.set_shard(lo, hi)
        st = eng.run()
        tot += st["n_candidates"]
        for v in range(lo, hi):
            a2, b2, c2 = eng.get_best(int(sc.img_ids[v]))
            assert np.array_equal(best1[v][0], a2) and np.array_equal(best1[v][2], c2)
    assert tot == s1["n_candidates"]


def test_bulk_add_and_pipeline_groups_match_per_image_adds():
    """lm_tri_add_matches_bulk + lm_tri_set_pipeline_groups(n): same node records and valid connections as
    per-image adds in one group (groups split the run by source image; nodes are independent)."""
    from limap_b200.engine import TriEngine
    sc = make_scene(V=30, L=500, N=10, K=10, seed=23)
    ref = TriEngine(_cfg())
    ref.upload(sc)
    ref.set_ranges(*sc.ranges)
    for i in sc.img_ids:
        ref.add_image_matches(int(i), *sc.flat_matches(int(i)))
    s_ref = ref.run()
    nodes_ref = ref.get_nodes().copy()
    off_ref, edges_ref = ref.get_all_valid_edges()
    src, ng, off, pairs = sc.bulk_matches()
    for n_groups in (1, 3, 7):
        eng = TriEngine(_cfg())
        eng.upload(sc)
        eng.set_ranges(*sc.ranges)
        eng.set_pipeline_groups(n_groups)
        eng.add_matches_bulk(src, ng, off, pairs)
        st = eng.run()
        assert st["n_candidates"] == s_ref["n_candidates"] and st["n_valid_edges"] == s_ref["n_valid_edges"]
        assert eng.get_nodes().tobytes() == nodes_ref.tobytes()
        o2, e2 = eng.get_all_valid_edges()
        assert np.array_equal(o2, off_ref) and np.array_equal(e2[: o2[-1]], edges_ref[: off_ref[-1]])
        # lm_tri_set_node_sink: the records streamed to a (pinned) host buffer during the run are the getter's
        import torch
        from limap_b200._cabi import NODE_RECORD_DTYPE
        sink = torch.empty(len(nodes_ref) * NODE_RECORD_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(NODE_RECORD_DTYPE)
        sink.view(np.uint8)[...] = 0xAB
        eng.run(nodes_out=sink)
        assert sink.tobytes() == nodes_ref.tobytes()
        with pytest.raises(ValueError):
            eng.run(nodes_out=np.zeros(3, NODE_RECORD_DTYPE))
        # tracks (min_num_outer_edges = 0; the outer-edge filter runs in the C++-defaults test)
        tr = eng.build_tracks()
        tr_ref = ref.build_tracks()
        for k in ("track_off", "img_ids", "line_ids", "node_ids"):
            assert np.array_equal(tr[k], tr_ref[k]), k
        assert np.array_equal(tr["track_line"], tr_ref["track_line"])
        # distinct-image counts of the union-find: bit sets (few views) and sorted vectors (many views) agree
        import os
        os.environ["LIMAP_B200_UF_BITSET_MAX_VIEWS"] = "0"
        try:
            tr_vec = eng.build_tracks()
        finally:
            del os.environ["LIMAP_B200_UF_BITSET_MAX_VIEWS"]
        for k in ("track_off", "img_ids", "line_ids", "node_ids", "track_line"):
            assert np.array_equal(tr_vec[k], tr[k]), k


def test_full_size_hypersim100_properties():
    """BASELINE.json configs[1] at full size (V=100, L=1000, N=20, K=10: 2e7 match rows, the bench workload), through
    properties that do not need the oracle: counters are consistent with the node records, a second run and a
    pipelined run (5 groups) reproduce every node record and valid connection bit for bit, two half shards reproduce
    the full run, and the best candidate of every node is one of its valid connections' peers or scoreless."""
    from limap_b200.engine import TriEngine
    from limap_b200.synth import CONFIGS
    sc = make_scene(**CONFIGS["hypersim100"])
    src, ng, off, pairs = sc.bulk_matches()
    assert len(pairs) == 20_000_000

    def run(groups, shard=None):
        eng = TriEngine(_cfg())
        eng.upload(sc)
        eng.set_ranges(*sc.ranges)
        eng.set_pipeline_groups(groups)
        eng.add_matches_bulk(src, ng, off, pairs)
        if shard is not None:
            eng.set_shard(*shard)
        st = eng.run()
        nodes = eng.get_nodes().copy()
        if shard is not None:
            return eng, st, nodes, None, None
        eoff, edges = eng.get_all_valid_edges()
        return eng, st, nodes, eoff.copy(), edges[: int(eoff[-1])].copy()

    eng, st, nodes, eoff, edges = run(1)
    assert st["n_rows"] == 20_000_000 and st["n_nodes"] == 100_000
    assert int(nodes["n_cand"].sum()) == st["n_candidates"] > 5_000_000
    assert int(nodes["n_valid"].sum()) == st["n_valid_edges"] == int(eoff[-1]) > 500_000
    assert np.array_equal(np.diff(eoff), nodes["n_valid"])
    has = nodes["n_cand"] > 0
    assert np.isfinite(nodes["line"][has]).all() and (nodes["score"][has] >= 0).all()
    assert (nodes["score"][~has] == 0).all()
    assert (nodes["n_valid"] <= nodes["n_cand"]).all()
    assert edges[:, 1].min() >= 0 and edges[:, 1].max() < 1000 and set(np.unique(edges[:, 0])) <= set(sc.img_ids.tolist())
    # idempotence
    st2 = eng.run()
    assert st2["n_candidates"] == st["n_candidates"] and st2["n_valid_edges"] == st["n_valid_edges"]
    assert eng.get_nodes().tobytes() == nodes.tobytes()
    # pipelined groups
    _, st5, nodes5, eoff5, edges5 = run(5)
    assert nodes5.tobytes() == nodes.tobytes() and np.array_equal(eoff5, eoff) and np.array_equal(edges5, edges)
    # two half shards
    tot = 0
    for lo, hi in ((0, 50), (50, 100)):
        e2, s2, n2, _, _ = run(1, shard=(lo, hi))
        a, b = int(sc.line_off[lo]), int(sc.line_off[hi])
        assert n2[a:b].tobytes() == nodes[a:b].tobytes()
        tot += s2["n_candidates"]
    assert tot == st["n_candidates"]
