"""Shared helpers of the GPU parity tests: run the same seeded scene through the CUDA engine (C ABI)
and through the CPU oracle and compare per SURVEY.md §8 / BASELINE.json: candidate indices, valid
connections, best candidates and track membership bit-exact; 3D endpoints within 1e-4 absolute."""
import numpy as np

ENDPOINT_TOL = 1e-4   # BASELINE.json north_star: "within 1e-4 absolute on 3D line endpoint coordinates"
SCORE_TOL = 1e-6


def fake_vpresults(sc, seed):
    """Random but well-formed VPResults: ~60% of the lines of every image carry one of 3 VPs."""
    from limap_b200.vplib import VPResult
    rng = np.random.default_rng(seed)
    out = {}
    for v, i in enumerate(sc.img_ids):
        L = int(sc.line_off[v + 1] - sc.line_off[v])
        vps = rng.normal(size=(3, 3))
        vps[:, :2] *= 1000.0
        vps /= np.linalg.norm(vps, axis=1, keepdims=True)
        labels = rng.integers(0, 3, L)
        labels[rng.random(L) < 0.4] = -1
        out[int(i)] = VPResult(labels, vps)
    return out


def run_both(scene, cfg, exhaustive=False, use_ranges=True, vpresults=None, node_parallel=False):
    from limap_b200.engine import TriEngine
    from oracle.oracle import OracleTri
    eng, orc = TriEngine(cfg), OracleTri(cfg, node_parallel=node_parallel)
    for t in (eng, orc):
        t.upload(scene)
        if use_ranges:
            t.set_ranges(*scene.ranges)
        if vpresults is not None:
            t.set_vps(vpresults, scene.img_ids, scene.line_off)
        for i in scene.img_ids:
            if exhaustive:
                t.add_image_exhaustive(int(i), scene.neighbors[int(i)])
            else:
                t.add_image_matches(int(i), *scene.flat_matches(int(i)))
    eng.run()
    return eng, orc


def compare_nodes(scene, eng, orc, debug=False):
    n_nodes = n_cand = n_edges = 0
    for i in scene.img_ids:
        i = int(i)
        gl, gng, gnc = eng.get_best(i)
        ol, ong, onc = orc.get_best(i)
        assert np.array_equal(gnc, onc), f"candidate counts differ in image {i}"
        has = onc > 0
        assert np.array_equal(gng[has], ong[has]), f"best candidate index differs in image {i}"
        assert np.abs(gl[has, :6] - ol[has, :6]).max(initial=0) <= ENDPOINT_TOL
        assert np.abs(gl[has, 6:9] - ol[has, 6:9]).max(initial=0) <= ENDPOINT_TOL
        assert np.abs(gl[has, 9] - ol[has, 9]).max(initial=0) <= SCORE_TOL
        goff, ge = eng.get_valid_edges(i)
        ooff, oe = orc.get_valid_edges(i)
        assert np.array_equal(goff, ooff), f"valid connection counts differ in image {i}"
        # the reference stores valid edges in (score, tri_id)-descending order; membership is what
        # run_clustering consumes (a std::set), so compare per-node sets
        for l in range(len(goff) - 1):
            a = sorted(map(tuple, ge[goff[l]:goff[l + 1]]))
            b = sorted(map(tuple, oe[ooff[l]:ooff[l + 1]]))
            assert a == b, f"valid connections differ at node ({i},{l})"
        n_nodes += len(onc)
        n_cand += int(onc.sum())
        n_edges += len(oe)
        if debug:
            for l in range(len(onc)):
                cl, cng = eng.get_cands_node(i, l)
                rl, rng_ = orc.get_cands_node(i, l)
                assert np.array_equal(cng, rng_), f"candidate list differs at node ({i},{l})"
                if len(rl):
                    assert np.abs(cl[:, :9] - rl[:, :9]).max() <= ENDPOINT_TOL
                    assert np.abs(cl[:, 9] - rl[:, 9]).max() <= SCORE_TOL
    return dict(nodes=n_nodes, candidates=n_cand, valid_edges=n_edges)


def track_sets(tr):
    out = []
    for t in range(len(tr["track_off"]) - 1):
        a, b = tr["track_off"][t], tr["track_off"][t + 1]
        out.append(tuple(zip(tr["img_ids"][a:b].tolist(), tr["line_ids"][a:b].tolist())))
    return out


def compare_tracks(eng, orc):
    gt, ot = eng.build_tracks(), orc.build_tracks()
    gs, os_ = track_sets(gt), track_sets(ot)
    assert len(gs) == len(os_), "number of tracks differs"
    assert set(map(frozenset, gs)) == set(map(frozenset, os_)), "track membership differs"
    exact_order = gs == os_
    # endpoints (the TLS direction sign is arbitrary: compare up to a start/end swap)
    om = {frozenset(s): k for k, s in enumerate(os_)}
    worst = 0.0
    n_ties = 0
    for k, s in enumerate(gs):
        j = om[frozenset(s)]
        a, b = gt["track_line"][k], ot["track_line"][j]
        d = min(np.abs(a[:6] - b[:6]).max(), np.abs(a[:6] - np.concatenate([b[3:6], b[:3]])).max())
        if d > ENDPOINT_TOL and len(s) < 4:
            # aggregate_line3d_list_takebest (merging/aggregator.cc:9-29) keeps the first strict maximum of the
            # node scores. Two nodes of a track that triangulate each other carry the SAME infinite line, so
            # their scores agree to the last few bits and which one wins depends on rounding (compiler / libm),
            # in the reference as well. Accept any member whose score ties with the maximum within 1e-9.
            oa, ob = ot["track_off"][j], ot["track_off"][j + 1]
            sc = ot["line3d"][oa:ob, 9]
            tied = [m for m in range(ob - oa) if sc[m] >= sc.max() * (1 - 1e-9)]
            cand = [ot["line3d"][oa + m, :6] for m in tied]
            dd = min(np.abs(a[:6] - c).max() for c in cand)
            if len(tied) > 1 and dd <= ENDPOINT_TOL:
                n_ties += 1
                d = dd
        worst = max(worst, d)
        assert abs(a[6] - b[6]) <= ENDPOINT_TOL
    assert worst <= ENDPOINT_TOL, f"track endpoints differ by {worst}"
    return dict(tracks=len(gs), exact_order=exact_order, worst=worst, score_ties=n_ties)


def compare_nodes_fast(img_ids, eng, orc):
    """compare_nodes without per-node Python loops (for scenes of 1e5 nodes): candidate counts, best-candidate ids
    and per-node valid-connection sets bit-exact; endpoints / depths / uncertainty within 1e-4, scores within 1e-6."""
    n_nodes = n_cand = n_edges = 0
    worst = 0.0
    for i in img_ids:
        i = int(i)
        gl, gng, gnc = eng.get_best(i)
        ol, ong, onc = orc.get_best(i)
        assert np.array_equal(gnc, onc), f"candidate counts differ in image {i}"
        has = onc > 0
        assert np.array_equal(gng[has], ong[has]), f"best candidate index differs in image {i}"
        if has.any():
            worst = max(worst, float(np.abs(gl[has, :9] - ol[has, :9]).max()))
            assert np.abs(gl[has, 9] - ol[has, 9]).max() <= SCORE_TOL
        goff, ge = eng.get_valid_edges(i)
        ooff, oe = orc.get_valid_edges(i)
        assert np.array_equal(goff, ooff), f"valid connection counts differ in image {i}"
        node_of = np.repeat(np.arange(len(goff) - 1), np.diff(goff))
        if len(ge):
            ga = np.stack([node_of, ge[:, 0], ge[:, 1]], 1)
            oa = np.stack([node_of, oe[:, 0], oe[:, 1]], 1)
            ga = ga[np.lexsort((ga[:, 2], ga[:, 1], ga[:, 0]))]
            oa = oa[np.lexsort((oa[:, 2], oa[:, 1], oa[:, 0]))]
            assert np.array_equal(ga, oa), f"valid connections differ in image {i}"
        n_nodes += len(onc)
        n_cand += int(onc.sum())
        n_edges += len(oe)
    assert worst <= ENDPOINT_TOL, worst
    return dict(nodes=n_nodes, candidates=n_cand, valid_edges=n_edges, worst=worst)
