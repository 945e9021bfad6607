"""lm_tri_run puts the match rows in node order with a stable counting placement (tri_plumbing.cu: row_count, one scan,
row_place; a closed form for exhaustive matching). Every node must see its candidates in (neighbour block, row) order,
the reference's order: ties of the best candidate, GetScoredTrisNode's order and the valid connections depend on it.
These scenes stress the placement (shuffled and duplicated rows, an image matched with itself, empty tables, one line
holding a whole block, blocks of several row chunks) and are checked against the oracle, in debug mode, node by node; per-image adds, a bulk add, pipeline groups and a 2-way shard must give the same bytes."""
import numpy as np
import pytest

from limap_b200.config import DEFAULT_YAML_TRIANGULATION
from limap_b200.synth import concat_scenes, make_scene
from parity_utils import compare_nodes

pytestmark = pytest.mark.gpu

ROW_CHUNK = 8192  # lm::kRowChunk


def _cfg():
    c = dict(DEFAULT_YAML_TRIANGULATION)
    c["debug_mode"] = True
    return c


def _flat(blocks):
    """(ng_ids, row_off, pairs) of one image from [(ng_id, pairs), ...] in the given order."""
    ng = np.asarray([b[0] for b in blocks], np.int32)
    off = np.concatenate([[0], np.cumsum([len(b[1]) for b in blocks])]).astype(np.int64)
    parts = [np.asarray(b[1], np.int32).reshape(-1, 2) for b in blocks]
    pairs = np.concatenate(parts) if parts else np.zeros((0, 2), np.int32)
    return ng, off, np.ascontiguousarray(pairs)


def _blocks(sc, i):
    return [(int(g), np.asarray(sc.matches[i][g], np.int32)) for g in sorted(sc.matches[i])]


# ---- layouts: img_id -> (ng_ids, row_off, pairs); images left out get no matches --------------------------------------
def _plain(sc, rng):
    return {int(i): _flat(_blocks(sc, int(i))) for i in sc.img_ids}


def _shuffled(sc, rng):
    return {int(i): _flat([(g, m[rng.permutation(len(m))]) for g, m in _blocks(sc, int(i))]) for i in sc.img_ids}


def _duplicated(sc, rng):
    out = {}
    for i in sc.img_ids:
        bl = []
        for g, m in _blocks(sc, int(i)):
            extra = m[rng.integers(0, len(m), len(m) // 2)] if len(m) else m
            bl.append((g, np.concatenate([m, extra])[rng.permutation(len(m) + len(extra))]))
        out[int(i)] = _flat(bl)
    return out


def _own_neighbour(sc, rng):
    out = {}
    for v, i in enumerate(sc.img_ids):
        L = int(sc.line_off[v + 1] - sc.line_off[v])
        own = np.stack([rng.integers(0, L, 3 * L), rng.integers(0, L, 3 * L)], 1)
        out[int(i)] = _flat(_blocks(sc, int(i)) + [(int(i), own)])
    return out


def _empty(sc, rng):
    out = {}
    for v, i in enumerate(sc.img_ids):
        if v % 3 == 1:
            continue  # no matches at all
        bl = _blocks(sc, int(i))
        bl[0] = (bl[0][0], np.zeros((0, 2), np.int32))  # a neighbour with an empty table
        L = int(sc.line_off[v + 1] - sc.line_off[v])
        for k, (g, m) in enumerate(bl):
            bl[k] = (g, m[m[:, 0] >= L // 2])  # the first half of the lines has no rows
        out[int(i)] = _flat(bl)
    return out


def _one_line(sc, rng):
    out = {}
    for v, i in enumerate(sc.img_ids):
        bl = _blocks(sc, int(i))
        g, m = bl[-1]
        m = m.copy()
        m[:, 0] = 7  # every row of the last block on line 7
        out[int(i)] = _flat(bl[:-1] + [(g, m)])
    return out


LAYOUTS = dict(plain=_plain, shuffled=_shuffled, duplicated=_duplicated, own_neighbour=_own_neighbour, empty=_empty,
               one_line=_one_line)


def _engine(sc, groups=1):
    from limap_b200.engine import TriEngine
    eng = TriEngine(_cfg())
    eng.upload(sc)
    eng.set_ranges(*sc.ranges)
    eng.set_pipeline_groups(groups)
    return eng


def _oracle(sc, layout):
    from oracle.oracle import OracleTri
    orc = OracleTri(_cfg())
    orc.upload(sc)
    orc.set_ranges(*sc.ranges)
    for i, flat in layout.items():
        orc.add_image_matches(i, *flat)
    return orc


def _result(eng):
    off, edges = eng.get_all_valid_edges()
    return eng.get_nodes().tobytes(), off.copy(), edges.copy()


def _same(a, b):
    assert a[0] == b[0]
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_layout_matches_oracle(name):
    sc = make_scene(V=6, L=60, N=3, K=4, seed=611)
    layout = LAYOUTS[name](sc, np.random.default_rng(7))
    eng = _engine(sc)
    for i, flat in layout.items():
        eng.add_image_matches(i, *flat)
    eng.run()
    st = compare_nodes(sc, eng, _oracle(sc, layout), debug=True)
    assert st["candidates"] > 0


def test_blocks_of_several_chunks():
    """Blocks of 3000 lines x K = 12 rows span several row chunks; per-image adds, a bulk add, 4 pipeline groups and a
    2-way shard give the same bytes, and the oracle agrees."""
    sc = make_scene(V=4, L=3000, N=2, K=12, seed=613)
    layout = _shuffled(sc, np.random.default_rng(9))
    assert max(int(np.diff(f[1]).max()) for f in layout.values()) > 3 * ROW_CHUNK

    eng = _engine(sc)
    for i, flat in layout.items():
        eng.add_image_matches(i, *flat)
    eng.run()
    ref = _result(eng)
    rows = eng.stats()["n_rows"]
    compare_nodes(sc, eng, _oracle(sc, layout), debug=False)

    src, ng, off, parts = [], [], [0], []
    for i, (g, o, p) in layout.items():
        for k in range(len(g)):
            src.append(i)
            ng.append(int(g[k]))
            parts.append(p[o[k]:o[k + 1]])
            off.append(off[-1] + int(o[k + 1] - o[k]))
    bulk = _engine(sc)
    bulk.add_matches_bulk(np.asarray(src, np.int32), np.asarray(ng, np.int32), np.asarray(off, np.int64),
                          np.ascontiguousarray(np.concatenate(parts), np.int32))
    bulk.run()
    _same(_result(bulk), ref)

    grouped = _engine(sc, groups=4)
    for i, flat in layout.items():
        grouped.add_image_matches(i, *flat)
    assert rows >> 16 >= 4
    grouped.run()
    _same(_result(grouped), ref)

    V = len(sc.img_ids)
    nodes = np.frombuffer(ref[0], dtype=eng.get_nodes().dtype)
    for vb, ve in ((0, V // 2), (V // 2, V)):
        sh = _engine(sc)
        for i, flat in layout.items():
            sh.add_image_matches(i, *flat)
        sh.set_shard(vb, ve)
        sh.run()
        lo, hi = int(sc.line_off[vb]), int(sc.line_off[ve])
        assert sh.get_nodes()[lo:hi].tobytes() == nodes[lo:hi].tobytes()


def test_exhaustive_neighbours_of_different_line_counts():
    """TriangulateImageExhaustiveMatch over images of 30 and 50 lines, every other image a neighbour, listed in
    descending id order: the closed-form placement against the oracle's candidate order."""
    from oracle.oracle import OracleTri
    sc = concat_scenes([make_scene(V=3, L=30, N=2, K=3, seed=617), make_scene(V=3, L=50, N=2, K=3, seed=619)])
    assert len(set(np.diff(sc.line_off).tolist())) == 2
    eng, orc = _engine(sc), OracleTri(_cfg())
    orc.upload(sc)
    orc.set_ranges(*sc.ranges)
    for i in sc.img_ids:
        ngs = [int(j) for j in sc.img_ids[::-1] if j != i]
        eng.add_image_exhaustive(int(i), ngs)
        orc.add_image_exhaustive(int(i), ngs)
    eng.run()
    st = compare_nodes(sc, eng, orc, debug=True)
    assert st["candidates"] > 0
