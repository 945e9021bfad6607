"""The match-append entry points (lm_tri_add_image_matches[_device], lm_tri_add_matches_bulk,
lm_tri_add_image_exhaustive) reject bad calls with a fixed message and leave the context as it was: the valid adds that
follow give the node records and valid connections of a fresh context, byte for byte. And the staging-overflow repeat
of lm_tri_run counts the kernel launches of both attempts."""
import numpy as np
import pytest

from limap_b200.config import DEFAULT_YAML_TRIANGULATION
from limap_b200.synth import make_scene

pytestmark = pytest.mark.gpu

UNKNOWN = 999  # make_scene's image ids are 0 .. V-1


def _scene():
    return make_scene(V=5, L=40, N=3, K=3, seed=51)


def _engine(sc):
    from limap_b200.engine import TriEngine
    eng = TriEngine(dict(DEFAULT_YAML_TRIANGULATION))
    eng.upload(sc)
    eng.set_ranges(*sc.ranges)
    return eng


def _results(eng):
    eng.run()
    off, edges = eng.get_all_valid_edges()
    return eng.get_nodes().tobytes(), off.copy(), edges.copy()


def _add_rest(eng, sc, exhaustive, skip=()):
    for i in sc.img_ids:
        if int(i) in skip:
            continue
        if exhaustive:
            eng.add_image_exhaustive(int(i), sc.neighbors[int(i)])
        else:
            eng.add_image_matches(int(i), *sc.flat_matches(int(i)))


_FRESH = {}


def _fresh(sc, exhaustive):
    if exhaustive not in _FRESH:
        eng = _engine(sc)
        _add_rest(eng, sc, exhaustive)
        _FRESH[exhaustive] = _results(eng)
    return _FRESH[exhaustive]


def _assert_like_fresh(eng, sc, exhaustive, skip=()):
    _add_rest(eng, sc, exhaustive, skip)
    nodes, off, edges = _results(eng)
    f_nodes, f_off, f_edges = _fresh(sc, exhaustive)
    assert nodes == f_nodes
    assert np.array_equal(off, f_off) and np.array_equal(edges, f_edges)


def _rejects(call, message):
    from limap_b200._cabi import LimapB200Error
    with pytest.raises(LimapB200Error) as e:
        call()
    assert str(e.value) == message


# ---- per-image adds, host and device pairs --------------------------------------------------------------------------
def _add(eng, on_device, img_id, ng, off, pairs):
    if not on_device:
        return eng.add_image_matches(img_id, ng, off, pairs)
    import torch
    d_pairs = torch.from_numpy(np.ascontiguousarray(pairs, np.int32)).cuda(eng.ctx.device)
    torch.cuda.current_stream(d_pairs.device).synchronize()
    eng.ctx._keep.append(d_pairs)
    return eng.add_image_matches_device(img_id, ng, off, d_pairs.data_ptr())


def _per_image_cases(sc):
    """name -> (image added before the call, exhaustively?, arguments of the rejected call, message)."""
    i0, i1 = int(sc.img_ids[0]), int(sc.img_ids[1])
    ng, off, pairs = sc.flat_matches(i1)
    assert len(ng) >= 2 and off[1] > 0
    dup_ng = np.array([ng[0], ng[0]], np.int32)
    dup_off = np.array([0, off[1], 2 * off[1]], np.int64)
    dup_pairs = np.concatenate([pairs[: off[1]], pairs[: off[1]]])
    bad_off = off.copy()
    bad_off[1] = off[2] + 1
    unknown_ng = ng.copy()
    unknown_ng[-1] = UNKNOWN
    return {
        "unknown_image": (None, False, (UNKNOWN, ng, off, pairs), f"unknown image id {UNKNOWN}"),
        "already_triangulated": (i1, False, (i1, ng, off, pairs), f"image {i1} was already triangulated"),
        "mixing_with_exhaustive": (i0, True, (i1, ng, off, pairs),
                                   "cannot mix exhaustive and match-based triangulation in one run"),
        "unknown_neighbor": (None, False, (i1, unknown_ng, off, pairs), f"unknown neighbor image id {UNKNOWN}"),
        "duplicate_neighbor": (None, False, (i1, dup_ng, dup_off, dup_pairs),
                               "duplicate neighbor id in one TriangulateImage call"),
        "decreasing_row_off": (None, False, (i1, ng, bad_off, pairs), "row_off must be non-decreasing"),
    }


@pytest.mark.parametrize("on_device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", sorted(_per_image_cases(_scene())))
def test_per_image_add_rejections(case, on_device):
    sc = _scene()
    before, exhaustive, args, message = _per_image_cases(sc)[case]
    eng = _engine(sc)
    if before is not None:
        if exhaustive:
            eng.add_image_exhaustive(before, sc.neighbors[before])
        else:
            eng.add_image_matches(before, *sc.flat_matches(before))
    _rejects(lambda: _add(eng, on_device, *args), message)
    _assert_like_fresh(eng, sc, exhaustive, skip=() if before is None else (before,))


def test_per_image_add_needs_a_scene():
    from limap_b200.engine import TriEngine
    sc = _scene()
    eng = TriEngine(dict(DEFAULT_YAML_TRIANGULATION))
    i = int(sc.img_ids[0])
    _rejects(lambda: eng.add_image_matches(i, *sc.flat_matches(i)), "lm_scene_upload must precede TriangulateImage")
    _rejects(lambda: eng.add_matches_bulk(*sc.bulk_matches()), "lm_scene_upload must precede TriangulateImage")


# ---- bulk adds -------------------------------------------------------------------------------------------------------
def test_bulk_add_rejections():
    sc = _scene()
    src, ng, off, pairs = sc.bulk_matches()
    last = len(src) - 1  # the bad block comes last: the blocks before it must not be kept either
    i0 = int(sc.img_ids[0])
    cases = []
    s = src.copy(); s[last] = UNKNOWN
    cases.append(((s, ng, off, pairs), "unknown image id in matches", None, False))
    g = ng.copy(); g[last] = UNKNOWN
    cases.append(((src, g, off, pairs), "unknown image id in matches", None, False))
    o = off.copy(); o[last] = o[last + 1] + 1
    cases.append(((src, ng, o, pairs), "row_off must be non-decreasing", None, False))
    cases.append(((src, ng, off, pairs), f"image {int(src[last])} was already triangulated", int(src[last]), False))
    cases.append(((src, ng, off, pairs), "cannot mix exhaustive and match-based triangulation in one run", i0, True))
    for args, message, before, exhaustive in cases:
        eng = _engine(sc)
        if before is not None:
            if exhaustive:
                eng.add_image_exhaustive(before, sc.neighbors[before])
            else:
                eng.add_image_matches(before, *sc.flat_matches(before))
        _rejects(lambda: eng.add_matches_bulk(*args), message)
        _assert_like_fresh(eng, sc, exhaustive, skip=() if before is None else (before,))


# ---- exhaustive adds -------------------------------------------------------------------------------------------------
def test_exhaustive_add_rejections():
    sc = _scene()
    i0, i1 = int(sc.img_ids[0]), int(sc.img_ids[1])
    nbrs = np.asarray(sc.neighbors[i1], np.int32)
    cases = [
        ((UNKNOWN, nbrs), f"unknown image id {UNKNOWN}", None, True),
        ((i1, nbrs), f"image {i1} was already triangulated", i1, True),
        ((i1, nbrs), "cannot mix exhaustive and match-based triangulation in one run", i0, False),
        # the unknown neighbour comes last: the blocks of the neighbours before it must not be kept either
        ((i1, np.append(nbrs, UNKNOWN).astype(np.int32)), f"unknown neighbor image id {UNKNOWN}", None, True),
    ]
    for args, message, before, exhaustive in cases:
        eng = _engine(sc)
        if before is not None:
            if exhaustive:
                eng.add_image_exhaustive(before, sc.neighbors[before])
            else:
                eng.add_image_matches(before, *sc.flat_matches(before))
        _rejects(lambda: eng.add_image_exhaustive(*args), message)
        _assert_like_fresh(eng, sc, exhaustive, skip=() if before is None else (before,))


# ---- the staging-overflow repeat ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [1, 3])
def test_overflow_repeat_counts_both_attempts(groups):
    """A fresh context stages 224 candidate slots per node; the slab scene's largest node needs more, so its first run
    overflows and is repeated at the exact size. Its launches are those of both attempts; an identical second run, which
    starts from the exact hint, adds one attempt's. One attempt launches per pipeline group: the row expansion, the
    radix sort's passes (ceil(log2(2400)) = 12 key bits: two 8-bit passes plus one), the node offsets, the node kernel
    and the four launches of the edge compaction."""
    from test_tri_paths_gpu import _slab_scene
    sc = _slab_scene(K=300)
    assert sc.n_rows() >> 16 >= groups and int(sc.line_off[-1]) == 2400
    eng = _engine(sc)
    eng.set_pipeline_groups(groups)
    _add_rest(eng, sc, exhaustive=False)
    per_attempt = groups * (1 + 3 + 1 + 1 + 4)
    n0 = eng.stats()["n_kernel_launches"]
    first = eng.run()
    assert first["max_rows_per_node"] > 224  # the first attempt overflowed
    nodes = eng.get_nodes().tobytes()
    n1 = eng.stats()["n_kernel_launches"]
    second = eng.run()
    n2 = eng.stats()["n_kernel_launches"]
    assert n1 - n0 == 2 * per_attempt
    assert n2 - n1 == per_attempt
    assert eng.get_nodes().tobytes() == nodes
    for k in ("n_rows", "n_candidates", "n_valid_edges", "max_rows_per_node", "n_pairs_gated", "n_pairs_exact"):
        assert first[k] == second[k], k
    assert first["last_node_kernel_ms"] > 0 and first["last_run_ms"] >= first["last_node_kernel_ms"]
