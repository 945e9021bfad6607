"""Decisions of tri_node_kernel planted on their thresholds (tests/boundary_scenes.py): the phase-A gates (ray-plane angle,
epipolar IoU, also with grazing epipolar lines, sensitivity), the sub-tests of the 2D linker (angle on both branches of
angle2_deg, overlap, smart angle, perpendicular distance) and fullscore_th, at threshold * (1 -+ delta) or, for the IoU,
threshold -+ delta. Most of these are decided in a reduced form that falls back to the reference's form only inside a
narrow band, or with no band at all; random scenes never come within 1e-9 of a threshold, so only planted rows can tell
a wrong band, margin sign or comparison apart.

The reference's compiled outputs on the same scenes are stored under tests/golden/ref and arbitrate; the oracle is
compared node by node as well. Each family runs under both forms (tri_node_kernel<false, false, true>, and
<false, false, false> through gate2d + pair_score) and with use_vp, where every line is unlabelled: the VP
instantiations then run the same rows and must find exactly the same candidates."""
import pytest

from parity_utils import compare_nodes, run_both

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["fast_forms", "reference_forms"])
def forms(request, monkeypatch):
    if request.param == "reference_forms":
        monkeypatch.setenv("LIMAP_B200_REFERENCE_FORMS", "1")
    else:
        monkeypatch.delenv("LIMAP_B200_REFERENCE_FORMS", raising=False)
    return request.param


def _families():
    from boundary_scenes import PLANTED
    return sorted(PLANTED)


@pytest.mark.parametrize("use_vp", [False, True], ids=["novp", "vp"])
@pytest.mark.parametrize("name", _families())
def test_planted_decisions_against_compiled_reference(name, use_vp, forms):
    from boundary_scenes import (check_planted_family, planted_cfg, planted_golden, planted_scene, planted_score_tol,
                                 unlabelled_vps)
    from test_ref_pinning import _StoredTri, _gold, compare_stored
    sc, planted = planted_scene(name)
    eng, orc = run_both(sc, planted_cfg(name, use_vp=use_vp), vpresults=unlabelled_vps(sc) if use_vp else None)
    check_planted_family(name, eng, sc, planted)
    r = _StoredTri(_gold(planted_golden(name)), sc, every=1)
    compare_stored(sc, r, eng, 1e-7, planted_score_tol(name))
    assert eng.stats()["n_candidates"] == int(r.z["cand_cnt"].sum())
    compare_nodes(sc, eng, orc, debug=True)
