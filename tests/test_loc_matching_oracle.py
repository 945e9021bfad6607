"""The line-matching oracle (oracle/orc_locmatch.cpp, oracle/locmatch.py) against the reference's own functions.py
(tests/golden/ref/loc_matching.npz, tests/golden/make_locmatch_golden.py): the same pair lists in the same order."""
import os

import numpy as np
import pytest

import locmatch_cases as lc
from oracle import locmatch as om

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "loc_matching.npz")
CASES = {"seed0": dict(seed=0), "seed1_planted": dict(seed=1, planted=True)}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _as_list(a):
    return [tuple(map(int, p)) for p in np.asarray(a).reshape(-1, 2)]


@pytest.mark.parametrize("tag", sorted(CASES))
def test_oracle_2to2_and_filter_equal_reference(golden, tag):
    case = lc.make_case(**CASES[tag])
    cams, lines = case["cams"], case["lines"]
    for q in case["q_ids"]:
        for d in case["retrieval"][q]:
            for th in lc.THRESHOLDS:
                got = om.match_2to2(lines[q], cams[q], lines[d], cams[d], th)
                assert got == _as_list(golden[f"{tag}/m22/{q}/{d}/{th}"]), (q, d, th)
            got = om.filter_2to2(case["pairs"][q][d], lines[q], cams[q], lines[d], cams[d], 0.2)
            assert got == _as_list(golden[f"{tag}/f22/{q}/{d}"]), (q, d)


@pytest.mark.parametrize("tag", sorted(CASES))
@pytest.mark.parametrize("mode", ["epipolar", "learned", "learned_filter"])
@pytest.mark.parametrize("rf", [None] + list(lc.REPROJ_FUNCS))
def test_oracle_runner_order_equals_reference(golden, tag, mode, rf):
    case = lc.make_case(**CASES[tag])
    got = om.match_queries({q: (case["cams"][q], case["lines"][q]) for q in case["q_ids"]},
                           {d: (case["cams"][d], case["lines"][d]) for d in case["db_ids"]}, case["retrieval"],
                           case["line2track"], case["tracks"], 0.2,
                           pairs_2to2=None if mode == "epipolar" else case["pairs"],
                           epipolar_filter=mode == "learned_filter", reprojection_filter=rf)
    for q in case["q_ids"]:
        assert got[q] == _as_list(golden[f"{tag}/run/{mode}/{rf}/{q}"]), q


def test_planted_iou_decisions_straddle_each_threshold(golden):
    """The planted database lines match exactly on the + side of every threshold."""
    case = lc.make_case(**CASES["seed1_planted"])
    q = case["q_ids"][1]
    d = case["retrieval"][q][0]
    n = len(case["lines"][d])
    base = n - 2 * len(lc.PLANT_DELTAS) * len(lc.PLANT_THRESHOLDS)
    for k, th in enumerate(lc.PLANT_THRESHOLDS):
        got = {j for i, j in _as_list(golden[f"seed1_planted/m22/{q}/{d}/{th}"]) if i == 1 and j >= base}
        m = 2 * len(lc.PLANT_DELTAS)
        own = range(base + k * m, base + k * m + m)
        assert {j for j in own if j in got} == set(own[1::2]), th
