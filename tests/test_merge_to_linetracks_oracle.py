"""The fp64 restatement of merging.merging (oracle/orc_merge_fits.cpp: SetUncertaintySegs3d + MergeToLineTracks,
merging.cc:347-511) against the stored outputs of the reference's compiled merging.cc (tests/golden/ref)."""
import os

import numpy as np
import pytest

import merge_fit_cases as mc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")


def golden(name):
    with np.load(os.path.join(GOLD, f"merge_to_linetracks_{name}.npz")) as z:
        return {k: z[k] for k in z.files}


def without_self_loops(r):
    """Edges other than a line paired with itself. Whether such a pair passes depends on whether the last bit of
    |d . d| rounds above 1 (acos is NaN there), which the compilers decide differently (DESIGN.md §1); a self-loop
    joins no tracks."""
    keep = r["edges"][:, 0] != r["edges"][:, 1]
    return r["edges"][keep], r["sim"][keep]


def assert_same_merge(got, want, exact_self_loops=False):
    np.testing.assert_array_equal(got["node_line"], want["node_line"])
    if exact_self_loops:
        np.testing.assert_array_equal(got["edges"], want["edges"])
        assert got["sim"].tobytes() == want["sim"].tobytes()
    else:
        ge, gs = without_self_loops(got)
        we, ws = without_self_loops(want)
        np.testing.assert_array_equal(ge, we)
        assert gs.tobytes() == ws.tobytes()
    np.testing.assert_array_equal(got["track_off"], want["track_off"])
    np.testing.assert_array_equal(got["track_nodes"], want["track_nodes"])
    np.testing.assert_allclose(got["track_line"], want["track_line"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(got["unc"], want["unc"], rtol=1e-12, atol=0)


def check_precondition(name, r, fit):
    ne, nn = len(r["sim"]), len(r["node_line"])
    lines = np.asarray(fit.lines3d).reshape(-1, 6)
    zero = np.all(lines == 0, axis=1)
    degen = ~zero & np.all(lines[:, :3] == lines[:, 3:], axis=1)
    if name == "no_edges":
        assert nn > 0 and ne == 0 and len(r["track_off"]) == 1
        return
    assert ne > 0 and len(r["track_off"]) > 2
    assert zero.any() and degen.any() and nn == int((~zero & ~degen).sum()), "failed and degenerate fits are no nodes"
    node_img = np.searchsorted(fit.line_off, r["node_line"], side="right") - 1
    e = r["edges"]
    if name == "neighbor_lists":
        pairs = [tuple(x) for x in e.tolist()]
        assert len(pairs) > len(set(pairs)), "the duplicated neighbour produced duplicate edges"
        assert any(a == b and node_img[a] == 0 for a, b in pairs), "the self-listed image produced self-loops"
        assert sorted(fit.neighbors[int(fit.img_ids[0])]) != sorted(fit.neighbors[int(fit.img_ids[1])])
    if name == "ids_cameras":
        assert len(set(np.diff(fit.img_ids).tolist())) == 1 and np.diff(fit.img_ids)[0] > 1
        assert set(fit.model_ids.tolist()) == {0, 1}
        assert (node_img[e[:, 0]] != node_img[e[:, 1]]).any()


@pytest.mark.parametrize("name", mc.CASES)
def test_oracle_matches_reference_outputs(name):
    from oracle import merge_fits as orc
    fit, l2, l3, var2d = mc.case(name)
    want = golden(name)
    check_precondition(name, want, fit)
    got = orc.merge_to_linetracks(fit, l2, l3, var2d)
    assert_same_merge(got, want)
