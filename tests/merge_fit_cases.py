"""Seeded inputs of the MergeToLineTracks tests (merging.merging, merging.py:6-21 / merging.cc:347-511): per-image 3D fits
from limap_b200.synth.make_fits, the linker configurations and neighbour lists each case exercises, and planted pairs on
the 3D decision boundaries. tests/golden/make_merge_golden.py stores the reference's outputs on the cases as
tests/golden/ref/merge_to_linetracks_<case>.npz."""
import numpy as np

from limap_b200 import synth

# cfgs/fitnmerge/default.yaml:61-77 (merging.linker3d / merging.linker2d); var2d of the deeplsd detector (:47-52)
YAML_L2 = dict(score_th=0.5, th_angle=5.0, th_perp=2.0, th_overlap=0.05)
YAML_L3 = dict(score_th=0.5, th_angle=8.0, th_overlap=0.01, th_smartoverlap=0.1, th_smartangle=1.0, th_perp=0.75,
               th_innerseg=0.75)
YAML_VAR2D = 4.0


def _fit(V=8, L=60, N=4, seed=5, fail_frac=0.1, degenerate_frac=0.02, **kw):
    sc = synth.make_scene(V=V, L=L, N=N, seed=seed, **kw)
    return synth.make_fits(sc, depth_noise=1e-3, fail_frac=fail_frac, seed=seed + 1, degenerate_frac=degenerate_frac)


def case(name):
    """(fit, linker2d, linker3d, var2d) of a named case."""
    if name == "yaml":
        return _fit(), YAML_L2, YAML_L3, YAML_VAR2D
    if name == "innerseg2d":  # 2D inner-segment test on, perpendicular and smart-angle tests off
        l2 = dict(YAML_L2, use_innerseg=True, th_innerseg=3.0, use_perp=False, use_smartangle=False)
        return _fit(seed=11), l2, YAML_L3, YAML_VAR2D
    if name == "neighbor_lists":  # asymmetric lists, an image listing itself, a neighbour listed twice
        fit = _fit(V=5, L=50, seed=21)
        ids = [int(i) for i in fit.img_ids]
        fit.set_neighbors({ids[0]: [ids[1], ids[0], ids[2]], ids[1]: [ids[2], ids[2], ids[3]], ids[2]: [ids[0]],
                           ids[3]: [], ids[4]: [ids[3], ids[1]]})
        return fit, YAML_L2, YAML_L3, YAML_VAR2D
    if name == "ids_cameras":  # non-contiguous image ids, SIMPLE_PINHOLE and PINHOLE, many failed and degenerate fits
        return _fit(V=6, L=50, seed=31, id_stride=7, camera_mix=True, fail_frac=0.3, degenerate_frac=0.1), \
            YAML_L2, YAML_L3, 5.0
    if name == "no_edges":  # every fit is a node, no pair passes the 3D angle test
        return _fit(V=4, L=30, seed=41), YAML_L2, dict(YAML_L3, th_angle=1e-9), YAML_VAR2D
    raise KeyError(name)


CASES = ("yaml", "innerseg2d", "neighbor_lists", "ids_cameras", "no_edges")


# ---- planted 3D boundary pairs -----------------------------------------------------------------------------------------
def planted_fit(kind, depth, delta, f=500.0, var2d=5.0):
    """Two views with the identity pose. Pair k of view 0 is (l1_k, l2_k) and view 1 holds l2_k again, so each pair is
    tested as a self pair and as a cross pair. Pairs sit 50 * depth apart along x. The 3D linker of `planted_linkers`
    decides them on one threshold each:
      angle pairs:    l2 is l1 turned by th_angle * (1 -/+ delta) about its midpoint (inner-segment threshold huge);
      innerseg pairs: l2 is l1 moved by th_innerseg * uncertainty * (1 -/+ delta) across the viewing ray.
    Returns (fit, expected pass of every pair)."""
    th_angle, th_inner = 8.0, 0.75
    unc = var2d * depth / f  # Camera::uncertainty at the common depth of both endpoints
    h = 0.3 * depth
    l1s, l2s, expect = [], [], []
    k = 0
    for _ in range(2):
        for sgn in (-1.0, 1.0):
            x0 = 50.0 * depth * k * (1.0 + 0.25 * k)  # spacing that differs from pair to pair
            k += 1
            a = np.array([x0 - h, 0.0, depth]), np.array([x0 + h, 0.0, depth])
            if kind == "angle":
                t = np.radians(th_angle * (1.0 + sgn * delta))
                d = np.array([np.cos(t), np.sin(t), 0.0]) * h
                m = np.array([x0, 0.0, depth])
                b = (m - d, m + d)
            else:
                off = np.array([0.0, th_inner * unc * (1.0 + sgn * delta), 0.0])
                b = (a[0] + off, a[1] + off)
            l1s.append(np.stack(a))
            l2s.append(np.stack(b))
            expect.append(sgn < 0)
    v0 = [x for p in zip(l1s, l2s) for x in p]
    lines3d = np.concatenate([np.stack(v0), np.stack(l2s)])

    def proj(l):
        return np.concatenate([l[0, :2] / l[0, 2] * f, l[1, :2] / l[1, 2] * f]) + 400.0
    segs = np.stack([proj(l) for l in lines3d])
    fit = synth.FitScene(img_ids=np.array([0, 1], np.int32), model_ids=np.zeros(2, np.int32),
                         kvec=np.tile([f, f, 400.0, 400.0], (2, 1)), qvec=np.tile([1.0, 0, 0, 0], (2, 1)),
                         tvec=np.zeros((2, 3)), line_off=np.array([0, len(v0), len(lines3d)], np.int64), segs=segs,
                         lines3d=lines3d, neighbors={0: [1], 1: [0]})
    return fit, expect


def planted_linkers(kind):
    """2D tests all off (only the 3D linker decides); the angle pairs get an inner-segment threshold they always meet."""
    l2 = dict(use_angle=False, use_overlap=False, use_smartangle=False, use_perp=False, use_innerseg=False)
    l3 = dict(YAML_L3, th_innerseg=1e6) if kind == "angle" else dict(YAML_L3)
    return l2, l3
