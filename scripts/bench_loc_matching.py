"""Benchmark of the localization line matching on the GPU (lm_locmatch_*: the epipolar matcher of
runners/hybrid_localization.py with match_line_2to3 and the reprojection filter, for all queries in one pass).

Workload "locmatch100": 100 queries, each with 1000 lines and 10 retrieved database images of 1000 lines (1e9 epipolar
IoU tests), on a map of 20000 3D lines seen by 200 database cameras (PINHOLE, 800x600) around a 10 m box; 60 % of the
database lines are on tracks; query poses 2 degrees and 5 cm off; IoU_threshold 0.2 and the Midpoint reprojection filter
(dist_thres 2, as the runner calls it). Prints one JSON line: the card and its power limit; IoU tests/s of the test
kernel alone (sweep_count_kernel), of the sweep's kernels (the test kernel, the scan and the placement, without the host
read of the pair count between them) and end to end from host arrays (scene
upload, sweep, grouping, reprojection filter, copy back), median / min / max of --reps calls after a warm-up; the matched
2to2 / 2to3 / filtered counts; the reference's compiled compute_epipolar_IoU in a C loop on all host cores, and the fp64
oracle, on --ref-items items, with the agreement of the device's per-item pair lists.

    python scripts/bench_loc_matching.py [--queries 100] [--reps 5] [--ref-items 4]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in out.split(",")]
        return name, pl
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def spread(xs):
    xs = sorted(xs)
    return dict(median=xs[len(xs) // 2], min=xs[0], max=xs[-1])


def _look_at(C, rng):
    from limap_b200.synth import _rot_to_quat
    z = -C / np.linalg.norm(C)
    x = np.cross(z, np.array([0.0, 0.0, 1.0]) + rng.normal(scale=0.1, size=3))
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z], 0)
    return _rot_to_quat(R), -R @ C, R


def make_workload(n_q, n_db, n_ret, n_lines, n_tracks, seed=0):
    from limap_b200.synth import _quat_mul
    rng = np.random.default_rng(seed)
    S = rng.uniform(-5, 5, (n_tracks, 3))
    tracks = np.concatenate([S, S + rng.normal(size=(n_tracks, 3))], 1)
    kvec = np.array([600.0, 590.0, 400.0, 300.0])

    def image(C, noise=0.5):
        q, t, R = _look_at(C, rng)
        ids = rng.choice(n_tracks, n_lines, replace=False)
        h0 = tracks[ids, :3] @ R.T + t
        h1 = tracks[ids, 3:] @ R.T + t
        seg = np.concatenate([h0[:, :2] / h0[:, 2:] * kvec[:2] + kvec[2:], h1[:, :2] / h1[:, 2:] * kvec[:2] + kvec[2:]],
                             1) + rng.normal(size=(n_lines, 4)) * noise
        return q, t, seg, ids

    def sphere(n):
        d = rng.normal(size=(n, 3))
        return d / np.linalg.norm(d, axis=1, keepdims=True) * 12.0

    db = [image(C) for C in sphere(n_db)]
    qs = []
    for C in sphere(n_q):
        q, t, seg, _ = image(C)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        h = np.deg2rad(2.0) / 2
        q = _quat_mul(np.r_[np.cos(h), axis * np.sin(h)][None], q[None])[0]
        qs.append((q, t + rng.normal(size=3) * 0.05, seg))
    centers = np.array([-(_quat_R(d[0]).T @ d[1]) for d in db])
    ret = []
    for q, t, _ in qs:
        Cq = -(_quat_R(q).T @ t)
        ret.append(list(np.argsort(np.linalg.norm(centers - Cq, axis=1))[:n_ret]))
    kv = np.tile(kvec, (n_q + n_db, 1))
    qv = np.array([x[0] for x in qs] + [d[0] for d in db])
    tv = np.array([x[1] for x in qs] + [d[1] for d in db])
    lines = np.concatenate([x[2] for x in qs] + [d[2] for d in db])
    track = np.concatenate([np.full(n_lines * n_q, -1)] +
                           [np.where(rng.random(n_lines) < 0.6, d[3], -1) for d in db]).astype(np.int32)
    line_off = np.arange(n_q + n_db + 1, dtype=np.int64) * n_lines
    items = np.array([(qi, n_q + d) for qi in range(n_q) for d in ret[qi]], np.int32)
    return dict(kvec=kv, qvec=qv, tvec=tv, lines=lines, track=track, line_off=line_off, tracks=tracks, items=items)


def _quat_R(q):
    from limap_b200.base import _quat_to_R
    return _quat_to_R(q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--retrieved", type=int, default=10)
    ap.add_argument("--lines", type=int, default=1000)
    ap.add_argument("--db-images", type=int, default=200)
    ap.add_argument("--tracks", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-items", type=int, default=4)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    from limap_b200 import _cabi
    from limap_b200._cabi import check, lib, ptr
    from oracle import locmatch as om

    name, power = card()
    w = make_workload(a.queries, a.db_images, a.retrieved, a.lines, a.tracks)
    ctx = _cabi.Context(0)
    L, h = lib(), ctx.handle
    n_items = len(w["items"])

    def st():
        s = _cabi.LocMatchStats()
        check(L.lm_locmatch_get_stats(h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in _cabi.LocMatchStats._fields_}

    def upload():
        check(L.lm_locmatch_set_scene(h, len(w["kvec"]), ptr(w["kvec"]), ptr(w["qvec"]), ptr(w["tvec"]),
                                      ptr(w["line_off"]), ptr(w["lines"]), ptr(w["track"]), len(w["tracks"]),
                                      ptr(w["tracks"])))

    def run():
        """Host arrays -> filtered 2D-3D matches of every query on the host."""
        upload()
        n23 = check(L.lm_locmatch_sweep(h, n_items, ptr(w["items"]), 0.2, 1))
        sweep = st()
        n = check(L.lm_locmatch_group(h, 1, 2.0, 0.4, 1.0))
        off, pairs = np.zeros(a.queries + 1, np.int64), np.zeros((n, 2), np.int32)
        check(L.lm_locmatch_get(h, ptr(off), ptr(pairs), n))
        return sweep, n23, n

    run()  # warm-up
    sweep_ms, test_ms, wall_ms = [], [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        sweep, n23, n_final = run()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        sweep_ms.append(sweep["kernel_ms"])
        test_ms.append(sweep["test_ms"])
    tests = sweep["n_tests"]
    # plain 2to2 pair lists of the first items, against the oracle and the compiled reference
    k = min(a.ref_items, n_items)
    upload()
    n22 = check(L.lm_locmatch_sweep(h, k, ptr(np.ascontiguousarray(w["items"][:k])), 0.2, 0))
    off, pairs = np.zeros(k + 1, np.int64), np.zeros((n22, 2), np.int32)
    check(L.lm_locmatch_get(h, ptr(off), ptr(pairs), n22))
    cams = np.concatenate([np.ones((len(w["kvec"]), 1)), w["kvec"], w["qvec"], w["tvec"]], 1)
    lo = w["line_off"]
    agree, orc_s = True, 0.0
    for i, (qi, di) in enumerate(w["items"][:k]):
        t0 = time.perf_counter()
        o = om.match_2to2(w["lines"][lo[qi]:lo[qi + 1]], cams[qi], w["lines"][lo[di]:lo[di + 1]], cams[di], 0.2)
        orc_s += time.perf_counter() - t0
        agree &= o == [tuple(map(int, p)) for p in pairs[off[i]:off[i + 1]]]
    res = dict(workload="locmatch100", card=name, power_limit=power, queries=a.queries, retrieved=a.retrieved,
               lines=a.lines, iou_tests=int(tests), reps=a.reps, test_kernel_ms=spread(test_ms),
               sweep_ms=spread(sweep_ms), e2e_ms=spread(wall_ms),
               test_kernel_tests_per_s=tests / (spread(test_ms)["median"] * 1e-3),
               sweep_tests_per_s=tests / (spread(sweep_ms)["median"] * 1e-3),
               e2e_tests_per_s=tests / (spread(wall_ms)["median"] * 1e-3),
               pairs_2to2=int(sweep["n_pairs_2to2"]), pairs_2to3=int(n23), matches_after_reprojection_filter=int(n_final),
               check_items=k, check_tests=int(k * a.lines * a.lines), oracle_pairs_identical=bool(agree),
               oracle_tests_per_s_one_core=k * a.lines * a.lines / orc_s)
    try:
        it = w["items"][:k]
        t0 = time.perf_counter()
        cnt = om.ref_count(cams, it, lo, w["lines"], it, 0.2)
        dt = time.perf_counter() - t0
        res.update(reference_c_loop_tests_per_s=k * a.lines * a.lines / dt, reference_threads=os.cpu_count(),
                   reference_counts_identical=bool((cnt == np.diff(off)).all()))
    except RuntimeError as e:
        res.update(reference_c_loop_tests_per_s=f"not measured ({e})")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
