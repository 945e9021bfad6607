"""Benchmark of merging.merging on the GPU (lm_merge_fits_build, MergeToLineTracks of merging.cc:347-511).

Workload "fitnmerge100": V=100 images, L=1000 segments each, every image the neighbour of all 99 others (what
n_neighbors: 100 gives on a 100-image scene, cfgs/fitnmerge/default.yaml:11), the yaml's merging linkers. Prints one
JSON line: the card and its power limit; pair checks per second (the pairs the reference's loops test, over the pair
kernel's device time, and end to end from host arrays to host results); pairs past the fp32 gates, edges, tracks; a
roofline of the pair kernel; the fp64 oracle's CPU rate on a subset of source images (stated as such); and the parity of
the timed output with the oracle (graph nodes, edges in insertion order, tracks).

    python scripts/bench_merge_to_linetracks.py [--reps 5] [--oracle-images 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

# H100 SXM data sheet: fp32 (non-tensor) 67 TFLOP/s, HBM3 3.35 TB/s
PEAK_FP32 = 67e12
PEAK_BW = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in out.split(",")]
        return name, pl
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=100)
    ap.add_argument("--L", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-images", type=int, default=2, help="source images of the oracle's CPU rate subset")
    a = ap.parse_args()
    import merge_fit_cases as mc
    from limap_b200 import synth
    from limap_b200.config import LINKER2D_DEFAULTS, LINKER3D_DEFAULTS, make_linker
    from limap_b200.engine import MergeEngine
    from oracle import merge_fits as orc
    from oracle.oracle import usable_cpus

    sc = synth.make_scene(V=a.V, L=a.L, N=a.V - 1, seed=2024)
    fit = synth.make_fits(sc, depth_noise=1e-3, fail_frac=0.1, seed=2025)
    l2d, l3d = make_linker(LINKER2D_DEFAULTS, mc.YAML_L2), make_linker(LINKER3D_DEFAULTS, mc.YAML_L3)
    eng = MergeEngine()
    args = (fit.img_ids, fit.model_ids, fit.kvec, fit.qvec, fit.tvec, fit.line_off, fit.segs, fit.lines3d, fit.ng_off,
            fit.ng_ids, mc.YAML_VAR2D, l2d, l3d)
    eng.merge_fits(*args)  # warm-up: module load, buffer allocation
    kern, e2e = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        r = eng.merge_fits(*args)
        e2e.append(time.perf_counter() - t0)
        kern.append(eng.fit_merge_stats()["pair_kernel_ms"] * 1e-3)
    st = eng.fit_merge_stats()
    tk, te = float(np.median(kern)), float(np.median(e2e))
    tested = st["n_pairs_tested"]
    # roofline of the pair kernel: per tested pair ~12 fp32 operations of the ball gate (+5 of the angle gate on the
    # survivors of the ball gate, counted for all: an upper bound); bytes = the gate records (2 x float4) and node
    # flags of both sides of every tile, read once per tile
    flops = 17.0 * tested
    n_tiles_bytes = 0
    lines = np.diff(fit.line_off)
    for v in range(len(fit.img_ids)):
        na = -(-int(lines[v]) // 256)
        for k in range(fit.ng_off[v], fit.ng_off[v + 1] + 1):
            nb = na if k == fit.ng_off[v + 1] else -(-int(lines[np.searchsorted(fit.img_ids, fit.ng_ids[k])]) // 256)
            n_tiles_bytes += na * nb * 2 * 256 * 33
    t_min = max(flops / PEAK_FP32, n_tiles_bytes / PEAK_BW)
    # oracle CPU rate on the first source images (self + all their neighbour blocks), stated as such
    sub_ng = {int(i): (list(fit.neighbors[int(i)]) if v < a.oracle_images else []) for v, i in enumerate(fit.img_ids)}
    sub = synth.FitScene(img_ids=fit.img_ids, model_ids=fit.model_ids, kvec=fit.kvec, qvec=fit.qvec, tvec=fit.tvec,
                         line_off=fit.line_off, segs=fit.segs, lines3d=fit.lines3d, neighbors=sub_ng)
    eng.merge_fits(sub.img_ids, sub.model_ids, sub.kvec, sub.qvec, sub.tvec, sub.line_off, sub.segs, sub.lines3d,
                   sub.ng_off, sub.ng_ids, mc.YAML_VAR2D, l2d, l3d)
    sub_tested = eng.fit_merge_stats()["n_pairs_tested"]
    threads = usable_cpus()
    t0 = time.perf_counter()
    orc.merge_to_linetracks(sub, mc.YAML_L2, mc.YAML_L3, mc.YAML_VAR2D, threads=threads)
    t_orc = time.perf_counter() - t0
    # parity of the timed output with the oracle on the full workload
    want = orc.merge_to_linetracks(fit, mc.YAML_L2, mc.YAML_L3, mc.YAML_VAR2D, threads=threads)
    ge, we = set(map(tuple, r["edges"].tolist())), set(map(tuple, want["edges"].tolist()))
    same_tracks = bool(np.array_equal(r["track_off"], want["track_off"])
                       and np.array_equal(r["track_nodes"], want["track_nodes"]))
    parity = dict(nodes=bool(np.array_equal(r["node_line"], want["node_line"])),
                  edges_in_order=bool(np.array_equal(r["edges"], want["edges"])
                                      and r["sim"].tobytes() == want["sim"].tobytes()),
                  edges_only_cuda=len(ge - we), edges_only_oracle=len(we - ge), tracks=same_tracks,
                  max_track_line_diff=float(np.abs(r["track_line"] - want["track_line"]).max()) if same_tracks else None)
    parity["ok"] = bool(parity["nodes"] and parity["edges_in_order"] and same_tracks
                        and parity["max_track_line_diff"] <= 1e-9)
    name, pl = card()
    print(json.dumps(dict(
        workload="fitnmerge100" if (a.V, a.L) == (100, 1000) else f"V{a.V}_L{a.L}_all_neighbours",
        gpu=name, power_limit=pl, V=a.V, L=a.L, lines=int(fit.line_off[-1]), nodes=st["n_nodes"],
        pairs_tested=tested, pairs_past_gates=st["n_pairs_gated"], edges=st["n_edges"], tracks=st["n_tracks"],
        pair_kernel_ms=tk * 1e3, end_to_end_ms=te * 1e3, pair_checks_per_s_kernel=tested / tk,
        pair_checks_per_s_end_to_end=tested / te,
        roofline=dict(gate_flops=flops, tile_bytes=n_tiles_bytes, min_time_ms=t_min * 1e3,
                      bound="fp32" if flops / PEAK_FP32 > n_tiles_bytes / PEAK_BW else "bandwidth",
                      share_of_peak=t_min / tk),
        oracle_cpu=dict(source_images=a.oracle_images, pairs_tested=sub_tested, seconds=t_orc, threads=threads,
                        pair_checks_per_s=sub_tested / t_orc, note="fp64 oracle on a subset of source images"),
        parity_with_oracle=parity)))


if __name__ == "__main__":
    main()
