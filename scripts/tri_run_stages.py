"""Where the time of one resident lm_tri_run step goes: bench.py's value leg (the hypersim100 scene, its matches already
in HBM, one pipeline group) under torch.profiler with CUDA activities, in a run of its own. Prints the device time per
step of every kernel and copy the step launches, and last_run_ms - last_node_kernel_ms from the engine's own events
(measured with the profiler off, before the profiled steps). Writes stages.json (and the trace with --trace) under OUT.

    python scripts/tri_run_stages.py OUT [--steps 10] [--warmup 3] [--trace]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_name_and_power():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", action="store_true", help="also write the Chrome trace")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from limap_b200.config import DEFAULT_YAML_TRIANGULATION
    from limap_b200.engine import TriEngine
    from limap_b200.synth import CONFIGS, make_scene

    if not torch.cuda.is_available():
        raise SystemExit("tri_run_stages.py needs a CUDA device")
    scene = make_scene(**CONFIGS["hypersim100"])
    eng = TriEngine(dict(DEFAULT_YAML_TRIANGULATION))
    eng.ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    eng.upload(scene)
    eng.set_ranges(*scene.ranges)
    for i in scene.img_ids:
        eng.add_image_matches(int(i), *scene.flat_matches(int(i)))
    eng.set_pipeline_groups(1)

    for _ in range(args.warmup):
        eng.run()
    run_ms, node_ms = [], []
    for _ in range(args.steps):  # profiler off
        st = eng.run()
        run_ms.append(st["last_run_ms"])
        node_ms.append(st["last_node_kernel_ms"])
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            eng.run()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t and t > 0:
            per[ev.key] = dict(ms_per_step=t / 1e3 / args.steps, calls_per_step=ev.count / args.steps)
    rows = sorted(per.items(), key=lambda kv: -kv[1]["ms_per_step"])
    res = dict(gpu=gpu_name_and_power(), n_rows=int(scene.n_rows()), steps=args.steps,
               last_run_ms=float(np.median(run_ms)), last_node_kernel_ms=float(np.median(node_ms)),
               outside_node_kernel_ms=float(np.median(np.asarray(run_ms) - np.asarray(node_ms))),
               kernels=[dict(name=k, **v) for k, v in rows])
    print(f"gpu: {res['gpu']}  rows: {res['n_rows']}")
    print(f"last_run_ms {res['last_run_ms']:.3f}  last_node_kernel_ms {res['last_node_kernel_ms']:.3f}  "
          f"outside the node kernel {res['outside_node_kernel_ms']:.3f} ms (medians over {args.steps} steps)")
    print(f"{'ms/step':>9} {'calls':>6}  kernel / copy")
    for k, v in rows:
        print(f"{v['ms_per_step']:9.4f} {v['calls_per_step']:6.1f}  {k[:110]}")
    with open(os.path.join(args.out, "stages.json"), "w") as f:
        json.dump(res, f, indent=1)
    if args.trace:
        prof.export_chrome_trace(os.path.join(args.out, "tri_run_stages.pt.trace.json"))


if __name__ == "__main__":
    main()
