"""Regenerates tests/golden/ref/*.npz: the outputs of the reference's own hot-path sources (compiled unchanged into
oracle/_ref by build(), which is only possible where the reference source tree is present) on the seeded inputs of
tests/test_ref_pinning.py, which compares the oracle and the Python mirror against them, and the results of the
reference's own runner file (src/limap/runners/line_triangulation.py) on the scene of tests/test_runner_dropin.py.

Run from the repository root:  python tests/golden/make_ref_golden.py [name ...]
(no names: every file; names: only tests/golden/ref/<name>.npz)"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

from oracle import ref  # noqa: E402
import test_ref_pinning as t  # noqa: E402
import test_runner_dropin as rd  # noqa: E402


def main():
    ref.build()
    if not ref.available():
        raise SystemExit("oracle/_ref/liblimap_ref.so is missing: the reference source tree is needed to build it")
    os.makedirs(t.GOLD, exist_ok=True)
    runner = os.path.join(ref.REFERENCE_SRC, "limap", "runners", "line_triangulation.py")
    outputs = dict(t.REFERENCE_OUTPUTS, runner_line_triangulation=lambda: rd.reference_runner_outputs(runner))
    names = sys.argv[1:] or list(outputs)
    unknown = sorted(set(names) - set(outputs))
    if unknown:
        raise SystemExit(f"unknown golden files: {unknown}")
    for name in names:
        make = outputs[name]
        path = os.path.join(t.GOLD, name + ".npz")
        np.savez_compressed(path, **make())
        print(f"{path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
