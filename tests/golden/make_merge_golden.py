"""Regenerates tests/golden/ref/merge_to_linetracks_*.npz: the outputs of the reference's own merging.merging
(SetUncertaintySegs3d + MergeToLineTracks of its merging.cc, compiled unchanged into oracle/_ref by build(), which is only
possible where the reference source tree is present) on the seeded cases of tests/merge_fit_cases.py.

Run from the repository root:  python tests/golden/make_merge_golden.py [case ...]   (no names: every case)"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import merge_fit_cases as mc  # noqa: E402
from oracle import merge_fits, ref  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "ref")


def main():
    ref.build()
    merge_fits.build()
    if not os.path.exists(merge_fits.REF_LIB):
        raise SystemExit("oracle/_ref/liblimap_ref_merge.so is missing: the reference source tree is needed to build it")
    names = sys.argv[1:] or list(mc.CASES)
    unknown = sorted(set(names) - set(mc.CASES))
    if unknown:
        raise SystemExit(f"unknown cases: {unknown}")
    for name in names:
        path = os.path.join(GOLD, f"merge_to_linetracks_{name}.npz")
        np.savez_compressed(path, **merge_fits.ref_merge_to_linetracks(*mc.case(name)))
        print(f"{path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
