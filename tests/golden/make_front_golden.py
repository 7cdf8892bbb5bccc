"""Writes tests/golden/ref_pin_front.npz: the reference's own A* front end (oracle/_ref/libref_front_portable.so, built by
`make -C oracle ref` where the reference tree exists) on the case matrix of tests/front_cases.py.  Large outputs (kernels, the
configuration-space map, the AABB point lists, the packed map) are SHA-256 digests; node-test outputs and paths are stored
whole.  Running it again writes the same bytes.  Also checks that the glibc variant gives the same booleans, yaws and paths.

    python tests/golden/make_front_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import front_cases as FC  # noqa: E402

if __name__ == "__main__":
    rec = FC.reference_records("portable")
    glibc = FC.reference_records("glibc")
    assert rec.keys() == glibc.keys()
    # glibc's last bit can flip a sub-swept-volume test where a sample lands on sdf = 0 (DESIGN.md §4); the matrix has no such
    # sample, and a change that brings one in must be looked at, not recorded
    differ = [k for k in rec if not np.array_equal(rec[k], glibc[k])]
    if differ:
        sys.exit(f"the glibc variant differs from the portable one in {differ}")
    FC.save_npz(os.path.join(HERE, "ref_pin_front.npz"), rec)
    print("ref_pin_front.npz:", len(rec), "arrays,", os.path.getsize(os.path.join(HERE, "ref_pin_front.npz")), "bytes")
