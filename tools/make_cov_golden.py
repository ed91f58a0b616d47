"""Writes tests/golden/ref_covariances.npz: the reference's own Slam::covariances().access (the unmodified Covariances.cpp
and covariance.cpp behind oracle/ref_shim) right after one Slam::update() on the graphs of tests/cov_golden.py.  Needs the
reference checkout and `make -C oracle ref`.

    python tools/make_cov_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cov_golden import CASES, GOLDEN, build  # noqa: E402
from cov_ref_api import RefCovAPI  # noqa: E402


def reference_blocks(case):
    r = RefCovAPI()
    pairs, dims = build(r, case)
    r.update()
    return np.concatenate([B.ravel() for B in r.covariance_blocks(pairs, dims)])


def main():
    np.savez_compressed(GOLDEN, **{case: reference_blocks(case) for case in CASES})
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
