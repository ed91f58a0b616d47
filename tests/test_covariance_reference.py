"""The covariance fixture tests/golden/ref_covariances.npz against the live reference, without a GPU: the unmodified
Covariances.cpp / covariance.cpp run against the CHOLMOD stand-in's R (oracle/ref_shim) after one Slam::update() and give
the fixture's values.  Skips where the reference checkout or oracle/_ref/obj is absent; the GPU side compares against the
fixture (tests/test_gpu_covariance.py)."""
import numpy as np
import pytest

import cov_ref_api
from cov_golden import CASES, GOLDEN, build

pytestmark = pytest.mark.skipif(not cov_ref_api.available(), reason="needs the reference checkout and oracle/_ref/obj")


@pytest.mark.parametrize("case", list(CASES))
def test_reference_covariances_match_the_fixture(case):
    r = cov_ref_api.RefCovAPI()
    pairs, dims = build(r, case)
    r.update()
    blocks = r.covariance_blocks(pairs, dims)
    got = np.concatenate([B.ravel() for B in blocks])
    want = np.load(GOLDEN)[case]
    assert got.shape == want.shape
    assert np.allclose(got, want, rtol=1e-12, atol=0), np.abs(got - want).max()
    n_own = sum(1 for a, b in pairs if a == b)
    for B in blocks[:n_own]:   # every node's own block: symmetric positive definite
        assert np.allclose(B, B.T, rtol=0, atol=1e-12 * np.abs(B).max())
        assert np.linalg.eigvalsh(0.5 * (B + B.T)).min() > 0
