"""The wgmma / TMA product of the tensor-core kernels against fp64 numpy, for each ring depth: tile capacities of 32
and 64 rows stream the weights through the three-stage ring (third stage in the A buffer's upper half), 128 rows
through the two-stage one.  Several repetitions in one launch wrap the ring, so every stage is refilled with both
barrier parities."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows", [32, 64, 128])
@pytest.mark.parametrize("reps", [1, 7])
def test_tc_product_matches_fp64(rows, reps):
    from ai2bmd_b200.engine import tc_selftest
    rng = np.random.default_rng(rows + reps)
    a = rng.normal(size=(rows, 128)).astype(np.float32)
    w = (rng.normal(size=(128, 128)) * 0.1).astype(np.float32)
    d, _ = tc_selftest(a, w, reps=reps, rows=rows)
    ref = a.astype(np.float64) @ w.astype(np.float64).T
    assert d.shape == (rows, 128)
    assert np.abs(d - ref).max() / np.abs(ref).max() < 2e-6
