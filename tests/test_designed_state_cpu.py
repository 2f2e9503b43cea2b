"""CPU: the designed-score construction of tests/designed_state.py is exact.  The reference's restatement
(O.search, m-ascending fp32 sums) and the scan kernels' own arithmetic (fp32_exact.search_cells_fp32: lane-rotated
sub-quantizers in four partial sums) must both return exactly the designed scores and addresses, so the GPU tests can
take their expected answers straight from the designed table."""
import numpy as np
import pytest

from oracle import ivfpq_oracle as O, fp32_exact as X
from designed_state import Designed, PATTERNS, design, score_range


def test_every_code_reaches_its_square_sum():
    from designed_state import FOUR
    assert (FOUR < 16).all() and np.array_equal((FOUR ** 2).sum(1), np.arange(256))


@pytest.mark.parametrize("distance, M, dsub", [("euclidean", 8, 4), ("euclidean", 16, 12), ("cosine", 8, 4)])
def test_extreme_and_random_scores_are_exact(distance, M, dsub):
    rng = np.random.default_rng(M + dsub)
    D = Designed([700, 1000, 300], M=M, dsub=dsub, distance=distance)
    lo, hi = score_range(distance)
    live = np.flatnonzero(D.st.is_empty == 0)
    s = rng.choice(np.arange(lo, hi + 1), live.shape[0], replace=False)
    s[:4] = [lo, hi, lo + 1, hi - 1]
    D.set_scores(live, s)
    D.st.n_probe = 3
    x = D.queries(2)
    k = 50
    ev, ea, ei = D.expected(np.array([[0, 1, 2]] * 2), np.array([3, 3]), k)
    ov, oi, oa = O.search(D.st, x * (2 if distance == "cosine" else 1), k=k, return_address=True)
    assert np.array_equal(ov, ev) and np.array_equal(oa, ea) and np.array_equal(oi, ei)
    xv, xa = X.search_cells_fp32(D.st, x.numpy(), np.array([[0, 1, 2]] * 2), np.array([3, 3]), k)
    assert np.array_equal(xv.view(np.uint32), ev.view(np.uint32)) and np.array_equal(xa, ea)


@pytest.mark.parametrize("pattern", PATTERNS)
def test_patterns_through_the_scan_arithmetic(pattern):
    """every pattern on a probe list that skips an entry, lists a cell twice apart and has holes"""
    rng = np.random.default_rng(len(pattern))
    D = Designed([520, 1000, 333, 64, 700], M=8, dsub=4)
    D.st.is_empty[D.cell_slots(2)[::5]] = 1
    row = [1, 1, 4, 2, 3, 4]
    design(D, row, pattern, rng, k=100, nw=8, leaders=40)
    cells, npl = np.array([row, row[:3] + [0, 0, 0]]), np.array([6, 3])
    for k in (1, 33, 100, 1024):
        ev, ea, _ = D.expected(cells, npl, k)
        xv, xa = X.search_cells_fp32(D.st, D.queries(2).numpy(), cells, npl, k)
        assert np.array_equal(xv.view(np.uint32), ev.view(np.uint32)) and np.array_equal(xa, ea)
    if pattern == "bound":
        ev, ea, _ = D.expected(cells[:1], npl[:1], 100)
        assert np.array_equal(ev[0], (score_range("euclidean")[1] - np.arange(1, 101)).astype(np.float32))
