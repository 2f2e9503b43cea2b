"""GPU: the cell-major kernel's survivor log (scan.cu, ivfpq_cell_scan_kernel).  A warp appends a pair's survivors to
the pair's bucket of its CTA's log; after the window's last pair the CTA reserves every bucket's place in its query's
survivor list with one atomic per pair and copies the buckets whose query has not overflowed.  These cases reach what
the log adds: a bucket filled to its last key, a query that crosses its capacity inside one window's flush, and a query
that reaches its capacity exactly through pairs of different items and windows.

Every cell F* is 84 full blocks, exactly one work item (12 warps x 7 blocks), and E0 has fewer live vectors than k, so
a query whose entry 0 is E0 has the bound 0 and every live vector it probes afterwards survives: a pair on F* puts 2688
keys, one whole bucket, into the log.  Results must equal the designed answer and the query-major kernel's bit for
bit."""
import numpy as np
import pytest
import torch

from designed_state import Designed, score_range
from test_cell_scan_gpu import cell_major_index, in_small_batches
from test_scan_plan_gpu import launched
from test_topk_adversarial_gpu import assert_exact, batch

pytestmark = pytest.mark.gpu

NQ = 600                    # > 4 x 132 SMs: one unsliced batch, the cell-major scan
CAP = 8192                  # survivors kept per query at k <= 1024 (cell_cap)
FULL = 84 * 32              # keys of a full chunk: one bucket


def log_state():
    sizes = {"E0": 50, "F1": FULL, "F2": FULL, "F3": FULL, "F4": FULL, "T": CAP - 3 * FULL, "T1": CAP - 3 * FULL + 1}
    names = list(sizes)
    D = Designed([sizes[n] for n in names], M=64, dsub=4)
    live = np.flatnonzero(D.st.is_empty == 0)
    top = score_range("euclidean")[1]
    D.set_scores(live, top - 3 * np.random.default_rng(5).permutation(live.shape[0]))
    return D, {n: i for i, n in enumerate(names)}


def check(D, rows, k):
    ix = cell_major_index(D.st)
    cells, npl = batch(rows, NQ)
    x, cg, ng = D.queries(NQ).cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()
    assert "ivfpq_cell_scan_kernel<12, 7>" in launched(lambda: ix.search_cells(x, cg, n_probe_list=ng, k=k))
    big = ix.search_cells(x, cg, n_probe_list=ng, k=k, return_address=True, return_keys=True)
    assert_exact(D, big, cells, npl, k)
    small = in_small_batches(lambda s, e: ix.search_cells(x[:, s:e].contiguous(), cg[s:e].contiguous(),
                                                          n_probe_list=ng[s:e].contiguous(), k=k, return_address=True,
                                                          return_keys=True), NQ)
    for a, b in zip(big, small):
        assert torch.equal(a.cpu(), b.cpu())


@pytest.mark.parametrize("k", [100, 1024])
def test_full_buckets_and_capacity_across_items_and_windows(cuda_device, k):
    """Every query probes F1 (600 pairs: three windows), F2 and F3 (400 pairs: two windows) with the bound 0.  Row 0
    reaches the capacity exactly through four items (3 x 2688 + 128 = 8192 survivors, copied), row 1 passes it by one
    (re-run query-major), row 2 fills one bucket and nothing else."""
    D, c = log_state()
    E0, F1, F2, F3, T, T1 = (c[n] for n in ("E0", "F1", "F2", "F3", "T", "T1"))
    check(D, [[E0, F1, F2, F3, T], [E0, F1, F2, F3, T1], [E0, F1]], k)


@pytest.mark.parametrize("k", [100, 1024])
def test_capacity_crossed_inside_one_flush(cuda_device, k):
    """Six queries list F1 four times apart (4 x 2688 = 10752 survivors from one item) and T three times: F1 has 24
    pairs, all in one window, so whichever order the CTAs' flushes take, some of a query's F1 buckets fit under the
    capacity and are copied and the rest are not, and the query is re-run.  The other rows keep their survivors."""
    D, c = log_state()
    E0, F1, F2, F3, F4, T = (c[n] for n in ("E0", "F1", "F2", "F3", "F4", "T"))
    rows = [[E0, F1, T, F1, T, F1, T, F1]] + [[E0, F2], [E0, F3, F4], [E0, F4, T], [F2, F3]] * 25
    check(D, rows[:100], k)
