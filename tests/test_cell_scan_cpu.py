"""CPU model of the cell-major scan (csrc/scan.cu, ivfpq_cell_scan_kernel and its passes): the probe-entry visiting
rules (probe_count and probe_entry in csrc/scan_layout.cuh, which both scan kernels call), the pair list grouped by
cell, and bound -> survivors -> select, checked against a plain per-query top-k over the entries the query-major kernel
visits."""
import numpy as np
import pytest

INT64_MIN = np.iinfo(np.int64).min


def n_visited(npl_q, n_probe):
    """P = max(1, min((int) n_probe_list[q], n_probe)); the C cast keeps the low 32 bits (INT64_MIN -> 0)."""
    p = int(np.int64(npl_q).astype(np.int32))
    return max(1, min(p, n_probe))


def visited(cq, j, cell_start, n_blocks):
    """The cell of entry j if the query-major kernel scans it, else -1 (outside [0, C), same start as the entry
    before, or no live block)."""
    C = cell_start.shape[0]
    c = int(cq[j])
    if c < 0 or c >= C:
        return -1
    if j > 0:
        cp = int(cq[j - 1])
        if 0 <= cp < C and cell_start[c] == cell_start[cp]:
            return -1
    return c if n_blocks[c] > 0 else -1


def query_major(keys_of, cells, npl, cell_start, n_blocks, k):
    """Reference: top k (with multiplicity) of every visited entry's keys, zero-padded."""
    out = np.zeros((cells.shape[0], k), dtype=np.uint64)
    for q in range(cells.shape[0]):
        P = n_visited(npl[q], cells.shape[1])
        cand = [keys_of[c] for j in range(P) if (c := visited(cells[q], j, cell_start, n_blocks)) >= 0]
        allk = np.sort(np.concatenate(cand + [np.zeros(0, np.uint64)]))[::-1][:k]
        out[q, :allk.shape[0]] = allk
    return out


def cell_major(keys_of, cells, npl, cell_start, n_blocks, k, cap):
    """pass 1 (entry 0) -> bound; pairs of entries 1..P-1 grouped by cell (counting sort); survivors > bound per query;
    select top k of pass-1 list + survivors; queries over `cap` survivors are re-run query-major."""
    nq, n_probe = cells.shape
    C = cell_start.shape[0]
    pass1 = query_major(keys_of, cells[:, :1], np.ones(nq, np.int64), cell_start, n_blocks, k)
    bound = pass1[:, k - 1]
    cnt = np.zeros(C, np.int64)
    slot = -np.ones((nq, n_probe), np.int64)
    for q in range(nq):
        for j in range(1, n_visited(npl[q], n_probe)):
            c = visited(cells[q], j, cell_start, n_blocks)
            if c >= 0:
                slot[q, j] = cnt[c]
                cnt[c] += 1
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    pair_q = np.full(int(cnt.sum()), -1, np.int64)
    for q in range(nq):
        for j in range(n_probe):
            if slot[q, j] >= 0:
                pair_q[off[cells[q, j]] + slot[q, j]] = q
    assert (pair_q >= 0).all()
    surv = [[] for _ in range(nq)]
    for c in range(C):
        for q in pair_q[off[c]:off[c] + cnt[c]]:
            surv[q].extend(keys_of[c][keys_of[c] > bound[q]])
    out = pass1.copy()
    rerun = []
    for q in range(nq):
        if len(surv[q]) > cap:
            rerun.append(q)
            continue
        allk = np.sort(np.concatenate([pass1[q], np.array(surv[q], np.uint64)]))[::-1][:k]
        out[q] = allk
    if rerun:
        out[rerun] = query_major(keys_of, cells[rerun], npl[rerun], cell_start, n_blocks, k)
    return out, [len(s) for s in surv], rerun


def make_cells(rng, C, sizes):
    allk = rng.permutation(np.arange(1, int(sizes.sum()) * 4 + 1, dtype=np.uint64))[:int(sizes.sum())]   # unique keys
    return np.split(allk, np.cumsum(sizes)[:-1])


@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cell_major_equals_query_major(k, seed):
    rng = np.random.default_rng(seed)
    C, nq, n_probe = 12, 40, 8
    sizes = rng.integers(0, 300, C)
    sizes[0] = 3                                                      # a first cell with fewer than k vectors
    keys_of = make_cells(rng, C, sizes)
    cell_start = np.cumsum(np.concatenate([[0], sizes[:-1]])).astype(np.int64)
    cell_start[5] = cell_start[4]                                     # two cells that share a start
    n_blocks = (sizes + 31) // 32
    cells = rng.integers(-2, C + 2, (nq, n_probe))                    # entries outside [0, C) are empty
    cells[::4, 0] = 0                                                 # bound 0 from the small cell
    cells[1::4, 2] = cells[1::4, 1]                                   # skipped: same cell as the entry before
    cells[2::4, 6] = cells[2::4, 3]                                   # scanned twice
    cells[3::4, 3:5] = [4, 5]                                         # skipped: same start as the entry before
    npl = rng.integers(0, n_probe + 3, nq).astype(np.int64)           # smart-probing lists, clamped to n_probe
    npl[::5] = INT64_MIN                                              # the NaN quirk: scans entry 0 only
    want = query_major(keys_of, cells, npl, cell_start, n_blocks, k)
    got, n_surv, rerun = cell_major(keys_of, cells, npl, cell_start, n_blocks, k, cap=10 ** 9)
    assert not rerun
    assert np.array_equal(got, want)
    assert max(n_surv) > 0                                            # the survivors path was exercised


def test_overflow_is_rerun_query_major():
    rng = np.random.default_rng(7)
    C, nq, n_probe, k = 6, 30, 5, 10
    sizes = np.array([2, 400, 400, 400, 400, 400])
    keys_of = make_cells(rng, C, sizes)
    cell_start = np.cumsum(np.concatenate([[0], sizes[:-1]])).astype(np.int64)
    n_blocks = (sizes + 31) // 32
    cells = np.stack([np.concatenate([[0], rng.permutation(5) + 1])[:n_probe] for _ in range(nq)])
    npl = np.full(nq, n_probe, np.int64)
    npl[::2] = 2
    want = query_major(keys_of, cells, npl, cell_start, n_blocks, k)
    got, n_surv, rerun = cell_major(keys_of, cells, npl, cell_start, n_blocks, k, cap=500)
    assert rerun and set(rerun) == {q for q in range(nq) if n_surv[q] > 500}
    assert all(q % 2 == 1 for q in rerun)                             # bound 0 with 4 large cells: all overflow
    assert np.array_equal(got, want)
