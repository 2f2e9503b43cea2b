"""GPU: the cell-major scan (cells of > 1536 live vectors on average, M <= 64, unsliced batches) returns what the
query-major kernel returns, bit for bit.  The same index reaches the query-major kernel in batches small enough to be
sliced (fewer than 4 x SMs queries), so every test searches one large batch and compares it with the same queries
searched in small batches."""
import numpy as np
import pytest
import torch

from oracle import ivfpq_oracle as O, build_state as B
from helpers import make_index

pytestmark = pytest.mark.gpu

NQ = 600          # > 4 x 132 SMs: one unsliced batch
SMALL = 100       # sliced batches: the query-major kernel


def cell_major_index(st):
    """The index, after checking that the library takes the cell-major scan for NQ queries: only that path asks for
    LUT and survivor buffers, so its workspace exceeds that of the same index below the threshold by at least those."""
    import ctypes as C
    import torchpq_b200 as T
    ix = make_index(st)
    cix = ix.layout().cindex
    below = T._lib.TpqIndex.from_buffer_copy(cix)
    below.mean_cell_live = 0
    ws = lambda s, nq: T._lib.lib.tpq_search_workspace_bytes(C.byref(s), nq, 4, 1)
    assert ws(cix, NQ) - ws(below, NQ) >= NQ * (65536 + 8192 * 8), "fixture does not select the cell-major scan"
    assert ws(cix, SMALL) == ws(below, SMALL), "small batches must keep the query-major kernel"
    return ix


def in_small_batches(fn, nq):
    outs = [fn(s, min(nq, s + SMALL)) for s in range(0, nq, SMALL)]
    return [torch.cat(parts, 0) for parts in zip(*outs)]


def assert_same(big, small):
    for a, b in zip(big, small):
        assert torch.equal(a.cpu(), b.cpu())


def search_both(ix, x, k):
    big = ix.search(x, k=k, return_address=True, return_keys=True)
    small = in_small_batches(lambda s, e: ix.search(x[:, s:e].contiguous(), k=k, return_address=True,
                                                    return_keys=True), x.shape[1])
    return big, small


@pytest.mark.parametrize("k", [1, 100, 1024])
@pytest.mark.parametrize("smart", [False, True])
def test_integer_kat(cuda_device, k, smart):
    st, queries = B.integer_state(128, 64, 8, 16000, seed=21 + k)
    st.n_probe, st.use_smart_probing = 4, smart
    x = queries(NQ)
    ix = cell_major_index(st)
    big, small = search_both(ix, x.cuda(), k)
    assert_same(big, small)
    ov, oi, oa = O.search(st, x, k=k, return_address=True)
    assert np.array_equal(big[0].cpu().numpy(), ov)
    assert np.array_equal(big[2].cpu().numpy(), oa)
    assert np.array_equal(big[1].cpu().numpy(), oi)


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_randn(cuda_device, k):
    torch.manual_seed(5)
    base = torch.randn(128, 20000)
    st = B.build_state(base, 64, 8, vq_iters=3, pq_iters=2, n_train=8000)
    st.n_probe, st.use_smart_probing = 5, True
    ix = cell_major_index(st)
    big, small = search_both(ix, torch.randn(128, NQ).cuda(), k)
    assert_same(big, small)


def test_is_empty_holes(cuda_device):
    st, queries = B.integer_state(128, 64, 8, 20000, seed=4)
    rng = np.random.default_rng(1)
    live = np.flatnonzero(st.is_empty == 0)
    holes = rng.choice(live, 3000, replace=False)
    st.is_empty[holes] = 1
    st.n_probe, st.use_smart_probing = 4, False
    x = queries(NQ)
    ix = cell_major_index(st)
    big, small = search_both(ix, x.cuda(), 100)
    assert_same(big, small)
    ov, oi, oa = O.search(st, x, k=100, return_address=True)
    assert np.array_equal(big[0].cpu().numpy(), ov) and np.array_equal(big[2].cpu().numpy(), oa)
    assert not np.isin(big[2].cpu().numpy(), holes).any()


def search_cells_both(ix, x, cells, npl, k):
    big = ix.search_cells(x, cells, n_probe_list=npl, k=k, return_address=True, return_keys=True)
    small = in_small_batches(lambda s, e: ix.search_cells(x[:, s:e].contiguous(), cells[s:e].contiguous(),
                                                          n_probe_list=npl[s:e].contiguous(), k=k, return_address=True,
                                                          return_keys=True), x.shape[1])
    return big, small


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_search_cells_skipped_and_duplicate_entries(cuda_device, k):
    """Adjacent equal entries are skipped, a cell listed twice apart is scanned twice, entries outside [0, C) are empty,
    and per-query list lengths (with the NaN -> INT64_MIN quirk) cut the lists."""
    st, queries = B.integer_state(128, 64, 8, 16000, seed=9)
    x = queries(NQ).cuda()
    ix = cell_major_index(st)
    g = torch.Generator().manual_seed(3)
    cells = torch.randint(-1, 9, (NQ, 10), generator=g)                  # -1 and 8 are outside [0, 8)
    cells[::3, 1] = cells[::3, 0]                                         # skipped: same cell as the entry before
    cells[1::3, 5] = cells[1::3, 2]                                       # scanned twice
    npl = torch.randint(0, 12, (NQ,), generator=g)
    npl[::7] = torch.iinfo(torch.int64).min
    big, small = search_cells_both(ix, x, cells.cuda(), npl.cuda(), k)
    assert_same(big, small)


def test_overflow_reruns_query_major(cuda_device):
    """A first probed cell with fewer than k live vectors gives the bound 0: every live vector of the other probed cells
    survives, more than the survivor capacity (8192 at k = 100), so those queries are scanned again query-major."""
    st, queries = B.integer_state(128, 64, 8, 24000, seed=13)
    cell0 = np.arange(st.cell_start[0], st.cell_start[0] + st.cell_size[0])
    st.is_empty[cell0[10:]] = 1                                           # cell 0 keeps 10 live vectors
    x = queries(NQ).cuda()
    ix = cell_major_index(st)
    g = torch.Generator().manual_seed(4)
    cells = torch.stack([torch.randperm(7, generator=g) + 1 for _ in range(NQ)])
    cells = torch.cat([torch.zeros(NQ, 1, dtype=torch.long), cells], 1)  # entry 0 = the small cell
    live = np.array([(st.is_empty[s:s + n] == 0).sum() for s, n in zip(st.cell_start, st.cell_size)])
    assert live[1:].sum() > 8192 and live[0] < 100
    npl = torch.full((NQ,), 8, dtype=torch.long)
    npl[::2] = 2                                                          # and queries that stay below the capacity
    big, small = search_cells_both(ix, x, cells.cuda(), npl.cuda(), 100)
    assert_same(big, small)
