"""GPU: the cell-major scan (scan.cu, cell_stage) on every configuration its gate accepts (test_cell_major_gate_cpu.py):
d/M = 1, 2, 4 and 8, padded M (36 .. 60, padding sub-quantizers in the LUT and the code blocks), cosine, a batch of two
query chunks, and an index of 3000 cells where empty cells and cells under one block sit next to cells split into
several work items.

Each search is checked three ways: against the integer oracle (O.search, or O.ivfpq_topk on given probe lists), where
every score is exact, so values, addresses and ids must match bit for bit; against the fp32 restatement
(fp32_exact.search_cells_fp32) on real-valued data, which integers cannot give (fmaf against mul + add in a LUT entry);
and against the query-major kernel, which the same queries reach in sliced batches of 100.

The 1536 live vectors per cell from which the gate takes the cell-major scan are a speed threshold, not a correctness
one, so the skewed index forces the scan by raising the layout's mean_cell_live: skewed data at the scale of 4096 cells
reaches the same states naturally, and forcing only shrinks the data they need.  Any change of the index rebuilds its
layout, so the force holds only until then."""
import functools

import numpy as np
import pytest
import torch

from oracle import build_state as B, ivfpq_oracle as O
from helpers import make_index
from test_baseline_configs_gpu import _unit_queries
from test_cell_major_gate_cpu import takes_cell_major
from test_cell_scan_gpu import NQ, assert_same, in_small_batches
from test_fp32_exact_gpu import _randn, run_search
from test_scan_plan_gpu import CELL, launched

pytestmark = pytest.mark.gpu

N_PROBE = 4
KS = (1, 100, 1024)            # the oracle runs once at k = 1024; its prefixes are the answers at smaller k
CHUNK = 16384                  # queries per scan launch (scan.cu, kQueryChunk)
CAP = 8192                     # survivors kept per query at k <= 1024 (cell_cap)


def assert_cell_major(ix, nq, n_probe, k):
    assert takes_cell_major(ix.layout().cindex, nq, n_probe, k), "the search does not take the cell-major scan"


def force_cell_major(ix, nq, n_probe, k):
    ix.layout().cindex.mean_cell_live = 2 ** 31 - 1
    assert_cell_major(ix, nq, n_probe, k)


def searcher(ix, x):
    return lambda s, e, k: ix.search(x[:, s:e].contiguous(), k=k, return_address=True, return_keys=True)


def cells_searcher(ix, x, cells, npl):
    return lambda s, e, k: ix.search_cells(x[:, s:e].contiguous(), cells[s:e].contiguous(),
                                           n_probe_list=npl[s:e].contiguous(), k=k, return_address=True,
                                           return_keys=True)


def assert_oracle(got, want, k, rows=slice(None)):
    """got: (values, ids, address, keys) of the GPU; want: the oracle's (values, ids, address) at k = 1024"""
    v, i, a = (t.cpu().numpy() for t in got[:3])
    ov, oi, oa = (w[:, :k] for w in want)
    assert np.array_equal(v[rows].view(np.uint32), ov[rows].view(np.uint32)), "values differ from the oracle"
    assert np.array_equal(a[rows], oa[rows]), "addresses differ from the oracle"
    assert np.array_equal(i[rows], oi[rows]), "ids differ from the oracle"


def check(ix, fn, nq, n_probe, want):
    """for each k: the unsliced batch takes the cell-major scan and equals the oracle's prefix and the same queries
    in sliced batches (the query-major kernel), keys included"""
    for k in KS:
        assert_cell_major(ix, nq, n_probe, k)
        big = fn(0, nq, k)
        assert_oracle(big, want, k)
        assert_same(big, in_small_batches(lambda s, e: fn(s, e, k), nq))


def oracle_cells(st, x, cells, npl, k):
    """tpq_ivfpq_search_cells in the integer oracle: the given probe lists, list lengths and x as given"""
    x = torch.as_tensor(x, dtype=torch.float32)
    cells, npl = np.asarray(cells), np.asarray(npl)
    lut = O.precompute_adc(x, torch.from_numpy(st.pq_codebook), st.distance).numpy()
    v, a = O.ivfpq_topk(st.storage, lut, st.is_empty, st.cell_start[cells], st.cell_size[cells], npl, k)
    return v, O.get_id_by_address(st.address2id, a), a


# ----------------------------------------------------------------------------------------- unforced shapes
# 8 cells of 2000 live vectors on average: the gate takes the cell-major scan on its own
SHAPES = {                      # name -> (d, M, distance)
    "dsub1": (64, 64, "euclidean"),
    "dsub4": (256, 64, "euclidean"),
    "dsub8": (512, 64, "euclidean"),
    "m36_dsub1": (36, 36, "euclidean"),
    "m48_dsub2": (96, 48, "euclidean"),
    "m60_dsub8": (480, 60, "euclidean"),
    "cosine": (128, 64, "cosine"),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_integer(cuda_device, shape):
    d, M, distance = SHAPES[shape]
    if distance == "cosine":
        # +-1 on 64 coordinates: the norm is 8, so the normalised queries and every score are exact
        st, _ = B.integer_state(d, M, 8, 16000, seed=M + d, distance=distance, lo=-2, hi=3)
        x = _unit_queries(d, NQ, 64, seed=3)
    else:
        st, queries = B.integer_state(d, M, 8, 16000, seed=M + d)
        x = queries(NQ, qseed=d)
    st.n_probe, st.use_smart_probing = N_PROBE, False
    ix = make_index(st)
    assert ix.layout().m_pad == 64
    want = O.search(st, x, k=KS[-1], return_address=True)
    check(ix, searcher(ix, x.cuda()), NQ, N_PROBE, want)


@pytest.mark.parametrize("shape", ["dsub1", "dsub8", "m36_dsub1", "cosine"])
def test_real_valued(cuda_device, shape):
    """the fp32 restatement on a subset of the rows, with smart probing"""
    d, M, distance = SHAPES[shape]
    st = B.randn_state(d, M, 8, 16000, seed=M * d, distance=distance)
    st.n_probe = N_PROBE
    ix = make_index(st)
    assert_cell_major(ix, NQ, N_PROBE, 100)
    rows = np.r_[0:16, 296:304, NQ - 16:NQ]
    x = _randn((d, NQ), M + d, 4.0 if distance == "cosine" else 1.0)
    run_search(st, x, 100, ix=ix, rows=rows, m_pad=64)


@pytest.mark.parametrize("dsub", [1, 4, 8])
def test_launch_census(cuda_device, dsub):
    """the LUTs come from cell_lut_kernel<d/M>, never from lut_kernel"""
    st, queries = B.integer_state(64 * dsub, 64, 8, 16000, seed=21)
    st.n_probe, st.use_smart_probing = N_PROBE, False
    ix = make_index(st)
    assert_cell_major(ix, NQ, N_PROBE, 10)
    x = queries(NQ).cuda()
    names = launched(lambda: ix.search(x, k=10))
    assert names == CELL - {"cell_lut_kernel<2>"} | {f"cell_lut_kernel<{dsub}>"}
    assert not any(n.startswith("lut_kernel") for n in names)


# ----------------------------------------------------------------------------------------- the skewed index (forced)
SK_D, SK_M, SK_C = 128, 64, 3000


@functools.lru_cache(maxsize=None)
def skewed():
    """3000 cells: 4 of about 6000 vectors (188 blocks, three work items of at most 84 blocks each), 300 of about 300,
    1000 of 1 .. 31 (under one block) and 1696 empty.  The container starts at 8 slots per cell and grows the large
    cells as the reference's does, so its capacity stays near twice the vectors.  Every other cell with a partial last
    block has a hole in it, and each large cell 200 holes anywhere.  -> (state, integer queries, the cell groups)"""
    rng = np.random.default_rng(7)
    order = rng.permutation(SK_C)
    big, mid, tiny, empty = order[:4], order[4:304], order[304:1304], order[1304:]
    sizes = np.zeros(SK_C, np.int64)
    sizes[big] = 6000 + rng.integers(-16, 16, big.shape[0])
    sizes[mid] = rng.integers(250, 350, mid.shape[0])
    sizes[tiny] = rng.integers(1, 32, tiny.shape[0])
    cells = np.repeat(np.arange(SK_C), sizes)
    rng.shuffle(cells)
    vq = rng.integers(-3, 4, size=(SK_D, SK_C)).astype(np.float32)
    pq = rng.integers(-3, 4, size=(SK_M, SK_D // SK_M, 256)).astype(np.float32)
    codes = rng.integers(0, 256, size=(SK_M, cells.shape[0])).astype(np.uint8)
    st = O.empty_state(SK_D, SK_M, SK_C, 8, "euclidean", vq, pq)
    O.container_add(st, codes, cells)
    assert st.capacity < 2 * cells.shape[0]
    for c in np.flatnonzero(sizes % 32)[::2]:
        st.is_empty[st.cell_start[c] + sizes[c] // 32 * 32 + rng.integers(0, sizes[c] % 32)] = 1
    for c in big:
        st.is_empty[st.cell_start[c] + rng.choice(sizes[c], 200, replace=False)] = 1
    st.use_smart_probing = False

    def queries(nq, qseed=1):
        r = np.random.default_rng(qseed)
        return torch.from_numpy(r.integers(-3, 4, size=(SK_D, nq)).astype(np.float32))

    return st, queries, big, mid, tiny, empty


def live_of(st, c):
    s = int(st.cell_start[c])
    return int((st.is_empty[s:s + int(st.cell_size[c])] == 0).sum())


@pytest.mark.parametrize("n_probe", [1, 2, 16, 64])
def test_skewed_search(cuda_device, n_probe):
    """n_probe = 1: no pairs and no work items, pass 1 alone"""
    st, queries, *_ = skewed()
    st.n_probe = n_probe
    x = queries(NQ)
    want = O.search(st, x, k=KS[-1], return_address=True)
    ix = make_index(st)
    force_cell_major(ix, NQ, n_probe, KS[-1])
    check(ix, searcher(ix, x.cuda()), NQ, n_probe, want)


def designed_lists(st, nq, width, big, mid, tiny, empty, seed):
    """probe lists of `width` entries over the skewed index.  Entry 0 is an empty cell or a tiny one with fewer live
    vectors than k = 100, so the bound is 0 and every live vector of the later entries survives.  Rows 0, 4, 8, ...
    list two large cells (more than 8192 live vectors together: the query overflows its survivors and is re-run
    query-major); the other rows list medium and tiny cells.  Some rows repeat an entry in the next place (skipped) and
    some list a cell twice apart (scanned twice); some lists are cut short by their length."""
    rng = np.random.default_rng(seed)
    cells = np.empty((nq, width), np.int64)
    cells[:, 0] = np.where(np.arange(nq) % 2 == 0, rng.choice(empty, nq), rng.choice(tiny, nq))
    cells[:, 1:] = np.where(rng.random((nq, width - 1)) < 0.7, rng.choice(mid, (nq, width - 1)),
                            rng.choice(tiny, (nq, width - 1)))
    over = np.arange(0, nq, 4)
    pair = np.stack([rng.permutation(big)[:2] for _ in over])
    cells[over, 2], cells[over, width - 2] = pair[:, 0], pair[:, 1]
    cells[1::3, 4] = cells[1::3, 3]                                       # adjacent: skipped
    cells[2::5, 6] = cells[2::5, 1]                                       # apart: scanned twice
    npl = np.full(nq, width, np.int64)
    npl[3::8] = rng.integers(1, width, npl[3::8].shape[0])               # never rows 0, 4, 8, ...: they keep both
    assert min(live_of(st, a) + live_of(st, b) for a, b in pair) > CAP
    assert all(live_of(st, c) < 100 for c in cells[:, 0])
    return cells, npl


def test_skewed_search_cells(cuda_device):
    st, queries, big, mid, tiny, empty = skewed()
    x = queries(NQ, qseed=2)
    cells, npl = designed_lists(st, NQ, 12, big, mid, tiny, empty, seed=3)
    want = oracle_cells(st, x, cells, npl, KS[-1])
    ix = make_index(st)
    force_cell_major(ix, NQ, 12, KS[-1])
    check(ix, cells_searcher(ix, x.cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()), NQ, 12, want)


@pytest.mark.parametrize("k", [100, 1024])
def test_chunked_batch(cuda_device, k):
    """16384 + 700 queries run as two chunks of the cell-major stage (q_base 0 and 16384), with overflowing queries in
    both.  Every row equals the same rows searched as two batches of one chunk each, and the integer oracle on rows at
    both ends of both chunks.  The workspace is about 3 GB at k = 1024."""
    nq, width = CHUNK + 700, 12
    st, queries, big, mid, tiny, empty = skewed()
    x = queries(nq, qseed=4)
    cells, npl = designed_lists(st, nq, width, big, mid, tiny, empty, seed=5)
    ix = make_index(st)
    force_cell_major(ix, nq, width, k)
    for n in (CHUNK, nq - CHUNK):
        assert_cell_major(ix, n, width, k)
    fn = cells_searcher(ix, x.cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda())
    big_batch = fn(0, nq, k)
    parts = [fn(0, CHUNK, k), fn(CHUNK, nq, k)]
    assert_same(big_batch, [torch.cat(p, 0) for p in zip(*parts)])
    rows = np.r_[0:8, CHUNK - 8:CHUNK + 8, nq - 8:nq]
    want = oracle_cells(st, x[:, rows], cells[rows], npl[rows], k)
    assert_oracle([t[torch.from_numpy(rows).cuda()] for t in big_batch[:3]], want, k)
