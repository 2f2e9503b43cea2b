"""GPU: IVFPQIndex.range_search and tpq_ivfpq_range_search against the fp32 restatement (ivfpq_range_oracle.py), bit
for bit -- lims, the bits of values, ids and address -- on every LUT source (staged and in-CTA), code width, metric,
the residual index, sliced and unsliced batches and thresholds from +inf to -inf; and against search itself: strict
matching on integer scores, search(k)'s list as the head of the range result, cell shards, the add / remove / expand
life cycle and the edge cases."""
import ctypes as C

import numpy as np
import pytest
import torch

import ivfpq_range_oracle as PR
from range_oracle import key_order
from oracle import build_state as B, fp32_exact as X, ivfpq_oracle as O
from helpers import make_index
from test_cell_scan_gpu import NQ as CELL_NQ, cell_major_index

pytestmark = pytest.mark.gpu

F32 = np.float32


def g(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _randn(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(F32)


def make_residual_index(st):
    import torchpq_b200 as T
    ix = T.IVFPQIndex(st.d_vector, st.n_subvectors, st.n_cells, initial_size=1, device="cuda:0", pq_use_residual=True)
    return ix.load_state(st)


def state_of(ix):
    """The host copy of an IVFPQIndex's buffers and codebooks (smart probing off)."""
    h = lambda t: t.detach().cpu().numpy().copy()
    return O.IndexState(ix.d_vector, ix.n_subvectors, ix.n_cells, ix.distance, h(ix.vq_codec.codebook),
                        h(ix.pq_codec.codebook), h(ix._storage), h(ix._is_empty), h(ix._cell_start), h(ix._cell_size),
                        h(ix._cell_capacity), h(ix._address2id), ix._max_id, int(ix.n_probe), False, 30.0)


def host(res):
    return tuple(t.cpu().numpy() for t in res)


def assert_csr(got, want):
    lims, v, i, a = host(got) if isinstance(got[0], torch.Tensor) else got
    assert lims.tolist() == want[0].tolist(), "lims differ"
    assert np.array_equal(v.view(np.uint32), want[1].view(np.uint32)), "values differ"
    assert np.array_equal(a, want[3]), "addresses differ"
    assert np.array_equal(i, want[2]), "ids differ"


def thresholds(visited):
    """+inf, about 10 and about 1000 matches per query (the median over the queries of the r-th best visited score),
    -inf."""
    def rth(r):
        best = [np.sort(s)[::-1][min(r, s.size) - 1] for s, _ in visited if s.size]
        return float(np.median(best))
    return [np.inf, rth(10), rth(1000), -np.inf]


def oracle_end_to_end(st, x, residual=False):
    """(x as scanned, probe sims, cells, visited) of the restated coarse stage without smart probing."""
    xu = X.normalize_columns(x) if st.distance == "cosine" else x
    sims, cells = X.coarse_probe(xu, st.vq_codebook, st.n_probe)
    npl = np.full(x.shape[1], st.n_probe, np.int64)
    return xu, sims, cells, npl, PR.visited_scores(st, xu, cells, npl, sims, residual)


def check_end_to_end(st, ix, x, residual=False, ts=None):
    ix.n_probe, ix.use_smart_probing = st.n_probe, False
    xu, sims, cells, npl, visited = oracle_end_to_end(st, x, residual)
    for t in ts or thresholds(visited):
        want = PR.range_search_cells_fp32(st, xu, cells, npl, t, base_sims=sims, residual=residual)
        assert_csr(ix.range_search(g(x), t, return_address=True), want)


def abi_range(ix, x, cells, base_sims, npl, t, max_results=1 << 26):
    """tpq_ivfpq_range_search with the probe lists given, collected as range_search collects."""
    import torchpq_b200 as T
    from torchpq_b200 import _range
    lay = ix.layout()
    x, cells, npl = g(x), g(cells), g(npl)
    base_sims = g(base_sims) if base_sims is not None else None
    nq, n_probe = x.shape[1], cells.shape[1]
    ws_bytes = T._lib.lib.tpq_ivfpq_range_workspace_bytes(C.byref(lay.cindex), nq, n_probe)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=x.device)
    P = T._lib.ptr

    def run(keys, query, cap, total):
        T._lib.check(T._lib.lib.tpq_ivfpq_range_search(
            C.byref(lay.cindex), P(x), P(cells), P(base_sims), P(npl), nq, n_probe, 0, 0.0, t, P(keys), P(query), cap,
            P(total), P(ws), ws_bytes, T._lib.current_stream(x.device)))
    return _range.collect(run, nq, max_results, ix._address2id, True, x.device)


# ----------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
@pytest.mark.parametrize("dsub", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("M", [8, 16, 64, 96, 192])
def test_plain_index(cuda_device, M, dsub, distance):
    """In-CTA LUTs (d/M 1, 2, 4, 8) and staged ones (3), one to three 64-sub-quantizer units, 7 queries (sliced)."""
    st = B.randn_state(M * dsub, M, 16, 3000, seed=M + dsub, distance=distance)
    st.n_probe = 5
    check_end_to_end(st, make_index(st), _randn((M * dsub, 7), M * dsub))


@pytest.mark.parametrize("dsub", [2, 4, 8])
@pytest.mark.parametrize("M", [16, 64])
def test_residual_index(cuda_device, M, dsub):
    """Residual IVFPQ end to end (query half in the CTA at d/M 2, 4; staged at 8), and through the ABI with probe lists
    given: uneven list lengths, a repeated entry, and the caller's base similarities."""
    d = M * dsub
    st = B.randn_state(d, M, 16, 4000, seed=M * dsub)
    st.n_probe = 6
    ix = make_residual_index(st)
    x = _randn((d, 9), d)
    check_end_to_end(st, ix, x, residual=True)
    sims, cells = X.coarse_probe(x, st.vq_codebook, 6)
    sims = (sims + _randn(sims.shape, 1)).astype(F32)                  # the kernel seeds with what it is given
    cells[2, 3] = cells[2, 2]
    npl = np.array([6, 1, 6, 0, 3, 6, 2, 6, 5], np.int64)
    visited = PR.visited_scores(st, x, cells, npl, sims, True)
    for t in thresholds(visited):
        want = PR.range_search_cells_fp32(st, x, cells, npl, t, base_sims=sims, residual=True)
        assert_csr(abi_range(ix, x, cells, sims, npl, t), want)


@pytest.mark.parametrize("nq", [1, 7, 300, 600])
def test_batch_sizes(cuda_device, nq):
    """Sliced batches (fewer than 4 x SMs queries: several CTAs per query) and an unsliced one (600)."""
    st = B.randn_state(64, 16, 32, 20000, seed=nq)
    st.n_probe = 8
    check_end_to_end(st, make_index(st), _randn((64, nq), nq))


def test_plain_index_probe_lists_through_abi(cuda_device):
    st = B.randn_state(32, 8, 12, 3000, seed=8)
    ix = make_index(st)
    x = _randn((32, 6), 8)
    _, cells = X.coarse_probe(x, st.vq_codebook, 5)
    cells[1, 1] = cells[1, 0]                                         # a repeated entry is scanned once
    npl = np.array([5, 5, 0, 5, 2, 9], np.int64)
    for t in thresholds(PR.visited_scores(st, x, cells, npl)):
        assert_csr(abi_range(ix, x, cells, None, npl, t), PR.range_search_cells_fp32(st, x, cells, npl, t))


# ----------------------------------------------------------------------------------------- against search
def test_strict_on_integer_scores(cuda_device):
    """Integer LUTs: every score is exact.  A score equal to t is excluded; at the next float below t it is included."""
    st, queries = B.integer_state(64, 16, 16, 6000, seed=3)
    st.n_probe, st.use_smart_probing = 4, False
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 4, False
    x = queries(5)
    v, _ = ix.search(x.cuda(), k=20)
    t = float(v[0, 9])
    below = float(np.nextafter(F32(t), F32(-np.inf)))
    lims, vals, _ = host(ix.range_search(x.cuda(), t))
    assert (vals[lims[0]:lims[1]] > t).all() and t not in vals[lims[0]:lims[1]]
    lims2, vals2, _ = host(ix.range_search(x.cuda(), below))
    ties = int((vals2[lims2[0]:lims2[1]] == t).sum())
    assert ties >= 1 and lims2[1] - lims2[0] == lims[1] - lims[0] + ties
    for tt in (t, below):
        assert_csr(ix.range_search(x.cuda(), tt, return_address=True), PR.range_search_fp32(st, x.numpy(), tt))


def assert_head_is_search(ix, x, k):
    """range_search(t) with t below every query's k-th value: each query's first k matches are search(k)'s list."""
    v, i, a = ix.search(x, k=k, return_address=True)
    t = float(np.nextafter(F32(v[:, k - 1].min().item()), F32(-np.inf)))
    assert np.isfinite(t)
    lims, rv, ri, ra = ix.range_search(x, t, return_address=True)
    lims = lims.cpu()
    for q in range(x.shape[1]):
        s = int(lims[q])
        assert int(lims[q + 1]) - s >= k
        assert torch.equal(rv[s:s + k].view(torch.int32), v[q].view(torch.int32))
        assert torch.equal(ra[s:s + k], a[q]) and torch.equal(ri[s:s + k], i[q])


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_head_is_search(cuda_device, k):
    st = B.randn_state(64, 16, 64, 40000, seed=k)
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 16, False
    assert_head_is_search(ix, g(_randn((64, 40), k)), k)


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_head_is_search_where_search_runs_cell_major(cuda_device, k):
    st = B.randn_state(128, 64, 8, 16000, seed=13)
    st.n_probe = 4
    ix = cell_major_index(st)
    ix.n_probe, ix.use_smart_probing = 4, False
    assert_head_is_search(ix, g(_randn((128, CELL_NQ), 13)), k)


@pytest.mark.parametrize("residual", [False, True])
def test_head_is_search_with_smart_probing(cuda_device, residual):
    st = B.randn_state(64, 16, 64, 40000, seed=21)
    ix = make_residual_index(st) if residual else make_index(st)
    ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature = 24, True, 1.0
    assert_head_is_search(ix, g(_randn((64, 50), 21)), 100)


def test_shards_union_is_unsharded(cuda_device):
    st = B.randn_state(64, 16, 33, 20000, seed=5)
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 10, False
    x = g(_randn((64, 70), 5))
    xs = x.cpu().numpy()
    t = -np.inf
    for t in (float(ix.search(x, k=200)[0][:, -1].median()), -np.inf):
        whole = host(ix.range_search(x, t, return_address=True))
        parts = []
        for r in range(2):
            ix.set_shard(r, 2)
            parts.append(host(ix.range_search(x, t, return_address=True)))
        ix.set_shard(0, 1)
        for q in range(xs.shape[1]):
            v = np.concatenate([p[1][p[0][q]:p[0][q + 1]] for p in parts])
            a = np.concatenate([p[3][p[0][q]:p[0][q + 1]] for p in parts])
            o = key_order(v, a)
            s, e = whole[0][q], whole[0][q + 1]
            assert np.array_equal(v[o].view(np.uint32), whole[1][s:e].view(np.uint32))
            assert np.array_equal(a[o], whole[3][s:e])


def test_life_cycle_holes_never_match(cuda_device):
    """Holes left by remove, then filled by add, then an add that expands the cells: the oracle on each state."""
    st = B.randn_state(32, 8, 8, 2000, seed=6)
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 4, False
    x = _randn((32, 6), 6)
    rng = np.random.default_rng(6)
    ix.remove(ids=torch.from_numpy(rng.choice(2000, 700, replace=False)).cuda())
    s1 = state_of(ix)
    assert (s1.is_empty[:s1.cell_start[-1] + s1.cell_size[-1]] == 1).sum() >= 700
    check_end_to_end(s1, ix, x, ts=[np.inf, -np.inf, float(np.median(ix.search(g(x), k=50)[0][:, -1].cpu().numpy()))])
    ix.add(g(_randn((32, 400), 7)))                                   # refills holes
    check_end_to_end(state_of(ix), ix, x, ts=[-np.inf, 0.0])
    cap = ix._address2id.shape[0]
    ix.add(g(_randn((32, 3000), 8)))                                  # expands
    assert ix._address2id.shape[0] > cap
    s3 = state_of(ix)
    check_end_to_end(s3, ix, x, ts=[-np.inf])
    lims, v, i, a = host(ix.range_search(g(x), -np.inf, return_address=True))
    assert not s3.is_empty[a].any() and (i >= 0).all()


# ----------------------------------------------------------------------------------------- edge cases
def test_empty_cells_empty_index_and_empty_batch(cuda_device):
    import torchpq_b200 as T
    st = B.randn_state(32, 8, 64, 100, seed=9)                        # most cells empty
    st.n_probe = 8
    ix = make_index(st)
    check_end_to_end(st, ix, _randn((32, 20), 9))
    lims, v, i = ix.range_search(g(_randn((32, 0), 9)), 0.0)
    assert lims.tolist() == [0] and v.numel() == 0 and i.numel() == 0
    for initial_size in (0, 4):                                       # no blocks at all; blocks without a live slot
        e = O.empty_state(32, 8, 16, initial_size, "euclidean", st.vq_codebook[:, :16].copy(), st.pq_codebook)
        ex = T.IVFPQIndex(32, 8, 16, initial_size=1, device="cuda:0").load_state(e)
        ex.n_probe = 4
        lims, v, i, a = ex.range_search(g(_randn((32, 5), 1)), -np.inf, return_address=True)
        assert lims.tolist() == [0] * 6 and v.numel() == i.numel() == a.numel() == 0


def test_chunked_batch(cuda_device):
    """More than 16 384 queries run in chunks (the staged LUT, d/M = 3, is per chunk): equal to the same queries in two
    batches, and to the oracle on rows of both chunks."""
    st = B.randn_state(24, 8, 16, 3000, seed=10)
    st.n_probe, st.use_smart_probing = 3, False
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 3, False
    nq = 16384 + 700
    x = _randn((24, nq), 10)
    t = float(np.median(ix.search(g(x[:, :64]), k=20)[0][:, -1].cpu().numpy()))
    whole = host(ix.range_search(g(x), t, return_address=True))
    halves = [host(ix.range_search(g(x[:, s:e]), t, return_address=True)) for s, e in ((0, 9000), (9000, nq))]
    assert np.array_equal(whole[0], np.concatenate([halves[0][0], halves[1][0][1:] + halves[0][0][-1]]))
    for j in (1, 2, 3):
        assert np.array_equal(whole[j], np.concatenate([halves[0][j], halves[1][j]]))
    rows = np.r_[0:5, 16380:16390, nq - 5:nq]
    want = PR.range_search_fp32(st, x[:, rows], t)
    for n, q in enumerate(rows):
        s, e, ws, we = whole[0][q], whole[0][q + 1], want[0][n], want[0][n + 1]
        assert np.array_equal(whole[1][s:e].view(np.uint32), want[1][ws:we].view(np.uint32))
        assert np.array_equal(whole[3][s:e], want[3][ws:we])


def test_forced_rerun_and_max_results(cuda_device, monkeypatch):
    from torchpq_b200 import _range
    st = B.randn_state(32, 8, 8, 4000, seed=11)
    st.n_probe, st.use_smart_probing = 8, False
    ix = make_index(st)
    ix.n_probe, ix.use_smart_probing = 8, False
    x = _randn((32, 10), 11)
    want = PR.range_search_fp32(st, x, -np.inf)
    nnz = int(want[0][-1])
    assert nnz == 40000
    monkeypatch.setattr(_range, "_FIRST_CAP_MIN", 64)
    monkeypatch.setattr(_range, "_FIRST_CAP_PER_QUERY", 0)           # the first pass holds 64 of 40 000: one re-run
    assert_csr(ix.range_search(g(x), -np.inf, return_address=True), want)
    with pytest.raises(ValueError, match=f"{nnz} results exceed max_results={nnz - 1}"):
        ix.range_search(g(x), -np.inf, max_results=nnz - 1)
    assert_csr(ix.range_search(g(x), -np.inf, return_address=True, max_results=nnz), want)


def test_cap_zero_counts_only(cuda_device):
    import torchpq_b200 as T
    st = B.randn_state(32, 8, 8, 4000, seed=12)
    ix = make_index(st)
    lay = ix.layout()
    x = g(_randn((32, 3), 12))
    ws_bytes = T._lib.lib.tpq_ivfpq_range_workspace_bytes(C.byref(lay.cindex), 3, 8)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    total = torch.full((1,), -5, dtype=torch.long, device="cuda")
    T._lib.check(T._lib.lib.tpq_ivfpq_range_search(C.byref(lay.cindex), T._lib.ptr(x), None, None, None, 3, 8, 0, 30.0,
                                                   -np.inf, None, None, 0, T._lib.ptr(total), T._lib.ptr(ws), ws_bytes,
                                                   T._lib.current_stream(x.device)))
    assert int(total.item()) == 12000


def test_ivfpqr_range_search_raises(cuda_device):
    import torchpq_b200 as T
    rx = T.IVFPQRIndex(32, 8, 8, 8, initial_size=4, device="cuda:0")
    with pytest.raises(NotImplementedError):
        rx.range_search(torch.zeros(32, 2, device="cuda"), 0.0)
