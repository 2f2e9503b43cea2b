"""CPU: tpq_ivfpq_range_search's argument errors (each returns before any launch, so fake device pointers never get
dereferenced), its workspace size, IVFPQRIndex's refusal, and the IVFPQ range oracle against a filter of
fp32_exact.search_cells_fp32 taken with k = every visited item."""
import ctypes as C

import numpy as np
import pytest

import ivfpq_range_oracle as PR
from oracle import build_state as B, fp32_exact as X

FAKE = 256                                                  # never dereferenced: every failing call fails its checks first


def _lib():
    import torchpq_b200 as T
    return T._lib.lib, T._lib


def fake_index(E, *, M=16, d=32, n_cells=8, metric=0, residual=False, part2=True, n_blocks=10, shard_world=1):
    """A tpq_index whose pointers are fake but whose fields pass check_index."""
    ix = E.TpqIndex()
    ix.d_vector, ix.n_subvectors, ix.n_cells, ix.metric = d, M, n_cells, metric
    ix.capacity = 320
    for f in ("vq_codebook", "pq_codebook", "storage", "is_empty", "cell_start", "cell_size", "address2id",
              "codes_scan", "block_valid", "cell_block_start", "pq_codebook_t", "pq_norm_t"):
        setattr(ix, f, FAKE)
    ix.m_pad = (M + 31) // 32 * 32
    ix.shard_rank, ix.shard_world, ix.mean_cell_live = 0, shard_world, 40
    ix.n_blocks = n_blocks
    ix.residual = int(residual)
    ix.part2_scan = FAKE if residual and part2 else 0
    return ix


def test_ivfpq_range_abi_argument_errors():
    L, E = _lib()
    P = C.c_void_p(FAKE)

    def call(ix=None, x=P, cells=None, base_sims=None, npl=None, nq=4, n_probe=2, t=0.5, keys=P, query=P, cap=16,
             total=P, ws_bytes=1 << 40):
        ix = fake_index(E) if ix is None else ix
        return L.tpq_ivfpq_range_search(C.byref(ix), x, cells, base_sims, npl, nq, n_probe, 0, 30.0, t, keys, query,
                                         cap, total, P, ws_bytes, None)

    for m in (E.METRIC["inner"], E.METRIC["manhattan"], 7):
        assert call(fake_index(E, metric=m)) == E.TPQ_ERR_BAD_ARG and "unsupported distance" in E.last_error()
    assert call(t=float("nan")) == E.TPQ_ERR_BAD_ARG and "NaN" in E.last_error()
    assert call(cap=-1) == E.TPQ_ERR_BAD_ARG and "negative" in E.last_error()
    for kw in (dict(total=None), dict(keys=None), dict(query=None)):
        assert call(**kw) == E.TPQ_ERR_BAD_ARG and "null total or match buffer" in E.last_error()
    assert call(x=None) == E.TPQ_ERR_BAD_ARG and "bad query batch" in E.last_error()
    assert call(nq=-1) == E.TPQ_ERR_BAD_ARG
    assert call(cells=P) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert call(n_probe=0) == E.TPQ_ERR_BAD_ARG
    assert call(n_probe=9) == E.TPQ_ERR_BAD_ARG and "n_probe=9 must be in [1, n_cells=8]" in E.last_error()
    assert call(fake_index(E, n_cells=2000), n_probe=1025) == E.TPQ_ERR_UNSUPPORTED
    assert call(cells=P, npl=P, n_probe=9, base_sims=P, ws_bytes=0) == E.TPQ_ERR_WORKSPACE   # given lists: any length
    # residual: part2_scan is required, and base_sims with given probe lists; euclidean only
    assert call(fake_index(E, residual=True, part2=False)) == E.TPQ_ERR_BAD_ARG and "base_sims" in E.last_error()
    assert call(fake_index(E, residual=True), cells=P, npl=P) == E.TPQ_ERR_BAD_ARG and "base_sims" in E.last_error()
    assert call(fake_index(E, residual=True, metric=1)) == E.TPQ_ERR_UNSUPPORTED and "euclidean" in E.last_error()
    assert call(fake_index(E, M=196, d=196)) == E.TPQ_ERR_UNSUPPORTED and "192" in E.last_error()
    assert call(nq=0) == E.TPQ_OK                                            # an empty batch launches nothing
    # cap == 0 counts only: null match arrays are accepted with a total, and the call gets as far as the workspace
    assert call(cap=0, keys=None, query=None, ws_bytes=0) == E.TPQ_ERR_WORKSPACE
    need = L.tpq_ivfpq_range_workspace_bytes(C.byref(fake_index(E)), 4, 2)
    assert need > 0
    assert call(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()
    for t in (float("inf"), float("-inf")):                                  # infinite thresholds pass the checks
        assert call(t=t, ws_bytes=0) == E.TPQ_ERR_WORKSPACE
    assert call(fake_index(E, residual=True), cells=P, npl=P, base_sims=P, ws_bytes=0) == E.TPQ_ERR_WORKSPACE


def test_ivfpq_range_workspace_has_no_keys():
    """The range plan keeps no per-query top-k keys: its workspace is the search's at k = 1 less those keys, and
    it stops growing with nq only through the LUT chunk (staged LUTs) -- never by n_probe * k."""
    L, E = _lib()
    ws = lambda ix, nq, n_probe: L.tpq_ivfpq_range_workspace_bytes(C.byref(ix), nq, n_probe)
    ix = fake_index(E)
    assert ws(ix, 0, 2) == 0 and ws(ix, 4, 0) == 0
    assert L.tpq_ivfpq_range_workspace_bytes(None, 4, 2) == 0
    for nq in (1, 100, 20000):
        assert 0 < ws(ix, nq, 8) <= L.tpq_search_workspace_bytes(C.byref(ix), nq, 8, 1)


def test_ivfpqr_range_search_raises():
    import torchpq_b200 as T
    with pytest.raises(NotImplementedError, match="re-ranked"):
        T.IVFPQRIndex.range_search(object(), None, 0.0)


def _filter_of_search_cells(st, x, cells, npl, t, residual=False, base_sims=None):
    """search_cells_fp32 with k = every visited slot, cut to the scores > float32(t): the CSR the oracle must equal."""
    visited = PR.visited_scores(st, x, cells, npl, base_sims, residual)
    k = max(1, max(a.size for _, a in visited))
    v, a = X.search_cells_fp32(st, x, cells, npl, k, base_sims=base_sims, residual=residual)
    parts = []
    for q in range(x.shape[1]):
        assert (a[q] >= 0).sum() == visited[q][1].size                      # k covers every visited slot
        keep = (a[q] >= 0) & (v[q] > np.float32(t))
        parts.append((v[q][keep], a[q][keep]))
    from range_oracle import csr
    return csr(parts, st.address2id)


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_oracle_is_a_filter_of_search_cells(residual, distance):
    if residual and distance == "cosine":
        pytest.skip("residual IVFPQ is euclidean only")
    st = B.randn_state(32, 8, 6, 400, seed=3, distance=distance)
    rng = np.random.default_rng(4)
    st.is_empty[rng.choice(np.flatnonzero(st.is_empty == 0), 40, replace=False)] = 1     # holes never match
    x = (rng.standard_normal((32, 5))).astype(np.float32)
    if distance == "cosine":
        x = X.normalize_columns(x)
    sims, cells = X.coarse_probe(x, st.vq_codebook, 4)
    npl = np.array([4, 1, 3, 0, 4])                                         # short lists; 0: the plain scan enters one
    cells[4, 1] = cells[4, 0]                                               # a repeated entry is scanned once
    all_s = np.concatenate([s for s, _ in PR.visited_scores(st, x, cells, npl, sims, residual)])
    for t in (np.inf, float(np.quantile(all_s, 0.9)), float(np.median(all_s)), -np.inf):
        got = PR.range_search_cells_fp32(st, x, cells, npl, t, base_sims=sims, residual=residual)
        want = _filter_of_search_cells(st, x, cells, npl, t, residual, sims)
        assert got[0].tolist() == want[0].tolist()
        assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
        assert got[2].tolist() == want[2].tolist() and got[3].tolist() == want[3].tolist()
    lims = PR.range_search_cells_fp32(st, x, cells, npl, -np.inf, base_sims=sims, residual=residual)[0]
    assert lims[-1] == all_s.size and not np.isin(
        PR.range_search_cells_fp32(st, x, cells, npl, -np.inf, base_sims=sims, residual=residual)[3],
        np.flatnonzero(st.is_empty)).any()
    if residual:
        assert lims[4] == lims[3]                                           # the residual scan visits no entry at 0


def test_oracle_end_to_end_probe_is_search_fp32s():
    """range_search_fp32 at -inf visits exactly search_fp32's slots (same coarse probe, normalisation and lists)."""
    st = B.randn_state(32, 8, 6, 400, seed=5, distance="cosine")
    st.n_probe, st.use_smart_probing = 3, False
    x = np.random.default_rng(6).standard_normal((32, 4)).astype(np.float32)
    lims, v, i, a = PR.range_search_fp32(st, x, -np.inf)
    sv, sa, _ = X.search_fp32(st, x, int(np.diff(lims).max()))
    for q in range(4):
        n = lims[q + 1] - lims[q]
        assert a[lims[q]:lims[q + 1]].tolist() == sa[q, :n].tolist()
        assert np.array_equal(v[lims[q]:lims[q + 1]].view(np.uint32), sv[q, :n].view(np.uint32))
