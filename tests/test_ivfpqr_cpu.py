"""CPU: IVFPQRIndex's constructor, checkpoint keys and unsupported paths, tpq_rerank's argument errors (returned
before any launch), and the re-rank oracle against a float64 evaluation of the decoded candidates."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fp32_exact as E
from oracle import ivfpqr_oracle as R

# the buffers of torchpq.index.IVFPQRIndex once trained (CellContainer, BaseContainer and three codecs)
REFERENCE_KEYS = {
    "_address2id", "_storage", "_cell_start", "_cell_size", "_cell_capacity", "_is_empty",
    "vq_codec._is_trained", "vq_codec.kmeans.centroids",
    "pq_codec._is_trained", "pq_codec.kmeans.centroids",
    "pq_rerank_codec._is_trained", "pq_rerank_codec.kmeans.centroids",
}


def cpu_index(**kw):
    import torchpq_b200 as T
    args = dict(d_vector=32, n_subvectors=8, n_subvectors_rerank=16, n_cells=4, initial_size=4, device="cpu")
    args.update(kw)
    return T.IVFPQRIndex(**args)


def test_constructor_defaults_and_asserts():
    import torchpq_b200 as T
    ix = T.IVFPQRIndex(64, device="cpu")
    assert (ix.n_subvectors, ix.n_subvectors_rerank, ix.n_cells, ix.use_residual, ix.distance) == (8, 8, 128, True, "euclidean")
    assert ix.code_size == 16 and ix.k_factor == 4 and ix.n_probe == 1 and ix.use_smart_probing
    assert ix._storage.shape == (4, 128 * 128, 4)
    ix = cpu_index()
    assert ix._storage.shape == (6, 16, 4) and ix.d_subvector == 4 and ix.d_subvector_rerank == 2
    for bad in (dict(n_subvectors=6), dict(d_vector=36), dict(n_subvectors_rerank=6), dict(n_subvectors_rerank=12),
                dict(distance="manhattan"), dict(expand_mode="triple")):
        with pytest.raises(AssertionError):
            cpu_index(**bad)


def test_state_dict_keys_are_the_reference_keys():
    ix = cpu_index()
    for c, shape in ((ix.vq_codec, (32, 4)), (ix.pq_codec, (8, 4, 256)), (ix.pq_rerank_codec, (16, 2, 256))):
        c.set_codebook(torch.zeros(shape))
    assert set(ix.state_dict().keys()) == REFERENCE_KEYS
    ix2 = cpu_index()
    ix2.load_state_dict(ix.state_dict())
    assert ix2.pq_rerank_codec.is_trained and ix2.pq_rerank_codec.codebook.shape == (16, 2, 256)


def test_uncovered_paths_raise():
    import torchpq_b200 as T
    from torchpq_b200 import dist
    ix = cpu_index()
    for call in (ix.drop_reference_layout, lambda: ix.search_cells(None, None), lambda: ix.scan_push(None, 1, None, 1, 0),
                 lambda: T.patch(ix), lambda: dist.distribute(ix)):
        with pytest.raises(NotImplementedError):
            call()


def _rerank(lib, d=32, nq=1, k1=8, M=8, Mr=8, residual=1, metric=0, k=4):
    return lib.tpq_rerank(None, d, nq, None, k1, None, 100, M, Mr, None, None, residual, metric, k, None, None, None,
                          None, None, 0, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(metric=2), "unsupported metric"),
    (dict(metric=3), "unsupported metric"),
    (dict(k=0), "0 < k <= k1 <= 1024"),
    (dict(k=9, k1=8), "0 < k <= k1 <= 1024"),
    (dict(k=4, k1=1025), "0 < k <= k1 <= 1024"),
    (dict(M=6, d=36), "multiples of 4"),
    (dict(Mr=6, d=36), "multiples of 4"),
    (dict(M=8, d=36), "must be a multiple of"),
    (dict(Mr=16, d=40), "must be a multiple of"),
    (dict(nq=-1), "bad sizes"),
    (dict(), "null pointer"),
])
def test_rerank_argument_errors(kw, msg):
    import torchpq_b200 as T
    rc = _rerank(T._lib.lib, **kw)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and msg in T._lib.last_error()


def test_rerank_empty_batch_returns_at_once():
    import torchpq_b200 as T
    assert _rerank(T._lib.lib, nq=0) == T._lib.TPQ_OK
    assert T._lib.lib.tpq_rerank_workspace_bytes(32, 0, 4) == 0
    assert T._lib.lib.tpq_rerank_workspace_bytes(32, 10, 4) >= 10 * 4 * 8 + 32 * 10 * 4


def test_tpq_index_code_size_field():
    import torchpq_b200 as T
    ix = T._lib.TpqIndex()
    assert ix.code_size == 0                                          # zero-filled: "= n_subvectors" for every old caller
    assert T._lib.TpqIndex.code_size.offset == C.sizeof(T._lib.TpqIndex) - 4


def _random_state(d, M, Mr, n, distance, seed):
    rng = np.random.default_rng(seed)
    st = R.empty_state(d, M, Mr, 4, 2, distance, rng.standard_normal((d, 4)).astype(np.float32),
                       rng.standard_normal((M, d // M, 256)).astype(np.float32))
    codes = rng.integers(0, 256, size=(M + Mr, n)).astype(np.uint8)
    R.container_add(st, codes, rng.integers(0, 4, size=n).astype(np.int64))
    pqr = rng.standard_normal((Mr, d // Mr, 256)).astype(np.float32)
    return st, codes, pqr, rng


def test_oracle_wide_container_round_trip():
    st, codes, _, _ = _random_state(16, 4, 8, 50, "euclidean", 0)
    assert st.storage.shape[0] == 3
    a = np.flatnonzero(st.is_empty == 0)
    ids = st.address2id[a]
    assert np.array_equal(R.codes_at(st, a), codes[:, ids])
    assert R.scanned(st).storage.shape == (1, st.capacity, 4)


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
@pytest.mark.parametrize("use_residual", [True, False])
def test_oracle_against_float64(distance, use_residual):
    d, M, Mr, k = 24, 4, 8, 7
    st, codes, pqr, rng = _random_state(d, M, Mr, 60, distance, 1)
    x = rng.standard_normal((d, 3)).astype(np.float32)
    live = np.flatnonzero(st.is_empty == 0)
    cand = np.stack([rng.permutation(live)[:20] for _ in range(3)])
    cand[1, 9:] = -1                                                  # missing candidates are skipped
    cand[2, 3:] = -1                                                  # fewer live candidates than k: (-inf, -1) fill
    v, i, a = R.rerank(x, cand, st, st.pq_codebook, pqr, use_residual, k)
    x64 = x.astype(np.float64)
    if distance == "cosine":
        x64 = x64 / (np.linalg.norm(x64, axis=0) + 1e-9)
    for q in range(3):
        c = cand[q][cand[q] >= 0]
        cw = R.codes_at(st, c)
        y = np.stack([pqr[m, :, cw[M + m]] for m in range(Mr)], 0).transpose(0, 2, 1).reshape(d, -1).astype(np.float64)
        if use_residual:
            y = y + np.stack([st.pq_codebook[m, :, cw[m]] for m in range(M)], 0).transpose(0, 2, 1).reshape(d, -1)
        s = -((x64[:, q:q + 1] - y) ** 2).sum(0) if distance == "euclidean" else (x64[:, q:q + 1] * y).sum(0)
        n = min(k, c.shape[0])
        assert np.allclose(v[q, :n], np.sort(s)[::-1][:n], rtol=1e-5, atol=1e-4)
        s_of = dict(zip(c.tolist(), s))
        assert np.allclose(v[q, :n], [s_of[int(t)] for t in a[q, :n]], rtol=1e-5, atol=1e-4)
        assert np.all(a[q, n:] == -1) and np.all(np.isneginf(v[q, n:]))
        assert np.array_equal(i[q, :n], st.address2id[a[q, :n]])
        assert np.all(np.diff(v[q, :n]) <= 0)


def test_oracle_score_is_a_fma_chain():
    """The euclidean score of one candidate is fmaf(-dif, dif, acc) over e ascending from +0, nothing re-associated."""
    rng = np.random.default_rng(4)
    x = rng.standard_normal(8).astype(np.float32)
    y = rng.standard_normal((8, 1)).astype(np.float32)
    acc = np.float32(0)
    for e in range(8):
        dif = np.float32(x[e] - y[e, 0])
        acc = E.fma32(-dif, dif, acc)
    assert R.scores(x, y, "euclidean")[0] == acc
