"""CPU: IVFFlatIndex's constructor and checkpoint keys, the IVFFlat C ABI's argument errors (which return before any
launch), its workspace bound, and the numpy oracle against FlatOracle (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ivfflat_oracle as VO
from oracle.flat_oracle import FlatOracle


def _index(**kw):
    import torchpq_b200 as T
    return T.IVFFlatIndex(device="cpu", **kw)


@pytest.mark.parametrize("name", ["inner", "dot", "l2", "manhattan", "hamming"])
def test_unsupported_distances(name):
    with pytest.raises(NotImplementedError, match=name):
        _index(d_vector=8, distance=name)


def test_constructor_buffers_and_attributes():
    ix = _index(d_vector=6, n_cells=4, initial_size=3, distance="cosine")
    assert (ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature) == (1, True, 30.0)
    assert ix._storage.dtype == torch.float32 and ix._storage.shape == (6, 12, 1)
    assert ix._is_empty.tolist() == [1] * 12 and ix._address2id.tolist() == [-1] * 12
    assert ix._cell_start.tolist() == [0, 3, 6, 9] and ix._cell_capacity.tolist() == [3] * 4
    assert ix._cell_size.tolist() == [0] * 4 and ix.code_size == 24 and ix.capacity == 12
    assert not ix.vq_codec.is_trained and ix.n_items == 0 and ix.max_id == -1
    assert _index(d_vector=2, n_cells=2).capacity == 2 * 128                  # initial_size defaults to expand_step_size
    for bad in (dict(d_vector=0), dict(d_vector=2, n_cells=0), dict(d_vector=2, expand_mode="triple"),
                dict(d_vector=2, expand_step_size=0), dict(d_vector=2, initial_size=-1)):
        with pytest.raises(AssertionError):
            _index(**bad)


def test_state_dict_keys():
    import torchpq_b200 as T
    sd = _index(d_vector=4, n_cells=2, initial_size=1).state_dict()
    assert set(sd) == {"_address2id", "_storage", "_cell_start", "_cell_size", "_cell_capacity", "_is_empty",
                       "vq_codec._is_trained"}                               # None buffers are not saved
    pq = set(T.IVFPQIndex(8, 4, 2, initial_size=1, device="cpu").state_dict())
    assert set(sd) <= pq                                                     # IVFPQIndex's names


def test_load_state_dict_rederives_max_id():
    ix = _index(d_vector=2, n_cells=2, initial_size=2)
    sd = ix.state_dict()
    sd["_address2id"] = torch.tensor([3, -1, 17, -1])
    sd["_is_empty"] = torch.tensor([0, 1, 0, 1], dtype=torch.uint8)
    ix2 = _index(d_vector=2, n_cells=2, initial_size=0)
    ix2.load_state_dict(sd)
    assert ix2.max_id == 17 and ix2._has_holes and ix2.capacity == 4 and ix2.n_items == 2
    assert ix2.get_address_by_id(torch.tensor([17, 3, 5])).tolist() == [2, 0, -1]


def test_ivfflat_abi_argument_errors():
    import torchpq_b200 as T
    L, E = T._lib.lib, T._lib
    fake = C.c_void_p(256)                                  # never dereferenced: every call below fails its checks first

    def search(k=10, metric=0, nq=4, n_probe=2, cells=None, npl=None, capacity=100, ws_bytes=1 << 40, n_cells=8,
               values=fake):
        return L.tpq_ivfflat_search(fake, 8, nq, fake, n_cells, fake, capacity, fake, fake, fake, fake, metric, cells,
                                    npl, n_probe, 0, 30.0, k, fake, values, fake, None, fake, ws_bytes, None)

    assert search(k=0) == E.TPQ_ERR_BAD_ARG and "k must be in (0, 1024]" in E.last_error()
    assert search(k=1025) == E.TPQ_ERR_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        E.check(search(k=1025))
    for m in (E.METRIC["inner"], E.METRIC["manhattan"], 7):
        assert search(metric=m) == E.TPQ_ERR_UNSUPPORTED and "euclidean and cosine only" in E.last_error()
    assert search(nq=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert search(n_probe=0) == E.TPQ_ERR_BAD_ARG
    assert search(n_cells=0) == E.TPQ_ERR_BAD_ARG
    assert search(capacity=1 << 32) == E.TPQ_ERR_BAD_ARG and "32-bit address" in E.last_error()
    assert search(cells=fake) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert search(npl=fake) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert search(n_probe=9) == E.TPQ_ERR_BAD_ARG and "n_probe=9 must be in [1, n_cells=8]" in E.last_error()
    assert search(n_probe=1025, n_cells=2000) == E.TPQ_ERR_UNSUPPORTED
    assert search(values=None) == E.TPQ_ERR_BAD_ARG and "null output" in E.last_error()
    assert search(nq=0) == E.TPQ_OK                                           # an empty batch launches nothing
    assert search(nq=0, n_probe=3000, cells=fake, npl=fake) == E.TPQ_OK      # caller lists may be longer than n_cells
    need = L.tpq_ivfflat_workspace_bytes(8, 4, 8, 2, 10)
    assert need > 0
    assert search(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()


def test_workspace_bound():
    import torchpq_b200 as T
    ws = T._lib.lib.tpq_ivfflat_workspace_bytes
    for bad in ((0, 4, 8, 2, 10), (8, 0, 8, 2, 10), (8, 4, 0, 2, 10), (8, 4, 8, 0, 10), (8, 4, 8, 2, 0), (8, 4, 8, 2, 1025)):
        assert ws(*bad) == 0
    # the batch is processed in chunks whose keys fit 256 MB: past one chunk the workspace stops growing with nq
    for d, C_, n_probe, k in ((128, 4096, 32, 100), (128, 1024, 64, 10), (33, 64, 64, 1024)):
        big = ws(d, 10 ** 7, C_, n_probe, k)
        assert big == ws(d, 10 ** 6, C_, n_probe, k) == ws(d, 2 * 10 ** 7, C_, n_probe, k)
        assert 0 < ws(d, 1, C_, n_probe, k) <= big
        assert big < 2 * 1024 ** 3
    assert ws(128, 10 ** 5, 4096, 32, 100) >= ws(128, 10 ** 4, 4096, 32, 100)


def _oracle_store(rng, d, C_, n, distance, initial_size=4):
    st = VO.empty_state(d, C_, initial_size, distance, rng.standard_normal((d, C_)).astype(np.float32))
    x = rng.standard_normal((d, n)).astype(np.float32)
    ids, adr = VO.add(st, x, rng.integers(0, C_, n))
    return st, x, ids, adr


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_oracle_placement_stores_the_vectors(distance):
    rng = np.random.default_rng(0)
    st, x, ids, adr = _oracle_store(rng, 5, 6, 90, distance)
    assert np.array_equal(VO.vectors(st)[:, adr], x) and np.array_equal(st.address2id[adr], ids)
    assert st.cell_size.sum() == 90 and (st.is_empty == 0).sum() == 90


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_oracle_with_every_cell_probed_is_flat_oracle(distance):
    rng = np.random.default_rng(1)
    d, C_, n, k = 7, 8, 200, 15
    st, x, ids, adr = _oracle_store(rng, d, C_, n, distance)
    o = FlatOracle(d, distance=distance)
    o.add(x, ids)
    xq = rng.standard_normal((d, 9)).astype(np.float32)
    v, i, a = VO.search(st, xq, k, C_)
    fv, fi, _ = o.search(xq, k)
    assert np.array_equal(v.view(np.uint32), fv.view(np.uint32))
    assert np.array_equal(i, fi)                                             # randn scores: no ties
    assert np.array_equal(st.address2id[a], i)


def test_oracle_visiting_rule():
    st = VO.empty_state(2, 4, 3)
    VO.add(st, np.arange(14, dtype=np.float32).reshape(2, 7), [0, 0, 1, 2, 2, 2, 3])
    st.is_empty[st.cell_start[2] + 1] = 1                                   # a hole in cell 2
    live = {c: list(range(st.cell_start[c], st.cell_start[c] + st.cell_size[c])) for c in range(4)}
    live[2].remove(st.cell_start[2] + 1)
    row = np.array([1, 1, -3, 0, 9, 2, 1], np.int64)
    assert VO.visited(st, row, 7, 7).tolist() == live[1] + live[0] + live[2] + live[1]
    assert VO.visited(st, row, 1, 7).tolist() == live[1]
    assert VO.visited(st, row, 0, 7).tolist() == live[1]                    # at least the first entry
    assert VO.visited(st, row, np.iinfo(np.int64).min, 7).tolist() == live[1]
    assert VO.visited(st, row, 8, 7).tolist() == VO.visited(st, row, 7, 7).tolist()
    assert VO.visited(st, np.array([-1, 5], np.int64), 2, 2).tolist() == []
