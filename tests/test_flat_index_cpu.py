"""CPU: FlatIndex's container semantics against the numpy oracle, and the flat C ABI's argument errors, which return
before any launch (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.flat_oracle import FlatOracle


def _index(**kw):
    import torchpq_b200 as T
    return T.FlatIndex(device="cpu", **kw)


def _same(ix, o):
    assert ix.n_items == o.n_items and ix.capacity == o.capacity and ix.max_id == o.max_id
    assert np.array_equal(ix._address2id.numpy(), o.address2id)
    assert np.array_equal(ix._storage[:, :, 0].numpy(), o.storage)


@pytest.mark.parametrize("mode", ["double", "step"])
def test_add_and_expand(mode):
    rng = np.random.default_rng(0)
    ix, o = _index(d_vector=5, initial_size=3, expand_step_size=2, expand_mode=mode), \
        FlatOracle(5, initial_size=3, expand_step_size=2, expand_mode=mode)
    caps = []
    for n, with_ids in ((2, False), (4, True), (0, False), (7, False), (1, True)):
        x = rng.standard_normal((5, n)).astype(np.float32)
        ids = rng.integers(0, 1000, n) if with_ids else None
        got_ids, got_adr = ix.add(torch.from_numpy(x), None if ids is None else torch.from_numpy(ids), return_address=True)
        want_ids, want_adr = o.add(x, ids)
        assert np.array_equal(got_ids.numpy(), want_ids) and np.array_equal(got_adr.numpy(), want_adr)
        _same(ix, o)
        caps.append(ix.capacity)
    # the capacity sequence of the reference's expand(): "double" doubles the step before appending it
    assert caps == ([3, 7, 7, 15, 15] if mode == "double" else [3, 7, 7, 13, 15])


def test_ids_continue_across_adds():
    ix = _index(d_vector=2, initial_size=4)
    ix.add(torch.zeros(2, 3))
    ix.add(torch.zeros(2, 2), ids=torch.tensor([10, 4]))
    ids = ix.add(torch.zeros(2, 2))
    assert ids.tolist() == [11, 12] and ix.max_id == 12


@pytest.mark.parametrize("by", ["ids", "address"])
def test_compacting_remove(by):
    rng = np.random.default_rng(1)
    ix, o = _index(d_vector=3, initial_size=16), FlatOracle(3, initial_size=16)
    x = rng.standard_normal((3, 12)).astype(np.float32)
    ix.add(torch.from_numpy(x))
    o.add(x)
    for sel in ([2, 5], [11, 0, 10], [7, 7, 100, -3], [8, 1], []):          # tail hits, duplicates, misses, nothing
        sel = np.array(sel, np.int64)
        if by == "ids":
            got, want = ix.remove(ids=torch.from_numpy(sel)), o.remove(ids=sel)
        else:
            got, want = ix.remove(address=torch.from_numpy(sel)), o.remove(address=sel)
        assert got == want
        _same(ix, o)
        live = o.address2id[:o.n_items]
        assert np.array_equal(ix.get_address_by_id(torch.from_numpy(live)).numpy(), o.get_address_by_id(live))
    with pytest.raises(RuntimeError):
        ix.remove()


def test_maps_data_and_empty():
    rng = np.random.default_rng(2)
    ix, o = _index(d_vector=4, initial_size=8), FlatOracle(4, initial_size=8)
    x = rng.standard_normal((4, 6)).astype(np.float32)
    ids = np.array([9, 3, 7, 1, 0, 12], np.int64)
    ix.add(torch.from_numpy(x), torch.from_numpy(ids))
    o.add(x, ids)
    probe = np.array([12, 0, 5, -1, 3, 99], np.int64)
    assert np.array_equal(ix.get_address_by_id(torch.from_numpy(probe)).numpy(), o.get_address_by_id(probe))
    adr = np.array([0, 5, 6, -2, 8, 3], np.int64)
    assert np.array_equal(ix.get_id_by_address(torch.from_numpy(adr)).numpy(), o.get_id_by_address(adr))
    assert np.array_equal(ix.get_data_by_address(torch.from_numpy(adr)).numpy(), o.get_data_by_address(adr))
    new = rng.standard_normal((4, 6)).astype(np.float32)
    ix.set_data_by_address(torch.from_numpy(adr), torch.from_numpy(new))
    o.set_data_by_address(adr, new)
    _same(ix, o)
    ix.empty()
    o.empty()
    _same(ix, o)
    assert ix._id2address is None


def test_checkpoint_load_rederives_counts():
    # reference-shaped state: _storage [d, capacity, 1], _address2id, _id2address; n_items / max_id are not buffers
    ix = _index(d_vector=3, initial_size=4)
    sd = {"_storage": torch.arange(24, dtype=torch.float32).reshape(3, 8, 1),
          "_address2id": torch.tensor([4, 0, 9, 2, 5, -1, -1, -1]),
          "_id2address": -torch.ones(1, dtype=torch.long)}
    ix.load_state_dict(sd)
    o = FlatOracle.from_state(sd["_storage"].numpy(), sd["_address2id"].numpy())
    _same(ix, o)
    assert ix.n_items == 5 and ix.max_id == 9
    assert ix.get_address_by_id(torch.tensor([9, 5, 3])).tolist() == [2, 4, -1]
    assert ix.add(torch.zeros(3, 1)).tolist() == [10]
    ix2 = _index(d_vector=3)
    ix2.load_state_dict(ix.state_dict())
    o.add(np.zeros((3, 1), np.float32))
    _same(ix2, o)
    bad = dict(sd, _address2id=torch.tensor([4, -1, 9, 2, 5, -1, -1, -1]))
    with pytest.raises(AssertionError):
        _index(d_vector=3).load_state_dict(bad)


@pytest.mark.parametrize("name,canon", [("euclidean", "euclidean"), ("l2", "euclidean"), ("cosine", "cosine"),
                                        ("angular", "cosine"), ("inner", "inner"), ("dot", "inner")])
def test_distance_aliases(name, canon):
    assert _index(d_vector=2, distance=name).distance == canon


@pytest.mark.parametrize("name", ["manhattan", "l1", "hamming"])
def test_unsupported_distances(name):
    with pytest.raises(NotImplementedError):
        _index(d_vector=2, distance=name)


def test_no_cpu_search():
    ix = _index(d_vector=2)
    ix.add(torch.zeros(2, 3))
    with pytest.raises(AssertionError):
        ix.search(torch.zeros(2, 1))


def test_flat_abi_argument_errors():
    import torchpq_b200 as T
    L, E = T._lib.lib, T._lib
    fake = C.c_void_p(256)                                  # never dereferenced: every call below fails its checks first

    def search(k=10, metric=0, n=100, ws_bytes=1 << 30, nq=4):
        return L.tpq_flat_search(fake, 8, nq, fake, 128, n, fake, metric, k, fake, fake, fake, None, fake, ws_bytes, None)

    assert search(k=0) == E.TPQ_ERR_BAD_ARG and "k must be in (0, 1024]" in E.last_error()
    assert search(k=1025) == E.TPQ_ERR_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        E.check(search(k=1025))
    assert search(metric=E.METRIC["manhattan"]) == E.TPQ_ERR_UNSUPPORTED
    assert search(metric=7) == E.TPQ_ERR_UNSUPPORTED
    assert L.tpq_flat_search(fake, 8, 4, fake, 1 << 33, 1 << 32, fake, 0, 10, fake, fake, fake, None, fake, 1 << 30,
                             None) == E.TPQ_ERR_BAD_ARG
    assert search(n=200) == E.TPQ_ERR_BAD_ARG                              # n > ld
    need = L.tpq_flat_workspace_bytes(8, 4, 100, 10)
    assert need > 0 and L.tpq_flat_workspace_bytes(8, 4, 100, 1025) == 0
    assert search(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE
    # the workspace does not grow with n
    assert L.tpq_flat_workspace_bytes(128, 1000, 10 ** 9, 100) == L.tpq_flat_workspace_bytes(128, 1000, 10 ** 7, 100)
    assert L.tpq_flat_norms(fake, 128, 8, 100, E.METRIC["manhattan"], fake, None) == E.TPQ_ERR_BAD_ARG


def test_inner_metric_rejected_by_ivfpq_entry_points():
    import torchpq_b200 as T
    L, E = T._lib.lib, T._lib
    inner = E.METRIC["inner"]
    assert inner == 3
    fake = C.c_void_p(256)                                  # never dereferenced: the metric check fails first
    assert L.tpq_build_lut(fake, fake, 16, 4, 1, inner, fake, None) == E.TPQ_ERR_BAD_ARG
    assert "unsupported metric 3" in E.last_error()
    assert L.tpq_relayout_codebook(fake, 16, 4, inner, fake, fake, None) == E.TPQ_ERR_BAD_ARG
    assert "unsupported metric 3" in E.last_error()
    ix = E.TpqIndex()
    ix.d_vector, ix.n_subvectors, ix.n_cells, ix.metric, ix.capacity = 16, 4, 4, inner, 0
    for call in (lambda: L.tpq_ivfpq_search(C.byref(ix), C.c_void_p(256), 1, 1, 10, 0, 0.0, None, None, None, None,
                                            None, 0, None),
                 lambda: L.tpq_ivfpq_search_cells(C.byref(ix), C.c_void_p(256), C.c_void_p(256), None, C.c_void_p(256),
                                                  1, 1, 10, None, None, None, None, None, 0, None)):
        assert call() == E.TPQ_ERR_BAD_ARG and "unsupported distance" in E.last_error()
