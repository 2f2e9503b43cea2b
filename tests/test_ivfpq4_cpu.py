"""CPU: IVFPQ4Index's constructor checks and checkpoint keys, the 4-bit code packing, the tpq_ivfpq4_search C ABI's
argument errors (which return before any launch) and workspace rule, and the numpy oracle against a float64 ADC brute
force and on designed ties (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ivfpq4_oracle as P4
from oracle import ivfpq_oracle as O


def _index(**kw):
    import torchpq_b200 as T
    return T.IVFPQ4Index(device="cpu", **kw)


def test_constructor_checks():
    ix = _index(d_vector=32, n_subvectors=16, n_cells=4, initial_size=3)
    assert (ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature) == (1, True, 30.0)
    assert ix._storage.dtype == torch.uint8 and ix._storage.shape == (2, 12, 4)
    assert ix.code_size == 8 and ix.d_subvector == 2 and ix.capacity == 12 and not ix.pq_use_residual
    assert _index(d_vector=256, n_subvectors=256).code_size == 128                 # the largest M
    for bad in (dict(d_vector=24, n_subvectors=12), dict(d_vector=20, n_subvectors=4),   # M % 8
                dict(d_vector=36, n_subvectors=8), dict(d_vector=8, n_subvectors=16),     # d % M
                dict(d_vector=16, n_subvectors=8, distance="cosine", pq_use_residual=True),
                dict(d_vector=16, n_subvectors=8, expand_mode="triple"), dict(d_vector=16, n_subvectors=8, n_cells=0)):
        with pytest.raises(AssertionError):
            _index(**bad)
    with pytest.raises(NotImplementedError, match="264 > 256"):
        _index(d_vector=264, n_subvectors=264)
    for name in ("inner", "manhattan", "l2"):
        with pytest.raises(NotImplementedError, match=name):
            _index(d_vector=16, n_subvectors=8, distance=name)
    assert _index(d_vector=16, n_subvectors=8, pq_use_residual=True).pq_use_residual


def test_state_dict_keys_and_shapes():
    import torchpq_b200 as T
    ix = _index(d_vector=16, n_subvectors=8, n_cells=3, initial_size=2)
    ix.vq_codec.set_codebook(torch.zeros(16, 3))
    ix.pq_codec.set_codebook(torch.zeros(8, 2, 16))
    sd = ix.state_dict()
    ref = T.IVFPQIndex(16, 8, 3, initial_size=2, device="cpu")
    ref.vq_codec.set_codebook(torch.zeros(16, 3))
    ref.pq_codec.set_codebook(torch.zeros(8, 2, 256))
    assert set(sd) == set(ref.state_dict())                                       # IVFPQIndex's names
    assert sd["_storage"].shape == (1, 6, 4) and sd["pq_codec.kmeans.centroids"].shape == (8, 2, 16)
    sd["_address2id"] = torch.tensor([4, -1, -1, 9, -1, -1])
    sd["_is_empty"] = torch.tensor([0, 1, 1, 0, 1, 1], dtype=torch.uint8)
    ix2 = _index(d_vector=16, n_subvectors=8, n_cells=3, initial_size=0)
    ix2.load_state_dict(sd)
    assert ix2.max_id == 9 and ix2._has_holes and ix2.capacity == 6 and ix2.n_items == 2
    assert ix2.pq_codec.codebook.shape == (8, 2, 16)
    assert ix2.get_address_by_id(torch.tensor([9, 4, 5])).tolist() == [3, 0, -1]


@pytest.mark.parametrize("M", [8, 16, 24, 64, 256])
def test_packing_round_trip(M):
    from torchpq_b200.ivfpq4_index import _pack_codes, _unpack_codes
    rng = np.random.default_rng(M)
    codes = rng.integers(0, 16, size=(M, 37)).astype(np.uint8)
    packed = _pack_codes(torch.from_numpy(codes))
    assert packed.shape == (M // 2, 37) and np.array_equal(packed.numpy(), P4.pack(codes))
    assert np.array_equal(_unpack_codes(packed).numpy(), codes) and np.array_equal(P4.unpack(P4.pack(codes)), codes)
    # word g of a slot holds sub-quantizers 8 g .. 8 g + 7, code m in bits 4 (m % 8) .. 4 (m % 8) + 3
    words = P4.storage_words(codes).view(np.uint32)[:, :, 0]                       # [M / 8, n]
    for m in range(M):
        assert np.array_equal((words[m // 8] >> (4 * (m % 8))) & 15, codes[m])
    ix = _index(d_vector=M, n_subvectors=M, n_cells=1, initial_size=37)
    ix._storage.copy_(torch.from_numpy(P4.storage_words(codes)))
    assert np.array_equal(ix._codes_at(torch.arange(37)).numpy(), codes)


def _abi():
    import torchpq_b200 as T
    return T._lib.lib, T._lib


def test_abi_argument_errors():
    L, E = _abi()
    fake = C.c_void_p(256)                                  # never dereferenced: every call below fails its checks first

    def search(d=32, M=8, nq=4, metric=0, k=10, n_probe=2, n_cells=8, capacity=100, cells=None, npl=None, base=None,
               part2=None, values=fake, storage=fake, x=fake, ws_bytes=1 << 40):
        return L.tpq_ivfpq4_search(x, d, M, nq, metric, storage, fake, fake, fake, fake, capacity, n_cells, fake, fake,
                                   part2, cells, npl, base, n_probe, 0, 30.0, k, values, fake, None, fake, ws_bytes, None)

    for m in (E.METRIC["inner"], E.METRIC["manhattan"], 7):
        assert search(metric=m) == E.TPQ_ERR_UNSUPPORTED and "euclidean and cosine only" in E.last_error()
    assert search(k=0) == E.TPQ_ERR_BAD_ARG and "k must be in (0, 1024]" in E.last_error()
    assert search(k=1025) == E.TPQ_ERR_UNSUPPORTED
    assert search(M=12, d=24) == E.TPQ_ERR_BAD_ARG and "multiple of 8" in E.last_error()
    assert search(M=0) == E.TPQ_ERR_BAD_ARG
    assert search(M=264, d=264) == E.TPQ_ERR_UNSUPPORTED and "264 > 256" in E.last_error()
    with pytest.raises(NotImplementedError):
        E.check(search(M=264, d=264))
    assert search(d=36) == E.TPQ_ERR_BAD_ARG and "multiple of n_subvectors" in E.last_error()
    assert search(nq=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert search(n_probe=0) == E.TPQ_ERR_BAD_ARG and search(n_cells=0) == E.TPQ_ERR_BAD_ARG
    assert search(capacity=-1) == E.TPQ_ERR_BAD_ARG
    assert search(capacity=1 << 32) == E.TPQ_ERR_BAD_ARG and "32-bit address" in E.last_error()
    assert search(cells=fake) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert search(npl=fake) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert search(n_probe=9) == E.TPQ_ERR_BAD_ARG and "n_probe=9 must be in [1, n_cells=8]" in E.last_error()
    assert search(n_probe=1025, n_cells=2000) == E.TPQ_ERR_UNSUPPORTED
    assert search(part2=fake, metric=1) == E.TPQ_ERR_BAD_ARG and "euclidean" in E.last_error()
    assert search(part2=fake, cells=fake, npl=fake) == E.TPQ_ERR_BAD_ARG and "base_sims" in E.last_error()
    assert search(values=None) == E.TPQ_ERR_BAD_ARG and "null output" in E.last_error()
    assert search(nq=0) == E.TPQ_OK                                               # an empty batch launches nothing
    assert search(nq=0, n_probe=3000, cells=fake, npl=fake) == E.TPQ_OK          # caller lists may be longer than n_cells
    assert search(x=None) == E.TPQ_ERR_BAD_ARG and "null query" in E.last_error()
    assert search(storage=None) == E.TPQ_ERR_BAD_ARG and "null store" in E.last_error()
    assert search(storage=C.c_void_p(258)) == E.TPQ_ERR_BAD_ARG and "aligned" in E.last_error()
    assert search(k=1024, n_probe=30000, n_cells=30000, cells=fake, npl=fake) == E.TPQ_ERR_UNSUPPORTED
    assert "shared memory" in E.last_error()
    need = L.tpq_ivfpq4_workspace_bytes(32, 4, 8, 2, 10)
    assert need > 0
    assert search(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()


def test_workspace_rule():
    """The coarse stage of the whole batch (as tpq_ivfpq_search's), then the slices' keys of one chunk of at most 8192
    queries, each part 256-byte aligned; the slices per query make about eight CTAs per SM (at most 64 slices)."""
    L, _ = _abi()
    ws = L.tpq_ivfpq4_workspace_bytes
    for bad in ((0, 4, 8, 2, 10), (8, 0, 8, 2, 10), (8, 4, 0, 2, 10), (8, 4, 8, 0, 10), (8, 4, 8, 2, 0), (8, 4, 8, 2, 1025)):
        assert ws(*bad) == 0
    up = lambda b: (b + 255) // 256 * 256
    # the library sizes the slices from the current device's SM count, 132 (an H100 SXM) without a device
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count \
        if torch.cuda.is_available() else 132

    def rule(d, nq, C, n_probe, k):
        want = sms * 8
        S = 1 if nq >= want else min(64, -(-want // nq))
        chunk = min(nq, 8192)
        return (up(L.tpq_coarse_workspace_bytes(d, nq, C)) + up(nq * n_probe * 4) + up(nq * n_probe * 8) + up(nq * 8)
                + up(nq * d * 4) + up(S * chunk * k * 8))

    for args in ((32, 1, 16, 4, 10), (128, 100, 4096, 32, 100), (64, 20000, 256, 8, 1024), (16, 1056, 8, 8, 1)):
        assert ws(*args) == rule(*args), args


def _state(rng, d, M, C, n, distance="euclidean", cap_extra=3):
    st = O.empty_state(d, 8, C, 0, distance)                                       # container shape fixed below
    st.n_subvectors = M
    st.vq_codebook = rng.standard_normal((d, C)).astype(np.float32)
    st.pq_codebook = rng.standard_normal((M, d // M, 16)).astype(np.float32)
    cells = rng.integers(0, C, size=n)
    sizes = np.bincount(cells, minlength=C)
    cap = sizes + cap_extra
    st.cell_capacity = cap.astype(np.int64)
    st.cell_start = (np.cumsum(cap) - cap).astype(np.int64)
    st.cell_size = sizes.astype(np.int64)
    total = int(cap.sum())
    codes = rng.integers(0, 16, size=(M, n)).astype(np.uint8)
    st.storage = np.zeros((M // 8, total, 4), np.uint8)
    st.is_empty = np.ones(total, np.uint8)
    st.address2id = -np.ones(total, np.int64)
    order = np.argsort(cells, kind="stable")
    rank = np.empty(n, np.int64)
    rank[order] = np.arange(n) - np.searchsorted(cells[order], cells[order])
    addr = st.cell_start[cells] + rank
    st.storage[:, addr, :] = P4.storage_words(codes)
    st.is_empty[addr] = 0
    st.address2id[addr] = np.arange(n)
    st.max_id = n - 1
    return st, addr, cells


@pytest.mark.parametrize("distance,residual", [("euclidean", False), ("cosine", False), ("euclidean", True)])
def test_oracle_against_float64_adc(distance, residual):
    rng = np.random.default_rng(7)
    d, M, C, n, nq = 32, 16, 6, 400, 5
    st, addr, cells = _state(rng, d, M, C, n, distance)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    all_cells = np.tile(np.arange(C), (nq, 1))
    base = None
    if residual:
        from oracle import fp32_exact as FX
        base = FX.coarse_sims(x, st.vq_codebook)                                   # [nq, C]: each cell's coarse similarity
    v, a = P4.search_cells(st, x, all_cells, np.full(nq, C), n, base_sims=base, residual=residual)
    assert np.array_equal(np.sort(a, axis=1), np.tile(np.sort(addr), (nq, 1)))    # every live item, once
    cell_of = np.searchsorted(st.cell_start, a, side="right") - 1
    for q in range(nq):
        want = P4.adc_float64(st, x[:, q:q + 1], a[q], cells=cell_of[q] if residual else None)[0]
        scale = np.abs(want).max() + 1
        assert np.allclose(v[q], want, rtol=0, atol=1e-4 * scale), np.abs(v[q] - want).max()
        assert np.all(np.diff(v[q]) <= 0)


def test_oracle_ties_go_to_the_lower_address():
    rng = np.random.default_rng(3)
    d, M, C, n = 16, 8, 3, 60
    st, addr, cells = _state(rng, d, M, C, n)
    codes = P4.codes_at(st, addr)
    codes[:] = 5                                                                 # every item the same code: equal scores
    st.storage[:, addr, :] = P4.storage_words(codes)
    x = rng.standard_normal((d, 2)).astype(np.float32)
    v, a = P4.search_cells(st, x, np.tile(np.arange(C), (2, 1)), np.full(2, C), 20)
    assert np.all(v == v[:, :1])
    assert np.array_equal(a, np.tile(np.sort(addr)[:20], (2, 1)))
    # half the items one better code: they come first, each group by address
    better = P4.luts(x[:, :1], st.pq_codebook, "euclidean")[0].argmax(axis=1)     # [M] the best code per sub-quantizer
    codes[:, ::2] = better[:, None]
    st.storage[:, addr, :] = P4.storage_words(codes)
    v, a = P4.search_cells(st, x[:, :1], np.arange(C)[None], np.full(1, C), n)
    k_best = len(addr[::2])
    assert np.array_equal(a[0, :k_best], np.sort(addr[::2])) and np.array_equal(a[0, k_best:], np.sort(addr[1::2]))
    assert v[0, 0] > v[0, -1]
