"""CPU: the row-wise top-k C ABI's argument errors (they return before any launch), its workspace size, and the numpy
oracle's order on hand-made rows (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from oracle import select_oracle as SO


def _abi():
    import torchpq_b200 as T
    return T._lib.lib, T._lib


def test_topk_abi_argument_errors():
    L, E = _abi()
    fake = C.c_void_p(256)                                  # never dereferenced: every call below fails its checks first

    def topk(x=fake, m=4, n=100, dtype=0, k=10, values=fake, indices=fake, ws=None, ws_bytes=0):
        return L.tpq_topk(x, m, n, dtype, k, values, indices, ws, ws_bytes, None)

    assert topk(k=0) == E.TPQ_ERR_BAD_ARG and "k must be in [1, 1024]" in E.last_error()
    assert topk(k=-3) == E.TPQ_ERR_BAD_ARG
    assert topk(k=1025) == E.TPQ_ERR_UNSUPPORTED and "1025 > 1024" in E.last_error()
    with pytest.raises(NotImplementedError):
        E.check(topk(k=1025))
    assert topk(dtype=2) == E.TPQ_ERR_UNSUPPORTED and "dtype 2" in E.last_error()
    assert topk(dtype=-1) == E.TPQ_ERR_UNSUPPORTED
    assert topk(m=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert topk(n=-1) == E.TPQ_ERR_BAD_ARG
    with pytest.raises(AssertionError):
        E.check(topk(n=-1))
    assert topk(n=1 << 32) == E.TPQ_ERR_UNSUPPORTED and "32-bit column" in E.last_error()
    for kw in ({"x": None}, {"values": None}, {"indices": None}):
        assert topk(**kw) == E.TPQ_ERR_BAD_ARG and "null pointer" in E.last_error()
    # m == 0 returns at once, null pointers included
    assert topk(m=0, x=None, values=None, indices=None) == E.TPQ_OK
    # few long rows need the workspace of the sliced plan
    need = L.tpq_topk_workspace_bytes(1, 10 ** 8, 100, 0)
    assert need > 0
    assert topk(m=1, n=10 ** 8, k=100, ws=fake, ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE
    assert "workspace too small" in E.last_error()
    assert topk(m=1, n=10 ** 8, k=100, ws=None, ws_bytes=need) == E.TPQ_ERR_WORKSPACE


def test_topk_workspace_bytes():
    L, _ = _abi()
    for dtype in (0, 1):
        # one slice per row (short rows, or enough rows to fill the GPU): no workspace
        assert L.tpq_topk_workspace_bytes(3, 1000, 100, dtype) == 0
        assert L.tpq_topk_workspace_bytes(10000, 4096, 32, dtype) == 0
        assert L.tpq_topk_workspace_bytes(70000, 1 << 20, 1024, dtype) == 0
        # sliced rows: m * S * k keys of 8 bytes, S slices of at least max(8192, 8k) columns
        for m, n, k in ((1, 10 ** 8, 1), (1, 10 ** 8, 1024), (100, 10 ** 6, 1024), (1, 1 << 20, 100), (3, 1 << 20, 33)):
            ws = L.tpq_topk_workspace_bytes(m, n, k, dtype)
            assert ws > 0 and ws % (8 * m * k) == 0, (m, n, k, ws)
            S = ws // (8 * m * k)
            assert 2 <= S <= n // max(8192, 8 * k), (m, n, k, S)
        # the workspace is bounded in n: at most about two CTAs per SM
        assert L.tpq_topk_workspace_bytes(1, (1 << 32) - 1, 1024, dtype) == L.tpq_topk_workspace_bytes(1, 10 ** 9, 1024, dtype)
    # invalid arguments: 0
    for args in ((0, 100, 10, 0), (4, 100, 0, 0), (4, 100, 1025, 0), (4, 1 << 32, 10, 0), (4, 100, 10, 5), (4, -1, 10, 0)):
        assert L.tpq_topk_workspace_bytes(*args) == 0, args


def test_oracle_order_on_hand_made_rows():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    neg_nan = np.array([0xFFC00001], dtype=np.uint32).view(np.float32)[0]
    pos_nan = np.array([0x7F800001], dtype=np.uint32).view(np.float32)[0]
    row = np.array([0.0, -0.0, 1.0, neg_nan, -inf, inf, 1.0, pos_nan, -1.0, nan, -0.0, 0.0], dtype=np.float32)
    v, i = SO.topk(row[None], 12)
    # NaNs of both signs first (lower column first), then +inf, the two 1.0s by column, +0s, -0s, -1, -inf
    assert i[0].tolist() == [3, 7, 9, 5, 2, 6, 0, 11, 1, 10, 8, 4]
    assert np.isnan(v[0, :3]).all() and (v[0, :3].view(np.uint32) == 0x7FFFFFFF).all()
    assert SO.same_values(v[0, 3:], np.array([inf, 1, 1, 0, 0, -0.0, -0.0, -1, -inf], dtype=np.float32))
    assert np.signbit(v[0, 6:10]).tolist() == [False, False, True, True]
    # k > n: (-inf, -1) padding
    v, i = SO.topk(np.array([[2.0, -inf]], dtype=np.float32), 4)
    assert i.tolist() == [[0, 1, -1, -1]] and SO.same_values(v, np.array([[2.0, -inf, -inf, -inf]], dtype=np.float32))
    # equal values: columns ascending; fp16 widened exactly
    v, i = SO.topk(np.full((2, 5), 0.5, dtype=np.float16), 3)
    assert i.tolist() == [[0, 1, 2]] * 2 and (v == 0.5).all()
    # the image is the order: a sorted row stays sorted
    x = np.sort(np.random.default_rng(0).standard_normal(1000).astype(np.float32))[::-1].copy()
    v, i = SO.topk(x[None], 1000)
    assert i[0].tolist() == list(range(1000))


def test_topk_is_exported():
    import torchpq_b200 as T
    assert "topk" in T.__all__ and isinstance(T.topk, T.fn.Topk)


def test_topk_asserts_before_any_launch():
    import torch
    import torchpq_b200 as T
    with pytest.raises(AssertionError):
        T.topk(torch.zeros(4, 8), k=2)                      # a CPU tensor
    with pytest.raises(AssertionError):
        T.topk(torch.zeros(4), k=2)                         # 1-D
    with pytest.raises(AssertionError):
        T.topk(torch.zeros(4, 8), k=2, dim=0)
    with pytest.raises(AssertionError):
        T.topk(torch.zeros(8, 4).t(), k=2)                  # not contiguous
    with pytest.raises(AssertionError):
        T.topk(torch.zeros(4, 8), k=0)
