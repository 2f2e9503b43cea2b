"""CPU: the range-search C ABI's argument errors (which return before any launch), its workspace bound, the host-side
CSR assembly and threshold rounding, and the numpy oracle against a brute-force filter (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

import range_oracle as RO
from oracle import ivfflat_oracle as VO
from oracle.flat_oracle import flat_sims

FAKE = C.c_void_p(256)                                      # never dereferenced: every call below fails its checks first


def _lib():
    import torchpq_b200 as T
    return T._lib.lib, T._lib


def test_flat_range_abi_argument_errors():
    L, E = _lib()

    def call(metric=0, t=0.5, nq=4, n=100, keys=FAKE, query=FAKE, cap=16, total=FAKE, x=FAKE, base=FAKE, norms=FAKE,
             ws_bytes=1 << 40, ld=None):
        return L.tpq_flat_range_search(x, 8, nq, base, n if ld is None else ld, n, norms, metric, t, keys, query, cap,
                                       total, FAKE, ws_bytes, None)

    for m in (E.METRIC["manhattan"], 7, -1):
        assert call(metric=m) == E.TPQ_ERR_UNSUPPORTED and "unsupported metric" in E.last_error()
    assert call(t=float("nan")) == E.TPQ_ERR_BAD_ARG and "NaN" in E.last_error()
    assert call(nq=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert call(ld=50) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert call(cap=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert call(n=1 << 32) == E.TPQ_ERR_BAD_ARG and "32-bit address" in E.last_error()
    for kw in (dict(total=None), dict(keys=None), dict(query=None)):
        assert call(**kw) == E.TPQ_ERR_BAD_ARG and "null total or match buffer" in E.last_error()
    assert call(x=None) == E.TPQ_ERR_BAD_ARG and "null query" in E.last_error()
    assert call(base=None) == E.TPQ_ERR_BAD_ARG and "null base or norms" in E.last_error()
    assert call(norms=None) == E.TPQ_ERR_BAD_ARG
    assert call(nq=0) == E.TPQ_OK                                           # an empty batch launches nothing
    # cap == 0 counts only: null match arrays are accepted with a total, and the call gets as far as the workspace
    assert call(cap=0, keys=None, query=None, ws_bytes=0) == E.TPQ_ERR_WORKSPACE
    need = L.tpq_flat_range_workspace_bytes(8, 4, 100)
    assert need > 0
    assert call(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()
    for t in (float("inf"), float("-inf")):                                  # infinite thresholds pass the checks
        assert call(t=t, ws_bytes=0) == E.TPQ_ERR_WORKSPACE
    for inner_norms in (None, FAKE):                                        # INNER reads no norm table
        assert call(metric=E.METRIC["inner"], norms=inner_norms, ws_bytes=0) == E.TPQ_ERR_WORKSPACE


@pytest.mark.parametrize("entry", ["ivfflat", "ivfsq8", "ivfsq16"])
def test_ivf_range_abi_argument_errors(entry):
    L, E = _lib()

    def call(metric=0, t=0.5, nq=4, n_probe=2, n_cells=8, cells=None, npl=None, capacity=100, keys=FAKE, query=FAKE,
             cap=16, total=FAKE, ws_bytes=1 << 40, d=8, bits=8):
        head = (FAKE, d, nq, FAKE, n_cells)
        tail = (capacity, FAKE, FAKE, FAKE, FAKE, metric, cells, npl, n_probe, 0, 30.0, t, keys, query, cap, total, FAKE,
                ws_bytes, None)
        if entry == "ivfflat":
            return L.tpq_ivfflat_range_search(*head, FAKE, *tail)
        b = 16 if entry == "ivfsq16" else bits
        return L.tpq_ivfsq_range_search(*head, FAKE, b, FAKE, FAKE, *tail)

    for m in (E.METRIC["inner"], E.METRIC["manhattan"], 7):
        assert call(metric=m) == E.TPQ_ERR_UNSUPPORTED and "euclidean and cosine only" in E.last_error()
    assert call(t=float("nan")) == E.TPQ_ERR_BAD_ARG and "NaN" in E.last_error()
    assert call(nq=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert call(n_probe=0) == E.TPQ_ERR_BAD_ARG and call(n_cells=0) == E.TPQ_ERR_BAD_ARG
    assert call(capacity=1 << 32) == E.TPQ_ERR_BAD_ARG and "32-bit address" in E.last_error()
    assert call(cells=FAKE) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert call(n_probe=9) == E.TPQ_ERR_BAD_ARG and "n_probe=9 must be in [1, n_cells=8]" in E.last_error()
    assert call(n_probe=1025, n_cells=2000) == E.TPQ_ERR_UNSUPPORTED
    assert call(cap=-1) == E.TPQ_ERR_BAD_ARG and "negative" in E.last_error()
    for kw in (dict(total=None), dict(keys=None), dict(query=None)):
        assert call(**kw) == E.TPQ_ERR_BAD_ARG and "null total or match buffer" in E.last_error()
    assert call(nq=0) == E.TPQ_OK
    assert call(cap=0, keys=None, query=None, ws_bytes=0) == E.TPQ_ERR_WORKSPACE
    need = L.tpq_ivfflat_range_workspace_bytes(8, 4, 8, 2)
    assert need > 0
    assert call(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()
    if entry != "ivfflat":
        assert call(bits=4) == E.TPQ_ERR_UNSUPPORTED or entry == "ivfsq16"
        assert call(d=6) == E.TPQ_ERR_BAD_ARG or entry == "ivfsq16"          # 8 bits: d % 4 == 0
        assert call(d=7) == E.TPQ_ERR_BAD_ARG


def test_workspace_bounds():
    L, _ = _lib()
    ws = L.tpq_ivfflat_range_workspace_bytes
    for bad in ((0, 4, 8, 2), (8, 0, 8, 2), (8, 4, 0, 2), (8, 4, 8, 0)):
        assert ws(*bad) == 0
    # the batch runs in chunks whose gathered pair queries fit 256 MB: past one chunk the workspace stops growing with nq
    for d, C_, n_probe in ((128, 4096, 32), (128, 1024, 64), (33, 64, 64), (100, 16, 1)):
        big = ws(d, 10 ** 6, C_, n_probe)
        assert big == ws(d, 10 ** 5, C_, n_probe) == ws(d, 2 * 10 ** 7, C_, n_probe)
        assert 0 < ws(d, 1, C_, n_probe) <= big < 2 * 1024 ** 3
    fw = L.tpq_flat_range_workspace_bytes
    assert fw(0, 4, 10) == 0 and fw(8, 0, 10) == 0 and fw(8, 4, -1) == 0
    assert fw(8, 4, 10) == fw(8, 4, 10 ** 9) > 0                            # |x|^2 and the normalised queries only


def test_threshold_rounds_once_to_fp32():
    from torchpq_b200 import _range
    t = 0.1                                                                 # not an fp32
    assert _range.threshold_f32(t) == float(np.float32(t))
    assert _range.threshold_f32(torch.tensor(t, dtype=torch.float64)) == float(np.float32(t))
    assert _range.threshold_f32(torch.tensor(2.5)) == 2.5
    assert _range.threshold_f32(float("inf")) == float("inf") and _range.threshold_f32(-np.inf) == float("-inf")
    for bad in (float("nan"), torch.tensor(float("nan")), np.float32("nan")):
        with pytest.raises(ValueError, match="NaN"):
            _range.threshold_f32(bad)
    with pytest.raises(ValueError, match="0-d"):
        _range.threshold_f32(torch.zeros(2))


def _keys(scores, address):
    """The library's match keys as i64: (score_to_ord(score) << 32) | (0xFFFFFFFF - address)."""
    from oracle import fp32_exact as X
    k = (X.score_to_ord(np.asarray(scores, np.float32)).astype(np.uint64) << np.uint64(32)) | \
        (np.uint64(0xFFFFFFFF) - np.asarray(address, np.uint64))
    return k.view(np.int64)


def _fake_run(q, s, a, calls):
    """A range entry point on the CPU that writes the matches (q, s, a) in the given order, at most cap of them."""
    keys = torch.from_numpy(_keys(s, a))
    qs = torch.from_numpy(np.asarray(q, np.int32))

    def run(k_out, q_out, cap, total):
        calls.append(cap)
        m = min(cap, keys.numel())
        k_out[:m], q_out[:m] = keys[:m], qs[:m]
        total[0] = keys.numel()
    return run


def test_csr_assembly_with_empty_queries_and_one_rerun(monkeypatch):
    from torchpq_b200 import _range
    rng = np.random.default_rng(0)
    nq, a2i = 9, torch.arange(1000, 2000)
    # queries 0, 4 and 8 (start, middle, end) match nothing; ties in score are broken by address; -0 ranks below +0
    per_q = {1: ([1.0, 3.0, -2.0, 3.0], [5, 7, 9, 2]), 2: ([0.0, -0.0, np.inf], [1, 2, 3]), 3: ([-np.inf], [4]),
             5: ([2.0] * 5, [50, 10, 40, 20, 30]), 6: ([1e-30, -1e-30], [6, 7]), 7: ([7.0], [0])}
    q, s, a = [], [], []
    for qq, (ss, aa) in per_q.items():
        q += [qq] * len(ss); s += ss; a += aa
    perm = rng.permutation(len(q))                                          # the kernel's order is arbitrary
    q, s, a = np.array(q)[perm], np.array(s, np.float32)[perm], np.array(a)[perm]
    monkeypatch.setattr(_range, "_FIRST_CAP_MIN", 4)
    monkeypatch.setattr(_range, "_FIRST_CAP_PER_QUERY", 0)                 # first cap = 4 < 16 matches: one re-run
    calls = []
    lims, v, i, adr = _range.collect(_fake_run(q, s, a, calls), nq, 1 << 26, a2i, True, torch.device("cpu"))
    assert calls == [4, len(q)]
    want = RO.csr([(np.array(per_q[qq][0], np.float32), np.array(per_q[qq][1])) if qq in per_q
                   else (np.zeros(0, np.float32), np.zeros(0, np.int64)) for qq in range(nq)], a2i.numpy())
    assert lims.tolist() == want[0].tolist() == [0, 0, 4, 7, 8, 8, 13, 15, 16, 16]
    assert np.array_equal(v.numpy().view(np.uint32), want[1].view(np.uint32))
    assert i.tolist() == want[2].tolist() and adr.tolist() == want[3].tolist()
    assert adr[0:4].tolist() == [2, 7, 5, 9] and adr[8:13].tolist() == [10, 20, 30, 40, 50]
    assert np.signbit(v.numpy()[6]) and not np.signbit(v.numpy()[5])        # +0 before -0 (query 2: inf, +0, -0)
    assert v.dtype == torch.float32 and i.dtype == adr.dtype == lims.dtype == torch.int64


def test_csr_no_rerun_and_max_results(monkeypatch):
    from torchpq_b200 import _range
    q, s, a = np.array([2, 0, 2]), np.array([1, 2, 3], np.float32), np.array([3, 4, 5])
    calls = []
    lims, v, i = _range.collect(_fake_run(q, s, a, calls), 3, 1 << 26, torch.arange(10), False, torch.device("cpu"))
    assert calls == [_range.first_cap(3, 1 << 26)] and lims.tolist() == [0, 1, 1, 3] and v.tolist() == [2, 3, 1]
    calls = []
    with pytest.raises(ValueError, match="3 results exceed max_results=2"):
        _range.collect(_fake_run(q, s, a, calls), 3, 2, torch.arange(10), False, torch.device("cpu"))
    assert calls == [2]                                                     # counted once, never re-run
    lims, v, i = _range.collect(_fake_run([], [], [], []), 5, 0, torch.arange(10), False, torch.device("cpu"))
    assert lims.tolist() == [0] * 6 and v.numel() == 0 and i.numel() == 0
    with pytest.raises(ValueError):
        _range.collect(_fake_run([], [], [], []), 5, -1, torch.arange(10), False, torch.device("cpu"))
    assert _range.first_cap(10, 100) == 100 and _range.first_cap(1, 1 << 40) == 1 << 16
    assert _range.first_cap(10 ** 6, 1 << 40) == 1 << 24


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "inner"])
def test_oracle_is_a_filter_of_flat_sims(distance):
    rng = np.random.default_rng(1)
    d, n, nq = 9, 300, 6
    base = rng.standard_normal((d, n)).astype(np.float32)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    sims = flat_sims(x, base, distance)
    for t in (np.inf, float(np.quantile(sims, 0.97)), float(np.median(sims)), -np.inf):
        lims, v, i, a = RO.flat_range_search(x, base, distance, t)
        t32 = np.float32(t)
        for q in range(nq):
            brute = sorted((c for c in range(n) if sims[q, c] > t32), key=lambda c: (-float(sims[q, c]), c))
            assert a[lims[q]:lims[q + 1]].tolist() == brute
            assert np.array_equal(v[lims[q]:lims[q + 1]], sims[q, brute])
        assert np.array_equal(i, a)                                         # the default id map is the identity
    assert RO.flat_range_search(x, base[:, :0], distance, 0.0)[0].tolist() == [0] * (nq + 1)


def test_oracle_strictness_on_integer_scores():
    base = np.array([[1, 2, 3, 4]], np.float32)
    x = np.array([[1]], np.float32)
    lims, v, i, a = RO.flat_range_search(x, base, "inner", 2.0)
    assert a.tolist() == [3, 2] and v.tolist() == [4, 3]                   # the score 2 == t is excluded
    lims, v, i, a = RO.flat_range_search(x, base, "inner", np.nextafter(np.float32(2), np.float32(-np.inf)))
    assert a.tolist() == [3, 2, 1]


def test_ivf_oracle_is_the_flat_oracle_over_the_visited_slots():
    rng = np.random.default_rng(2)
    d, C_, n = 6, 5, 120
    st = VO.empty_state(d, C_, 4, "euclidean", rng.standard_normal((d, C_)).astype(np.float32))
    base = rng.standard_normal((d, n)).astype(np.float32)
    ids, adr = VO.add(st, base, rng.integers(0, C_, n))
    st.is_empty[adr[:7]] = 1                                                # holes never match
    x = rng.standard_normal((d, 4)).astype(np.float32)
    lims, v, i, a = RO.ivfflat_range_search(st, x, -np.inf, C_)             # every cell, every live slot
    assert lims.tolist() == [0, 113, 226, 339, 452]
    assert not np.isin(a, adr[:7]).any() and np.array_equal(i, st.address2id[a])
    flat = RO.flat_range_search(x, VO.vectors(st), "euclidean", -np.inf, st.address2id)
    for q in range(4):
        keep = np.isin(flat[3][flat[0][q]:flat[0][q + 1]], a[lims[q]:lims[q + 1]])
        assert np.array_equal(flat[3][flat[0][q]:flat[0][q + 1]][keep], a[lims[q]:lims[q + 1]])
