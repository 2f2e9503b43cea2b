"""GPU: range_search of FlatIndex, IVFFlatIndex and IVFSQIndex bit for bit against the numpy oracle (range_oracle.py),
its strictness at the threshold, its agreement with search and across the indexes, the overflow re-run of the C ABI,
max_results, the add / remove / expand life cycle and the edge cases of the batch."""
import numpy as np
import pytest
import torch

import range_oracle as RO
from oracle import ivfflat_oracle as VO
from oracle import ivfsq_oracle as SO
from oracle.flat_oracle import flat_sims

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _T():
    import torchpq_b200 as T
    return T


def _same(got, want):
    """got: range_search(..., return_address=True) on the GPU; want: the oracle's CSR."""
    lims, v, i, a = (t.cpu().numpy() for t in got)
    assert np.array_equal(lims, want[0]), "lims differ from the oracle"
    assert np.array_equal(v.view(np.uint32), want[1].view(np.uint32)), "values differ from the oracle"
    assert np.array_equal(i, want[2]), "ids differ from the oracle"
    assert np.array_equal(a, want[3]), "addresses differ from the oracle"


def _thresholds(sims):
    """Thresholds giving nothing, about 10 and about 1000 matches per query, and everything."""
    s = np.sort(sims, axis=1)[:, ::-1]
    r = lambda k: float(np.median(s[:, min(k, s.shape[1]) - 1]))
    return [np.inf, r(10), r(1000), -np.inf]


def _flat(base, distance, ids=None):
    fx = _T().FlatIndex(base.shape[0], distance=distance, device=DEV, initial_size=64, expand_step_size=64)
    fx.add(torch.from_numpy(base).to(DEV), None if ids is None else torch.from_numpy(ids).to(DEV))
    return fx


def _rs(ix, x, t, **kw):
    return ix.range_search(torch.from_numpy(x).to(DEV), t, return_address=True, **kw)


# ---------------------------------------------------------------- FlatIndex
@pytest.mark.parametrize("distance", ["euclidean", "cosine", "inner"])
@pytest.mark.parametrize("d", [33, 100, 128])
@pytest.mark.parametrize("nq", [1, 7, 300])
def test_flat_matches_oracle(distance, d, nq):
    rng = np.random.default_rng(d * 7 + nq)
    base = rng.standard_normal((d, 2000)).astype(np.float32)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    ids = rng.permutation(10 ** 6)[:2000].astype(np.int64)
    fx = _flat(base, distance, ids)
    sims = flat_sims(x, base, distance)
    for t in _thresholds(sims):
        _same(_rs(fx, x, t), RO.flat_range_search(x, base, distance, t, ids, sims))


@pytest.mark.parametrize("distance", ["euclidean", "inner"])
def test_strict_threshold_on_integer_scores(distance):
    rng = np.random.default_rng(5)
    base = rng.integers(-3, 4, (16, 2000)).astype(np.float32)              # integer scores, many ties with t
    x = rng.integers(-3, 4, (16, 40)).astype(np.float32)
    fx = _flat(base, distance)
    sims = flat_sims(x, base, distance)
    for t in (float(np.median(sims)), float(np.quantile(sims, 0.99))):
        at = int((sims == np.float32(t)).sum())
        assert at > 0
        got = _rs(fx, x, t)
        _same(got, RO.flat_range_search(x, base, distance, t, sims=sims))
        assert not (got[1] == t).any()                                      # score == t is excluded
        below = float(np.nextafter(np.float32(t), np.float32(-np.inf)))
        lo = _rs(fx, x, below)
        _same(lo, RO.flat_range_search(x, base, distance, below, sims=sims))
        assert int((lo[1] == t).sum()) == at                                # ... and in just above the next float down
        assert int(lo[0][-1]) == int(got[0][-1]) + at


def test_flat_agrees_with_search():
    rng = np.random.default_rng(6)
    base = rng.standard_normal((64, 20000)).astype(np.float32)
    fx = _flat(base, "euclidean")
    x = torch.from_numpy(rng.standard_normal((64, 50)).astype(np.float32)).to(DEV)
    for k in (1, 10, 100, 1024):
        v, i, a = fx.search(x, k=k, return_address=True)
        t = float(v[:, -1].min()) - 1.0                                      # below every query's k-th value
        lims, rv, ri, ra = fx.range_search(x, t, return_address=True)
        for q in range(50):
            s = slice(int(lims[q]), int(lims[q]) + k)
            assert torch.equal(rv[s].view(torch.int32), v[q].view(torch.int32))
            assert torch.equal(ri[s], i[q]) and torch.equal(ra[s], a[q])
        t2 = float(v[:, k // 2].median())                                   # search's results > t2: a prefix
        lims, rv, ri, ra = fx.range_search(x, t2, return_address=True)
        for q in range(50):
            m = int((v[q] > t2).sum())
            assert int(lims[q + 1] - lims[q]) >= m and torch.equal(ra[int(lims[q]):int(lims[q]) + m], a[q, :m])


# ---------------------------------------------------------------- IVFFlatIndex / IVFSQIndex
def _ivf(kind, d, n_cells, n, distance, seed=0, initial_size=16):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((d, n_cells)).astype(np.float32) * 3
    x = centres[:, rng.integers(0, n_cells, n)] + rng.standard_normal((d, n)).astype(np.float32)
    T = _T()
    if kind == "flat":
        ix = T.IVFFlatIndex(d, n_cells, initial_size=initial_size, distance=distance, device=DEV)
    else:
        ix = T.IVFSQIndex(d, n_cells, bits=int(kind[2:]), initial_size=initial_size, distance=distance, device=DEV)
    xt = torch.from_numpy(x).to(DEV)
    ix.train(xt, seed=seed)
    ix.add(xt)
    return ix, x, rng


def _state(ix):
    return SO.state_of(ix) if isinstance(ix, _T().IVFSQIndex) else VO.state_of(ix)


@pytest.mark.parametrize("kind", ["flat", "sq8", "sq16"])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
@pytest.mark.parametrize("d", [33, 100, 128])
@pytest.mark.parametrize("nq", [1, 7, 300])
def test_ivf_matches_oracle(kind, distance, d, nq):
    if kind != "flat" and d == 33:
        d = 32 if kind == "sq8" else 34                                     # SQ codes need d % 4 (8 bits) or d % 2 == 0
    ix, _, rng = _ivf(kind, d, 16, 2000, distance, seed=d + nq)
    ix.n_probe, ix.use_smart_probing = 5, False
    st = _state(ix)
    x = rng.standard_normal((d, nq)).astype(np.float32) * 2
    sims = flat_sims(x, VO.vectors(st), distance)
    for t in _thresholds(sims):
        _same(_rs(ix, x, t), RO.ivfflat_range_search(st, x, t, 5, sims))


def _by_value_then_id(lims, v, i):
    """The ids of each query's matches, ordered by score descending, then id ascending."""
    lims, v, i = lims.cpu().numpy(), v.cpu().numpy(), i.cpu().numpy()
    return np.concatenate([i[s:e][RO.key_order(v[s:e], i[s:e])] for s, e in zip(lims[:-1], lims[1:])])


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_ivfflat_all_cells_equals_flat(distance):
    ix, base, rng = _ivf("flat", 48, 12, 5000, distance, seed=3)
    ix.n_probe, ix.use_smart_probing = 12, False
    fx = _flat(base, distance)
    x = rng.standard_normal((48, 64)).astype(np.float32)
    for t in _thresholds(flat_sims(x, base, distance))[1:]:
        lims, v, i, a = _rs(ix, x, t)
        flims, fv, fi, fa = _rs(fx, x, t)
        assert torch.equal(lims, flims) and torch.equal(v.view(torch.int32), fv.view(torch.int32))
        assert torch.equal(ix._address2id[a], i) and torch.equal(fx._address2id[fa], fi)
        # ids are the add order in both; within a run of equal scores the two address orders may differ
        assert np.array_equal(_by_value_then_id(lims, v, i), _by_value_then_id(flims, fv, fi))


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_ivfsq_equals_ivfflat_on_the_decoded_store(bits, distance):
    ix, _, rng = _ivf(f"sq{bits}", 64, 24, 4000, distance, seed=31)
    ix.remove(ids=torch.arange(0, 4000, 7, device=DEV))
    T = _T()
    fl = T.IVFFlatIndex(64, 24, initial_size=0, distance=distance, device=DEV)
    sd = {k: v for k, v in ix.state_dict().items() if not k.startswith("sq_codec.")}
    sd["_storage"] = ix.decode(ix._codes_at(slice(0, ix.capacity)).contiguous())[:, :, None].contiguous()
    fl.load_state_dict(sd)
    x = torch.from_numpy(rng.standard_normal((64, 120)).astype(np.float32)).to(DEV)
    for ixx in (ix, fl):
        ixx.n_probe, ixx.use_smart_probing = 6, True
    v, _ = fl.search(x, k=100)
    for t in (float(v[:, 9].median()), float(v[:, 99].median()), float("-inf")):
        for u, w in zip(ix.range_search(x, t, return_address=True), fl.range_search(x, t, return_address=True)):
            assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                               w.view(torch.int32) if w.dtype == torch.float32 else w)


@pytest.mark.parametrize("kind", ["flat", "sq8"])
def test_ivf_agrees_with_search_under_smart_probing(kind):
    ix, _, rng = _ivf(kind, 64, 32, 8000, "euclidean", seed=9)
    ix.n_probe, ix.use_smart_probing = 8, True
    x = torch.from_numpy(rng.standard_normal((64, 200)).astype(np.float32) * 2).to(DEV)
    for k in (10, 100):
        v, i, a = ix.search(x, k=k, return_address=True)
        t = float(v[:, -1].min()) - 1.0
        lims, rv, ri, ra = ix.range_search(x, t, return_address=True)
        for q in range(200):
            s = slice(int(lims[q]), int(lims[q]) + k)
            assert torch.equal(rv[s].view(torch.int32), v[q].view(torch.int32))
            assert torch.equal(ri[s], i[q]) and torch.equal(ra[s], a[q])


def test_ivf_life_cycle_holes_never_match():
    ix, base, rng = _ivf("flat", 40, 8, 3000, "euclidean", seed=4, initial_size=4)
    ix.n_probe, ix.use_smart_probing = 8, False
    x = rng.standard_normal((40, 30)).astype(np.float32)
    gone = torch.arange(0, 3000, 3, device=DEV)
    ix.remove(ids=gone)
    more = torch.from_numpy(rng.standard_normal((40, 2500)).astype(np.float32) * 2).to(DEV)
    ix.add(more[:, :700])                                                    # refills holes first
    ix.remove(ids=torch.arange(3000, 3100, device=DEV))
    ix.add(more[:, 700:])                                                    # expands
    st = VO.state_of(ix)
    sims = flat_sims(x, VO.vectors(st), "euclidean")
    for t in (-400.0, -np.inf):
        got = _rs(ix, x, t)
        _same(got, RO.ivfflat_range_search(st, x, t, 8, sims))
        ids = got[2]
        assert not torch.isin(ids, gone).any() and not torch.isin(ids, torch.arange(3000, 3100, device=DEV)).any()
    assert int(got[0][1]) == ix.n_items


def test_edge_cases_and_batch_split():
    T = _T()
    ix, base, rng = _ivf("flat", 32, 8, 2000, "cosine", seed=8)
    ix.n_probe, ix.use_smart_probing = 3, False
    fx = _flat(base, "cosine")
    x = rng.standard_normal((32, 101)).astype(np.float32)
    for index in (ix, fx):
        lims, v, i, a = _rs(index, x[:, :0], 0.5)                          # nq = 0
        assert lims.tolist() == [0] and v.numel() == i.numel() == a.numel() == 0
        whole = _rs(index, x, 0.3)
        halves = [_rs(index, x[:, :50], 0.3), _rs(index, x[:, 50:], 0.3)]
        assert torch.equal(whole[0], torch.cat([halves[0][0], halves[1][0][1:] + halves[0][0][-1]]))
        for j in (1, 2, 3):
            assert torch.equal(whole[j], torch.cat([halves[0][j], halves[1][j]]))
        thr = torch.tensor(0.3, dtype=torch.float64, device=DEV)            # a 0-d tensor, rounded once to fp32
        for u, w in zip(_rs(index, x, thr), whole):
            assert torch.equal(u, w)
        with pytest.raises(ValueError, match="NaN"):
            index.range_search(torch.from_numpy(x).to(DEV), float("nan"))
    empty_ivf = T.IVFFlatIndex(32, 8, initial_size=4, device=DEV)
    empty_ivf.train(torch.from_numpy(base).to(DEV))
    empty_flat = T.FlatIndex(32, device=DEV)
    for index in (empty_ivf, empty_flat):
        lims, v, i = index.range_search(torch.from_numpy(x).to(DEV), float("-inf"))
        assert lims.tolist() == [0] * 102 and v.numel() == i.numel() == 0


# ---------------------------------------------------------------- overflow
def test_abi_overflow_is_counted_and_guarded():
    T = _T()
    L, E = T._lib.lib, T._lib
    rng = np.random.default_rng(11)
    d, n, nq = 24, 1500, 9
    base = rng.standard_normal((d, n)).astype(np.float32)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    fx = _flat(base, "euclidean")
    t = float(np.median(flat_sims(x, base, "euclidean")))
    want = RO.flat_range_search(x, base, "euclidean", t)
    nnz = int(want[0][-1])
    xt = torch.from_numpy(x).to(DEV)
    norms = fx._norm_table()
    ws_bytes = L.tpq_flat_range_workspace_bytes(d, nq, n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    st = T._lib.current_stream(torch.device(DEV))
    guard = 4096
    for cap in (0, 5, 1000, nnz):
        keys = torch.full((cap + guard,), -7, dtype=torch.long, device=DEV)
        query = torch.full((cap + guard,), -7, dtype=torch.int32, device=DEV)
        total = torch.full((1,), -1, dtype=torch.long, device=DEV)
        E.check(L.tpq_flat_range_search(E.ptr(xt), d, nq, E.ptr(fx._storage), fx.capacity, n, E.ptr(norms), 0, t,
                                        E.ptr(keys) if cap else None, E.ptr(query) if cap else None, cap,
                                        E.ptr(total), E.ptr(ws), ws_bytes, st))
        assert int(total) == nnz                                             # the exact total, whatever cap is
        assert (keys[cap:] == -7).all() and (query[cap:] == -7).all()       # nothing past cap
        assert (keys[:cap] != -7).all() and ((query[:cap] >= 0) & (query[:cap] < nq)).all()
    from torchpq_b200 import _range                                          # the re-run with cap = total: the oracle's
    got = _range.collect(lambda k, q, c, tot: E.check(L.tpq_flat_range_search(
        E.ptr(xt), d, nq, E.ptr(fx._storage), fx.capacity, n, E.ptr(norms), 0, t, E.ptr(k), E.ptr(q), c, E.ptr(tot),
        E.ptr(ws), ws_bytes, st)), nq, 1 << 26, fx._address2id, True, torch.device(DEV))
    _same(got, want)


def test_forced_rerun_and_max_results():
    rng = np.random.default_rng(12)
    d, n, nq = 16, 200000, 2
    base = rng.standard_normal((d, n)).astype(np.float32)
    fx = _flat(base, "inner")
    x = rng.standard_normal((d, nq)).astype(np.float32)
    got = _rs(fx, x, -np.inf)                                               # 400 000 matches > the first cap (65 536)
    assert got[0].tolist() == [0, n, 2 * n]
    assert torch.equal(got[3][:n].sort().values, torch.arange(n, device=DEV))
    sims = flat_sims(x[:, :1], base[:, :5000], "inner")
    t = float(np.sort(sims[0])[-40])
    with pytest.raises(ValueError, match="exceed max_results=10"):
        _rs(fx, x, t, max_results=10)
    _same(_rs(fx, x[:, :1], np.inf, max_results=0), RO.flat_range_search(x[:, :1], base, "inner", np.inf))
    ix, _, _ = _ivf("flat", 16, 4, 3000, "euclidean", seed=2)
    ix.n_probe, ix.use_smart_probing = 4, False
    with pytest.raises(ValueError, match="results exceed max_results=100"):
        _rs(ix, x, -np.inf, max_results=100)
    _same(_rs(ix, x, -50.0), RO.ivfflat_range_search(VO.state_of(ix), x, -50.0, 4))   # still usable
