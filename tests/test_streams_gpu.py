"""GPU: the stream contract of include/tpq_b200.h and INTEGRATION.md section 5, for every entry point.

  a. search / search_cells of every index, every fn operator, SQCodec and the four range entry points capture into a
     CUDA graph once the index is warm (a host sync, an allocation by the library or a launch off the caller's stream
     fails the capture), and two replays on new inputs equal the same calls made eagerly, bit for bit;
  b. the synchronising paths (add with expansion and holes, remove, train, the scan layout's build, range_search,
     KMeans.fit) run on a side stream while a sleep occupies the legacy default stream: the host gets its answer
     before the sleep ends, and the results equal the same calls made without the sleep;
  c. a cache built on one stream (the norm tables, the scan layout) and read by a search on another stream is waited
     for: the search cannot finish before the build, and returns the oracle's values;
  d. one index searched from four streams at once returns, per stream, what the serial searches return.
Every state is small and seeded; every sleep is calibrated once and runs once per case."""
import time

import numpy as np
import pytest
import torch

from oracle import build_state as B, flat_oracle as FO, ivfflat_oracle as VO, ivfpq_oracle as O, \
    ivfsq_oracle as QO, kmeans_oracle as KO, select_oracle as SO
from helpers import make_index
from test_cell_scan_gpu import NQ as CELL_NQ, cell_major_index
import test_ivfpqr_gpu as RQ

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SLEEP_S = 0.3


def _T():
    import torchpq_b200 as T
    return T


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(t):
    """A tensor's bit pattern, so that NaN == NaN and -0 != +0."""
    t = t.detach()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    if t.dtype == torch.float16:
        return t.view(torch.int16)
    return t


def assert_same(got, want):
    if isinstance(got, torch.Tensor):
        got, want = (got,), (want,)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert torch.equal(_bits(g).cpu(), _bits(w).cpu())


def assert_oracle(got, want):
    """got: (values, ids[, address]) CUDA tensors, want: the oracle's numpy arrays."""
    for g, w in zip(got, want):
        g = g.cpu().numpy()
        assert g.dtype == w.dtype and np.array_equal(g.view(np.int32) if g.dtype == np.float32 else g,
                                                     w.view(np.int32) if w.dtype == np.float32 else w)


@pytest.fixture(scope="module")
def sleep_cycles(cuda_device):
    """torch.cuda._sleep cycles for SLEEP_S, measured once with events."""
    torch.cuda._sleep(1000)
    torch.cuda.synchronize()
    n = 20_000_000
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(n)
    b.record()
    b.synchronize()
    return int(n * SLEEP_S * 1000 / a.elapsed_time(b))


# ============================================================================ a. capture and replay

def capture_replay(call, inputs, fresh):
    """Warm `call` on a side stream S, capture it on S, then for each set in `fresh` copy it into `inputs` (the tensors
    the graph reads), replay, and require the graph's outputs to equal `call()` run eagerly on those inputs.  -> the
    outputs of the last replay."""
    S = torch.cuda.Stream()
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        call()
    S.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=S):
        out = call()
    for new in fresh:
        for t, v in zip(inputs, new):
            t.copy_(v)
        g.replay()
        S.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(S):
            want = call()
        torch.cuda.synchronize()
        assert_same(out, want)
    return out


def _randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.fixture(scope="module")
def flat_base(cuda_device):
    return np.random.default_rng(11).standard_normal((48, 5000)).astype(np.float32)


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "inner"])
@pytest.mark.parametrize("k", [1, 100, 1024])
def test_capture_flat_search(flat_base, distance, k):
    T = _T()
    ix = T.FlatIndex(48, distance=distance, device=DEV)
    ix.add(_t(flat_base))
    x = _randn(48, 64, seed=k)
    fresh = [(_randn(48, 64, seed=100 + s),) for s in range(2)]
    out = capture_replay(lambda: ix.search(x, k=k, return_address=True), [x], fresh)
    if distance == "euclidean" and k == 100:
        o = FO.FlatOracle(48)
        o.add(flat_base)
        assert_oracle(out, o.search(fresh[-1][0].cpu().numpy(), k))


def _ivf_data(d, n_cells, n, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((d, n_cells)).astype(np.float32) * 3
    return centres[:, rng.integers(0, n_cells, n)] + rng.standard_normal((d, n)).astype(np.float32)


@pytest.fixture(scope="module")
def ivfflat(cuda_device):
    base = _ivf_data(32, 16, 4000, 5)
    ix = _T().IVFFlatIndex(32, 16, initial_size=8, device=DEV)
    ix.train(_t(base))
    ix.add(_t(base))
    ix.n_probe, ix.use_smart_probing = 4, False
    return ix


def test_capture_ivfflat_search(ivfflat):
    x = _randn(32, 40, seed=3)
    fresh = [(_randn(32, 40, seed=30 + s),) for s in range(2)]
    out = capture_replay(lambda: ivfflat.search(x, k=20, return_address=True), [x], fresh)
    assert_oracle(out, VO.search(VO.state_of(ivfflat), fresh[-1][0].cpu().numpy(), 20, 4))


def test_capture_ivfflat_search_cells(ivfflat):
    x = _randn(32, 40, seed=4)
    g = torch.Generator().manual_seed(4)
    cells = torch.randint(-1, 17, (40, 5), generator=g).to(DEV)
    npl = torch.randint(0, 6, (40,), generator=g).to(DEV)
    fresh = [(_randn(32, 40, seed=40 + s), torch.randint(-1, 17, (40, 5), generator=g), torch.randint(0, 6, (40,), generator=g))
             for s in range(2)]
    out = capture_replay(lambda: ivfflat.search_cells(x, cells, n_probe_list=npl, k=16, return_address=True),
                         [x, cells, npl], fresh)
    want = VO.search_cells(VO.state_of(ivfflat), fresh[-1][0].cpu().numpy(), fresh[-1][1].numpy(), fresh[-1][2].numpy(), 16)
    assert_oracle(out, want)


@pytest.mark.parametrize("bits", [8, 16])
def test_capture_ivfsq_search(bits):
    base = _ivf_data(32, 16, 4000, 6)
    ix = _T().IVFSQIndex(32, 16, bits=bits, initial_size=8, device=DEV)
    ix.train(_t(base))
    ix.add(_t(base))
    ix.n_probe, ix.use_smart_probing = 4, False
    x = _randn(32, 40, seed=5)
    fresh = [(_randn(32, 40, seed=50 + s),) for s in range(2)]
    out = capture_replay(lambda: ix.search(x, k=20, return_address=True), [x], fresh)
    assert_oracle(out, QO.search(QO.state_of(ix), fresh[-1][0].cpu().numpy(), 20, 4))


@pytest.mark.parametrize("bits", [8, 16])
def test_capture_sq_codec(bits):
    codec = _T().codec.SQCodec(bits=bits)
    codec.train(_randn(24, 3000, seed=6) * 4)
    x = _randn(24, 1000, seed=7) * 4
    fresh = [(_randn(24, 1000, seed=70 + s) * 4,) for s in range(2)]
    enc = capture_replay(lambda: codec.encode(x), [x], fresh)
    lo, rg = (codec.lower.cpu().numpy(), codec.range.cpu().numpy()) if bits == 8 else (None, None)
    assert np.array_equal(enc.cpu().numpy(), QO.encode(fresh[-1][0].cpu().numpy(), bits, lo, rg))
    code = enc.clone()
    dec = capture_replay(lambda: codec.decode(code), [code], [(codec.encode(v.to(DEV)),) for (v,) in fresh])
    assert_same(dec, _t(QO.decode(code.cpu().numpy(), bits, lo, rg)))


@pytest.fixture(scope="module")
def pq_small(cuda_device):
    """An integer-valued IVFPQ state whose cells are small: every batch takes the query-major kernel."""
    st, queries = B.integer_state(64, 16, 32, 6000, seed=3)
    st.n_probe, st.use_smart_probing = 6, True
    return st, queries, make_index(st)


@pytest.mark.parametrize("nq", [32, 600])                              # sliced, unsliced
def test_capture_ivfpq_search(pq_small, nq):
    st, queries, ix = pq_small
    x = queries(nq, 1).to(DEV)
    fresh = [(queries(nq, 10 + s),) for s in range(2)]
    out = capture_replay(lambda: ix.search(x, k=50, return_address=True, return_keys=True), [x], fresh)
    ov, oi, oa = O.search(st, fresh[-1][0], k=50, return_address=True)
    assert_oracle(out[:3], (ov, oi, oa))


def test_capture_ivfpq_search_cells(pq_small):
    st, queries, ix = pq_small
    g = torch.Generator().manual_seed(8)
    x = queries(64, 2).to(DEV)
    cells = torch.randint(-1, 33, (64, 6), generator=g).to(DEV)
    npl = torch.randint(0, 7, (64,), generator=g).to(DEV)
    fresh = [(queries(64, 20 + s), torch.randint(-1, 33, (64, 6), generator=g), torch.randint(0, 7, (64,), generator=g))
             for s in range(2)]
    capture_replay(lambda: ix.search_cells(x, cells, n_probe_list=npl, k=30, return_address=True), [x, cells, npl], fresh)


@pytest.fixture(scope="module")
def pq_cell_major(cuda_device):
    st, queries = B.integer_state(128, 64, 8, 16000, seed=22)
    st.n_probe, st.use_smart_probing = 4, False
    return st, queries, cell_major_index(st)


def test_capture_ivfpq_cell_major(pq_cell_major):
    st, queries, ix = pq_cell_major
    x = queries(CELL_NQ, 1).to(DEV)
    fresh = [(queries(CELL_NQ, 30 + s),) for s in range(2)]
    out = capture_replay(lambda: ix.search(x, k=100, return_address=True), [x], fresh)
    ov, oi, oa = O.search(st, fresh[-1][0], k=100, return_address=True)
    assert_oracle(out, (ov, oi, oa))


def test_capture_ivfpq_cell_major_overflow_rerun(cuda_device):
    """test_cell_scan_gpu.test_overflow_reruns_query_major's batch: its overflowing queries are scanned again by the
    query-major kernel, inside the same captured launch sequence."""
    st, queries = B.integer_state(128, 64, 8, 24000, seed=13)
    cell0 = np.arange(st.cell_start[0], st.cell_start[0] + st.cell_size[0])
    st.is_empty[cell0[10:]] = 1
    ix = cell_major_index(st)
    g = torch.Generator().manual_seed(4)

    def lists():
        cells = torch.stack([torch.randperm(7, generator=g) + 1 for _ in range(CELL_NQ)])
        return torch.cat([torch.zeros(CELL_NQ, 1, dtype=torch.long), cells], 1)
    npl = torch.full((CELL_NQ,), 8, dtype=torch.long, device=DEV)
    npl[::2] = 2
    x, cells = queries(CELL_NQ, 1).to(DEV), lists().to(DEV)
    fresh = [(queries(CELL_NQ, 40 + s), lists()) for s in range(2)]
    capture_replay(lambda: ix.search_cells(x, cells, n_probe_list=npl, k=100, return_address=True), [x, cells], fresh)


def test_capture_ivfpq_residual(cuda_device):
    st = B.build_state_residual(torch.randn(32, 6000, generator=torch.Generator().manual_seed(9)), 8, 16, vq_iters=3,
                                pq_iters=2)
    st.n_probe, st.use_smart_probing = 4, False
    ix = _T().IVFPQIndex(32, 8, 16, initial_size=1, device=DEV, pq_use_residual=True).load_state(st)
    ix.n_probe, ix.use_smart_probing = 4, False
    x = _randn(32, 48, seed=9)
    fresh = [(_randn(32, 48, seed=90 + s),) for s in range(2)]
    capture_replay(lambda: ix.search(x, k=20, return_address=True), [x], fresh)
    vq = ix.vq_codec.codebook
    cells = _T().fn.coarse_probe(x, vq, 4, False)[1]
    base = torch.zeros(48, 4, device=DEV)
    fresh = [(_randn(32, 48, seed=95 + s), _T().fn.coarse_probe(_randn(32, 48, seed=95 + s), vq, 4, False)[1],
              _T().fn.coarse_probe(_randn(32, 48, seed=95 + s), vq, 4, False)[0]) for s in range(2)]
    capture_replay(lambda: ix.search_cells(x, cells, base_sims=base, k=20, return_address=True), [x, cells, base], fresh)


def test_capture_ivfpqr_search(cuda_device):
    ix, queries = RQ.make_index(32, 8, 16, 8, 3000, seed=2, kind="int", n_probe=4)
    x = queries(24, 1)
    fresh = [(queries(24, 10 + s),) for s in range(2)]
    out = capture_replay(lambda: ix.search(x, k=10, return_address=True), [x], fresh)
    assert_oracle(out, RQ.oracle_search(ix, fresh[-1][0], 10)[:3])


@pytest.mark.parametrize("family", ["flat", "ivfflat", "ivfsq", "ivfpq"])
def test_capture_cache_built_on_another_stream(family, flat_base, ivfflat, pq_small):
    """The cache (norm table or scan layout) is built on the default stream and the search captured on a side stream:
    the capture must skip the wait on the cache's event (a capture rejects a wait on an event recorded outside it;
    the device is synchronised when the capture begins), and the replay returns the oracle's values."""
    T = _T()
    if family == "flat":
        ix = T.FlatIndex(48, device=DEV)
        ix.add(_t(flat_base))
        x = _randn(48, 64, seed=1)
        fresh = _randn(48, 64, seed=2)
        oracle = FO.FlatOracle(48)
        oracle.add(flat_base)
        want = lambda: oracle.search(x.cpu().numpy(), 10)
    elif family in ("ivfflat", "ivfsq"):
        ix = ivfflat
        if family == "ivfsq":
            base = _ivf_data(32, 16, 4000, 6)
            ix = T.IVFSQIndex(32, 16, bits=8, initial_size=8, device=DEV)
            ix.train(_t(base))
            ix.add(_t(base))
            ix.n_probe, ix.use_smart_probing = 4, False
        x, fresh = _randn(32, 64, seed=1), _randn(32, 64, seed=2)
        st = (VO if family == "ivfflat" else QO).state_of(ix)
        want = lambda: VO.search(st, x.cpu().numpy(), 10, 4)
    else:
        st, queries, ix = pq_small
        x, fresh = queries(64, 5).to(DEV), queries(64, 6)
        want = lambda: O.search(st, x.cpu(), k=10, return_address=True)
    if family == "ivfpq":
        ix._layout = None
    else:
        ix._norms = None
    ix.search(x, k=10)                                                   # builds the cache on the default stream
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=S):
        out = ix.search(x, k=10, return_address=True)
    x.copy_(fresh)
    g.replay()
    torch.cuda.synchronize()
    assert_oracle(out, want())


def test_capture_refuses_to_build_a_cache(flat_base):
    """A first search inside a capture would build the norm table in the graph's pool, filled only on replay: it raises
    instead, keeps no cache, and the next eager search builds a complete one."""
    ix = _T().FlatIndex(48, device=DEV)
    ix.add(_t(flat_base))
    x = _randn(48, 16, seed=3)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(AssertionError, match="run the call once eagerly"):
        with torch.cuda.graph(g, stream=torch.cuda.Stream()):
            ix.search(x, k=10)
    del g
    assert ix._norms is None
    oracle = FO.FlatOracle(48)
    oracle.add(flat_base)
    assert_oracle(ix.search(x, k=10, return_address=True), oracle.search(x.cpu().numpy(), 10))


# -------------------------------------------------------------------- range entry points, through the C ABI
def _range_pairs(keys, query, total):
    n = int(total.item())
    pairs = torch.stack([query[:n].long(), keys[:n]], 1).cpu().numpy()
    return n, pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))]


def capture_range(ix, x, t, fresh, monkeypatch):
    """ix.range_search's own launch (its `run` closure), into buffers of `cap` entries: the host half that reads the
    total back (_range.collect) is replaced by one launch, so that the launch alone is captured."""
    from torchpq_b200 import _range
    cap = 1 << 16
    bufs = (torch.empty(cap, dtype=torch.long, device=DEV), torch.empty(cap, dtype=torch.int32, device=DEV),
            torch.empty(1, dtype=torch.long, device=DEV))
    monkeypatch.setattr(_range, "collect", lambda run, *a: run(bufs[0], bufs[1], cap, bufs[2]))
    S = torch.cuda.Stream()
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        ix.range_search(x, t)
    S.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=S):
        ix.range_search(x, t)
    for (new,) in fresh:
        x.copy_(new)
        g.replay()
        torch.cuda.synchronize()
        got = _range_pairs(*bufs)
        with torch.cuda.stream(S):
            ix.range_search(x, t)
        torch.cuda.synchronize()
        want = _range_pairs(*bufs)
        assert 0 < got[0] <= cap and got[0] == want[0] and np.array_equal(got[1], want[1])


def test_capture_range_search_entry_points(flat_base, ivfflat, pq_small, monkeypatch):
    T = _T()
    fx = T.FlatIndex(48, device=DEV)
    fx.add(_t(flat_base))
    x = _randn(48, 16, seed=12)
    t = float(fx.search(x, k=20)[0][:, -1].median())
    capture_range(fx, x, t, [(_randn(48, 16, seed=120 + s),) for s in range(2)], monkeypatch)

    x = _randn(32, 16, seed=13)
    t = float(ivfflat.search(x, k=20)[0][:, -1].median())
    capture_range(ivfflat, x, t, [(_randn(32, 16, seed=130 + s),) for s in range(2)], monkeypatch)

    base = _ivf_data(32, 16, 4000, 6)
    sx = T.IVFSQIndex(32, 16, bits=8, initial_size=8, device=DEV)
    sx.train(_t(base))
    sx.add(_t(base))
    sx.n_probe, sx.use_smart_probing = 4, False
    t = float(sx.search(x, k=20)[0][:, -1].median())
    capture_range(sx, x, t, [(_randn(32, 16, seed=140 + s),) for s in range(2)], monkeypatch)

    st, queries, px = pq_small
    xq = queries(16, 3).to(DEV)
    t = float(px.search(xq, k=20)[0][:, -1].median())
    capture_range(px, xq, t, [(queries(16, 150 + s),) for s in range(2)], monkeypatch)


# -------------------------------------------------------------------- fn operators
TOPK_PLANS = [(16 * 132, 64, 8), (3, 4096, 100), (1, 1 << 20, 1000)]  # rows, slices, slices + parts


@pytest.mark.parametrize("m,n,k", TOPK_PLANS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_capture_topk(m, n, k, dtype):
    x = _randn(m, n, seed=m).to(dtype)
    fresh = [(_randn(m, n, seed=m + 1 + s).to(dtype),) for s in range(2)]
    v, i = capture_replay(lambda: _T().fn.Topk()(x, k=k), [x], fresh)
    ov, oi = SO.topk(fresh[-1][0].cpu().numpy(), k)
    assert SO.same_values(v.float().cpu().numpy(), ov) and np.array_equal(i.cpu().numpy(), oi)


def test_capture_probe_lut_normalize_ivfpq_topk(pq_small):
    st, queries, _ = pq_small
    fn = _T().fn
    vq, pq = _t(st.vq_codebook), _t(st.pq_codebook)
    x = queries(40, 1).to(DEV)
    fresh = [(queries(40, 60 + s),) for s in range(2)]
    capture_replay(lambda: fn.coarse_probe(x, vq, 6, True, 30.0), [x], fresh)
    capture_replay(lambda: fn.precompute_adc(x, pq, "euclidean"), [x], fresh)
    capture_replay(lambda: fn.normalize(x), [x], fresh)

    _, cells, npl = fn.coarse_probe(x, vq, 6, False)
    lut = fn.precompute_adc(x, pq)
    cs, cz = _t(st.cell_start)[cells], _t(st.cell_size)[cells]
    data, empty = _t(st.storage), _t(st.is_empty)
    topk = fn.IVFPQTopk(16)

    def inputs(seed):
        xs = queries(40, seed).to(DEV)
        c = fn.coarse_probe(xs, vq, 6, False)[1]
        return fn.precompute_adc(xs, pq), _t(st.cell_start)[c], _t(st.cell_size)[c]
    capture_replay(lambda: topk.topk(data, lut, cs, cz, empty, npl, k=40), [lut, cs, cz], [inputs(70), inputs(71)])


@pytest.mark.parametrize("kernel,l,d,n,k", [("exact", 2, 12, 1000, 300), ("assign_tc", 2, 64, 1024, 256),
                                            ("assign_wide", 1, 128, 2000, 4096)])
def test_capture_kmeans_assign_and_max_sim(kernel, l, d, n, k):
    """Integer data in [-4, 4]: every TF32 product and sum is exact, so each kernel equals the exact one, which equals
    kmeans_oracle.max_sim (checked here where the oracle is quick)."""
    fn = _T().fn
    g = torch.Generator().manual_seed(k)
    data = torch.randint(-4, 5, (l, d, n), generator=g).float().to(DEV)
    cent = torch.randint(-4, 5, (l, d, k), generator=g).float().to(DEV)
    fresh = [(torch.randint(-4, 5, (l, d, n), generator=g).float(),) for _ in range(2)]
    s, lab = capture_replay(lambda: fn.kmeans_assign(data, cent, "euclidean", exact_values=True), [data], fresh)
    es, el = fn.max_sim(data, cent, exact=True)
    assert_same((s, lab), (es, el))
    if kernel != "assign_wide":
        os_, ol = KO.max_sim(fresh[-1][0].numpy(), cent.cpu().numpy())
        assert np.array_equal(lab.cpu().numpy(), ol) and np.array_equal(s.cpu().numpy(), os_)
    if kernel != "assign_wide":
        capture_replay(lambda: fn.max_sim(data, cent, exact=True), [data], fresh)
        capture_replay(lambda: fn.max_sim(data, cent, exact=False, exact_values=False), [data], fresh)


def test_capture_compute_centroids_pq_decode_merge(pq_small):
    st, queries, ix = pq_small
    fn = _T().fn
    g = torch.Generator().manual_seed(3)
    data = torch.randint(-4, 5, (2, 16, 3000), generator=g).float().to(DEV)
    labels = torch.randint(0, 300, (2, 3000), generator=g).to(DEV)
    fresh = [(torch.randint(-4, 5, (2, 16, 3000), generator=g).float(), torch.randint(0, 300, (2, 3000), generator=g))
             for _ in range(2)]
    cent = capture_replay(lambda: fn.compute_centroids(data, labels, 300), [data, labels], fresh)
    want = KO.compute_centroids(fresh[-1][0].numpy(), fresh[-1][1].numpy(), 300)
    assert np.allclose(cent.cpu().numpy(), want, rtol=1e-6, atol=1e-6)

    pq = _t(st.pq_codebook)
    code = torch.randint(0, 256, (16, 500), generator=g, dtype=torch.uint8).to(DEV)
    fresh = [(torch.randint(0, 256, (16, 500), generator=g, dtype=torch.uint8),) for _ in range(2)]
    out = capture_replay(lambda: fn.pq_decode(pq, code), [code], fresh)
    assert np.array_equal(out.cpu().numpy(), KO.pq_decode(st.pq_codebook, fresh[-1][0].numpy()).reshape(-1, 500))

    def parts(seed):
        xs = queries(30, seed).to(DEV)
        return torch.stack([ix.search(xs[:, :], k=20, return_keys=True)[2],
                            ix.search_cells(xs, fn.coarse_probe(xs, ix.vq_codec.codebook, 3, False)[1], k=20,
                                            return_keys=True)[2]]).contiguous()
    keys = parts(1)
    capture_replay(lambda: fn.merge_topk(keys, ix._address2id), [keys], [(parts(2),), (parts(3),)])


def test_capture_placement_kernels(cuda_device):
    fn = _T().fn
    ix = _T().IVFPQIndex(64, 16, 32, initial_size=200, device=DEV)        # room for every item: no write past a cell
    g = torch.Generator().manual_seed(5)
    cells = torch.randint(0, 32, (2000,), generator=g).to(DEV)
    is_empty = ix._is_empty.clone()
    fresh_c = [(torch.randint(0, 32, (2000,), generator=g),) for _ in range(2)]
    capture_replay(lambda: fn.get_ioa(cells, 32), [cells], fresh_c)
    fresh_e = [((torch.rand(is_empty.shape[0], generator=g) < 0.3).to(torch.uint8),) for _ in range(2)]
    capture_replay(lambda: fn.empty_prefix(is_empty), [is_empty], fresh_e)
    ioa = fn.get_ioa(cells, 32)[0]
    prefix = fn.empty_prefix(ix._is_empty)
    capture_replay(lambda: fn.get_write_address(cells, ioa, ix._cell_start, ix._cell_size, ix._cell_capacity, prefix),
                   [cells, ioa], [(c.to(DEV), fn.get_ioa(c.to(DEV), 32)[0]) for (c,) in fresh_c])


# ============================================================================ b. synchronising paths on a side stream

def beside_sleep(fn, side, cycles):
    """Run fn() on `side` while a sleep of SLEEP_S occupies the legacy default stream; require the host to get fn's
    answer while the sleep still runs.  -> fn()'s result."""
    torch.cuda.synchronize()
    torch.cuda._sleep(cycles)
    t0 = time.perf_counter()
    with torch.cuda.stream(side):
        out = fn()
    side.synchronize()
    busy, took = not torch.cuda.default_stream().query(), time.perf_counter() - t0
    torch.cuda.synchronize()
    assert busy, f"the call took {took:.3f} s: it waited for the default stream (a launch on, or a sync with, stream 0)"
    return out


def _state(ix):
    return {k: v for k, v in ix.state_dict().items() if v is not None}


def assert_same_state(a, b):
    sa, sb = _state(a), _state(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert_same(sa[k], sb[k])


def _life_cycle(make, d, seed):
    """A train (where the index has one), add with expansion, remove, add into the holes, then search and range search:
    -> a function running it on a new index, returning (index, outputs)."""
    base = _ivf_data(d, 8, 3000, seed)

    def run():
        ix = make()
        xt = _t(base)
        if not isinstance(ix, _T().FlatIndex):
            ix.train(xt[:, :2000])
        ix.add(xt[:, :2000])
        ix.remove(ids=torch.arange(0, 2000, 3, device=DEV))
        ix.add(xt[:, 2000:])
        q = xt[:, :20] + 0.5
        out = ix.search(q, k=10, return_address=True)
        if not isinstance(ix, _T().IVFPQRIndex):
            t = float(out[0][:, -1].median())
            out = out + ix.range_search(q, t, return_address=True)
        return ix, out
    return run


def _families():
    T = _T()
    return {
        "flat": lambda: T.FlatIndex(32, initial_size=100, expand_step_size=64, device=DEV),
        "ivfflat": lambda: T.IVFFlatIndex(32, 8, initial_size=4, device=DEV),
        "ivfsq": lambda: T.IVFSQIndex(32, 8, bits=8, initial_size=4, device=DEV),
        "ivfpq": lambda: T.IVFPQIndex(32, 8, 8, initial_size=4, device=DEV),
        "ivfpqr": lambda: T.IVFPQRIndex(32, 8, 8, 8, initial_size=4, device=DEV),
    }


@pytest.mark.parametrize("family", ["flat", "ivfflat", "ivfsq", "ivfpq", "ivfpqr"])
def test_sync_paths_on_a_side_stream(family, sleep_cycles):
    run = _life_cycle(_families()[family], 32, 3)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):                                        # eager, and warms the side stream's pool
        ref_ix, ref_out = run()
    side.synchronize()
    ix, out = beside_sleep(run, side, sleep_cycles)
    assert_same(out, ref_out)
    assert_same_state(ix, ref_ix)
    assert ix.capacity > (100 if family == "flat" else 32), "the add did not expand the container"


def test_kmeans_fit_on_a_side_stream(sleep_cycles):
    T = _T()
    data = _t(_ivf_data(16, 8, 4000, 4))
    multi = _t(np.stack([_ivf_data(8, 8, 2000, s) for s in range(3)]))

    def run():
        km, mkm = T.KMeans(32, max_iter=10, seed=1), T.MultiKMeans(16, max_iter=10, seed=2)
        return (km.fit(data), km.centroids, mkm.fit(multi), mkm.centroids)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        want = run()
    side.synchronize()
    assert_same(beside_sleep(run, side, sleep_cycles), want)


# ============================================================================ c. a cache built on one stream, read on another

def cross_stream(build, search, cycles):
    """On stream A: a sleep, then build(); at once, on stream B: search().  -> (search's result, whether the sleep had
    ended when B's work was complete).  An event recorded right after the sleep decides the order, with no clock."""
    A, Bs = torch.cuda.Stream(), torch.cuda.Stream()
    for s in (A, Bs):                                                     # warms the kernels and both streams' pools
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            build()
            search()
    torch.cuda.synchronize()
    slept = torch.cuda.Event()
    with torch.cuda.stream(A):
        torch.cuda._sleep(cycles)
        slept.record(A)
        build()
    with torch.cuda.stream(Bs):
        out = search()
    Bs.synchronize()
    waited = slept.query()
    torch.cuda.synchronize()
    return out, waited


def _drop_norms(ix):
    def build():
        ix._norms = None
        ix._norm_table()
    return build


WAIT_MSG = "the search on stream B completed before the build on stream A began: it read the cache unfinished"


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_flat_norm_table_across_streams(flat_base, distance, sleep_cycles):
    ix = _T().FlatIndex(48, distance=distance, device=DEV)
    ix.add(_t(flat_base))
    x = _randn(48, 32, seed=14)
    o = FO.FlatOracle(48, distance=distance)
    o.add(flat_base)
    out, waited = cross_stream(_drop_norms(ix), lambda: ix.search(x, k=10, return_address=True), sleep_cycles)
    assert waited, WAIT_MSG
    assert_oracle(out, o.search(x.cpu().numpy(), 10))


def test_ivfflat_norm_table_across_streams(ivfflat, sleep_cycles):
    x = _randn(32, 32, seed=15)
    out, waited = cross_stream(_drop_norms(ivfflat), lambda: ivfflat.search(x, k=10, return_address=True), sleep_cycles)
    assert waited, WAIT_MSG
    assert_oracle(out, VO.search(VO.state_of(ivfflat), x.cpu().numpy(), 10, 4))


def test_ivfsq_norm_table_across_streams(sleep_cycles):
    base = _ivf_data(32, 16, 4000, 6)
    ix = _T().IVFSQIndex(32, 16, bits=8, initial_size=8, device=DEV)
    ix.train(_t(base))
    ix.add(_t(base))
    ix.n_probe, ix.use_smart_probing = 4, False
    x = _randn(32, 32, seed=16)
    out, waited = cross_stream(_drop_norms(ix), lambda: ix.search(x, k=10, return_address=True), sleep_cycles)
    assert waited, WAIT_MSG
    assert_oracle(out, QO.search(QO.state_of(ix), x.cpu().numpy(), 10, 4))


def test_scan_layout_across_streams(pq_small, sleep_cycles):
    """A regression pin of values only: the layout's build reads a size back (.item() on stream A), which holds the
    host until A's sleep has ended, before B's search is even enqueued, so the order check below holds whether or not
    the search waits.  What can regress for the layout, the capture that skips that wait, is pinned by
    test_capture_cache_built_on_another_stream."""
    st, queries, ix = pq_small
    x = queries(32, 4).to(DEV)

    def build():
        ix._layout = None
        ix.layout()
    out, waited = cross_stream(build, lambda: ix.search(x, k=10, return_address=True), sleep_cycles)
    assert waited
    assert_oracle(out, O.search(st, x.cpu(), k=10, return_address=True))


# ============================================================================ d. concurrent searches

def _concurrent(search, xs):
    serial = [search(x) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    outs = []
    for s, x in zip(streams, xs):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            outs.append(search(x))
    torch.cuda.synchronize()
    for o, w in zip(outs, serial):
        assert_same(o, w)


def test_concurrent_searches(flat_base, ivfflat, pq_small, pq_cell_major):
    T = _T()
    fx = T.FlatIndex(48, device=DEV)
    fx.add(_t(flat_base))
    _concurrent(lambda x: fx.search(x, k=100, return_address=True), [_randn(48, 50 + 10 * s, seed=s) for s in range(4)])
    _concurrent(lambda x: ivfflat.search(x, k=20, return_address=True), [_randn(32, 40, seed=s) for s in range(4)])
    st, queries, px = pq_small
    _concurrent(lambda x: px.search(x, k=50, return_address=True), [queries(n, s).to(DEV) for s, n in
                                                                     enumerate((32, 64, 600, 100))])
    st, queries, cx = pq_cell_major
    _concurrent(lambda x: cx.search(x, k=100, return_address=True), [queries(n, s).to(DEV) for s, n in
                                                                     enumerate((CELL_NQ, 64, CELL_NQ, 100))])
    rx, rq = RQ.make_index(32, 8, 16, 8, 3000, seed=2, kind="int", n_probe=4)
    _concurrent(lambda x: rx.search(x, k=10, return_address=True), [rq(24, s) for s in range(4)])


# ============================================================================ e. an index on another device

@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible CUDA devices")
def test_index_on_another_device(cuda_device, flat_base, ivfflat, pq_small):
    """Every index and operator on cuda:1 while cuda:0 is current returns what the same call returns on cuda:0, and
    leaves cuda:0 current."""
    T = _T()
    other = torch.device("cuda:1")
    torch.cuda.set_device(0)

    def on(dev, fn):
        return [t.cpu() if isinstance(t, torch.Tensor) else t for t in fn(dev)]

    def flat(dev):
        ix = T.FlatIndex(48, initial_size=100, device=dev)
        ix.add(torch.from_numpy(flat_base).to(dev))
        ix.remove(ids=torch.arange(0, 5000, 7, device=dev))
        x = torch.from_numpy(flat_base[:, :20] + 0.5).to(dev)
        return list(ix.search(x, k=10, return_address=True)) + list(ix.range_search(x, -40.0))

    def ivf(dev):
        base = _ivf_data(32, 16, 4000, 5)
        ix = T.IVFSQIndex(32, 16, bits=8, initial_size=8, device=dev)
        ix.train(torch.from_numpy(base).to(dev))
        ix.add(torch.from_numpy(base).to(dev))
        ix.remove(ids=torch.arange(0, 4000, 5, device=dev))
        ix.n_probe = 4
        x = torch.from_numpy(base[:, :20]).to(dev)
        cells = torch.randint(0, 16, (20, 3), generator=torch.Generator().manual_seed(1)).to(dev)
        return list(ix.search(x, k=10, return_address=True)) + list(ix.search_cells(x, cells, k=10)) + \
            list(ix.range_search(x, -20.0))

    def pq(dev):
        st, queries, _ = pq_small
        ix = make_index(st, device=str(dev))
        x = queries(600, 7).to(dev)
        before = list(ix.search(x, k=20, return_address=True)) + list(ix.range_search(x[:, :16], -10.0))
        ix.add(queries(300, 8).to(dev))
        return before + list(ix.search(x[:, :32], k=20))

    def ops(dev):
        fn = T.fn
        x = torch.randn(64, 300, generator=torch.Generator().manual_seed(2)).to(dev)
        cb = torch.randn(64, 40, generator=torch.Generator().manual_seed(3)).to(dev)
        codec = T.codec.SQCodec(bits=8)
        codec.train(x)
        data = torch.randint(-4, 5, (1, 64, 1000), generator=torch.Generator().manual_seed(4)).float().to(dev)
        cent = torch.randint(-4, 5, (1, 64, 300), generator=torch.Generator().manual_seed(5)).float().to(dev)
        return [*fn.coarse_probe(x, cb, 8), *T.topk(x, k=16), fn.normalize(x), codec.decode(codec.encode(x)),
                *fn.kmeans_assign(data, cent), *fn.max_sim(data, cent, exact=False)]

    for case in (flat, ivf, pq, ops):
        got = on(other, case)
        assert torch.cuda.current_device() == 0
        assert_same(tuple(got), tuple(on(torch.device(DEV), case)))
