"""GPU: IVFFlatIndex.search bit for bit against the numpy oracle (oracle/ivfflat_oracle.py), against FlatIndex with every
cell probed, against IVFPQIndex's coarse stage, through the add / remove life cycle, and on the edge cases of the
probe lists and of the batch."""
import numpy as np
import pytest
import torch

from oracle import ivfflat_oracle as VO

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _T():
    import torchpq_b200 as T
    return T


def _bits(v):
    return np.asarray(v, np.float32).view(np.uint32)


def _same(got, want, address=True):
    v, i = got[0].cpu().numpy(), got[1].cpu().numpy()
    assert np.array_equal(_bits(v), _bits(want[0])), "values differ from the oracle"
    assert np.array_equal(i, want[1]), "ids differ from the oracle"
    if address:
        assert np.array_equal(got[2].cpu().numpy(), want[2]), "addresses differ from the oracle"


def _build(d, n_cells, n, distance, seed=0, initial_size=16):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((d, n_cells)).astype(np.float32) * 3
    x = (centres[:, rng.integers(0, n_cells, n)] + rng.standard_normal((d, n)).astype(np.float32))
    ix = _T().IVFFlatIndex(d, n_cells, initial_size=initial_size, distance=distance, device=DEV)
    xt = torch.from_numpy(x).to(DEV)
    ix.train(xt, seed=seed)
    ix.add(xt)
    return ix, rng


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
@pytest.mark.parametrize("d", [33, 100, 128])
@pytest.mark.parametrize("n_probe", [1, 8, "all"])
def test_search_matches_oracle(distance, d, n_probe):
    C_ = 32
    n_probe = C_ if n_probe == "all" else n_probe
    ix, rng = _build(d, C_, 2500, distance, seed=d)
    ix.n_probe, ix.use_smart_probing = n_probe, False
    st = VO.state_of(ix)
    xq = rng.standard_normal((d, 300)).astype(np.float32)
    want = VO.search(st, xq, 1024, n_probe)
    x = torch.from_numpy(xq).to(DEV)
    for k in (1, 10, 100, 1024):
        for nq in (1, 7, 300):
            got = ix.search(x[:, :nq], k=k, return_address=True)
            _same(got, tuple(w[:nq, :k] for w in want))


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_every_cell_probed_equals_flat_index(distance):
    T = _T()
    ix, rng = _build(64, 16, 3000, distance, seed=5)
    ix.n_probe, ix.use_smart_probing = 16, False
    live = (ix._is_empty == 0).nonzero().flatten()
    fx = T.FlatIndex(64, distance=distance, device=DEV)
    fx.add(ix.get_data_by_address(live).contiguous(), ids=ix._address2id[live])
    x = torch.from_numpy(rng.standard_normal((64, 50)).astype(np.float32)).to(DEV)
    for k in (1, 10, 100):
        v, i = ix.search(x, k=k)
        fv, fi = fx.search(x, k=k)
        assert torch.equal(v.view(torch.int32), fv.view(torch.int32))
        # ids on rows whose k-th value is not tied with the next one (addresses differ between the two stores)
        fv2, _ = fx.search(x, k=k + 1)
        untied = fv2[:, k - 1] != fv2[:, k]
        assert torch.equal(i[untied], fi[untied])


def test_search_equals_search_cells_with_smart_probing():
    T = _T()
    ix, rng = _build(48, 64, 4000, "euclidean", seed=7)
    ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature = 12, True, 1.0    # a sharp softmax: short lists
    x = torch.from_numpy(rng.standard_normal((48, 200)).astype(np.float32)).to(DEV)
    _, cells, npl = T.fn.coarse_probe(x, ix.vq_codec.codebook, 12, True, ix.smart_probing_temperature)
    assert int(npl.min()) < 12                                             # smart probing shortened some lists
    a = ix.search(x, k=20, return_address=True)
    b = ix.search_cells(x, cells, npl, k=20, return_address=True)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    st = VO.state_of(ix)
    _same(b, VO.search_cells(st, x.cpu().numpy(), cells.cpu().numpy(), npl.cpu().numpy(), 20))


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_same_coarse_stage_as_ivfpq(distance):
    T = _T()
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.standard_normal((32, 3000)).astype(np.float32)).to(DEV)
    fl = T.IVFFlatIndex(32, 24, distance=distance, device=DEV)
    pq = T.IVFPQIndex(32, 8, 24, distance=distance, device=DEV)
    fl.train(x, seed=3)
    pq.train(x, seed=3)
    assert torch.equal(fl.vq_codec.codebook, pq.vq_codec.codebook)
    fl.add(x)
    pq.add(x)
    assert torch.equal(fl._cell_size, pq._cell_size) and torch.equal(fl._address2id, pq._address2id)


def test_life_cycle_with_expansion_remove_and_refill():
    ix, rng = _build(40, 8, 100, "euclidean", seed=13, initial_size=4)
    ix.n_probe, ix.use_smart_probing = 3, False
    xq = rng.standard_normal((40, 30)).astype(np.float32)
    x = torch.from_numpy(xq).to(DEV)

    def check():
        _same(ix.search(x, k=25, return_address=True), VO.search(VO.state_of(ix), xq, 25, 3))

    check()
    caps = [ix.capacity]
    for n in (50, 300, 7):                                                   # adds that expand cells
        new = torch.from_numpy(rng.standard_normal((40, n)).astype(np.float32) * 2).to(DEV)
        ids, adr = ix.add(new, return_address=True)
        assert torch.equal(ix.get_data_by_address(adr), new)
        caps.append(ix.capacity)
        check()
    assert caps[-1] > caps[0]
    ix.remove(ids=torch.arange(0, ix.max_id + 1, 3, device=DEV))
    assert ix._has_holes
    check()
    cap = ix.capacity
    new = torch.from_numpy(rng.standard_normal((40, 40)).astype(np.float32)).to(DEV)
    _, adr = ix.add(new, return_address=True)                               # fills holes first
    assert ix.capacity == cap and torch.equal(ix.get_data_by_address(adr), new)
    check()


def test_edge_cases():
    T = _T()
    ix, rng = _build(16, 8, 40, "euclidean", seed=17, initial_size=2)      # cells of a few items: k > live items
    ix.n_probe, ix.use_smart_probing = 2, False
    st = VO.state_of(ix)
    xq = rng.standard_normal((16, 5)).astype(np.float32)
    x = torch.from_numpy(xq).to(DEV)
    got = ix.search(x, k=64, return_address=True)
    _same(got, VO.search(st, xq, 64, 2))
    assert (got[1] == -1).any() and torch.isinf(got[0]).any()
    # nq = 0
    v, i = ix.search(torch.zeros(16, 0, device=DEV), k=5)
    assert v.shape == (0, 5) and i.shape == (0, 5)
    # caller probe lists: out-of-range cells, consecutive duplicates, a cell listed twice apart, odd n_probe_list
    cells = torch.tensor([[3, 3, -1, 9, 5, 3], [0, 1, 2, 3, 4, 5], [7, 100, 7, 6, -5, 7],
                          [2, 2, 2, 2, 2, 2], [4, 5, 6, 7, 0, 1]], dtype=torch.long, device=DEV)
    for npl in ([6, 0, 7, 6, np.iinfo(np.int64).min], [1, 6, 3, 0, 2], [7, 7, 7, 7, 7]):
        npl_t = torch.tensor(npl, dtype=torch.long, device=DEV)
        got = ix.search_cells(x, cells, npl_t, k=30, return_address=True)
        _same(got, VO.search_cells(st, xq, cells.cpu().numpy(), np.array(npl, np.int64), 30))
    # a trained but empty index
    ex = T.IVFFlatIndex(16, 8, initial_size=0, device=DEV)
    ex.vq_codec.set_codebook(ix.vq_codec.codebook.clone())
    ex.n_probe = 8
    v, i, a = ex.search(x, k=7, return_address=True)
    assert torch.isinf(v).all() and (v < 0).all() and (i == -1).all() and (a == -1).all()


def test_plan_independence():
    ix, rng = _build(64, 64, 6000, "cosine", seed=19)
    ix.n_probe, ix.use_smart_probing = 64, False
    # n_probe * k * 8 B = 512 KB of keys per query: 600 queries are searched in two chunks
    x = torch.from_numpy(rng.standard_normal((64, 600)).astype(np.float32)).to(DEV)
    T = _T()
    assert T._lib.lib.tpq_ivfflat_workspace_bytes(64, 600, 64, 64, 1024) == \
        T._lib.lib.tpq_ivfflat_workspace_bytes(64, 6000, 64, 64, 1024)       # chunked: the workspace stopped growing
    big = ix.search(x, k=1024, return_address=True)
    small = ix.search(x[:, :20], k=1024, return_address=True)
    for u, w in zip(big, small):
        assert torch.equal(u[:20], w)
    one = [ix.search(x[:, q:q + 1].contiguous(), k=1024, return_address=True) for q in range(0, 600, 97)]
    for j, q in enumerate(range(0, 600, 97)):
        for u, w in zip(big, one[j]):
            assert torch.equal(u[q:q + 1], w)


def test_inputs_unchanged_and_checkpoint_round_trip():
    T = _T()
    ix, rng = _build(24, 16, 2000, "cosine", seed=23)
    ix.n_probe, ix.use_smart_probing = 4, True
    ix.remove(ids=torch.arange(0, 2000, 5, device=DEV))
    x = torch.from_numpy(rng.standard_normal((24, 64)).astype(np.float32)).to(DEV)
    x0 = x.clone()
    cells = torch.randint(0, 16, (64, 4), device=DEV)
    c0 = cells.clone()
    a = ix.search(x, k=10, return_address=True)
    b = ix.search_cells(x, cells, k=10)
    assert torch.equal(x, x0) and torch.equal(cells, c0)
    ix2 = T.IVFFlatIndex(24, 16, initial_size=0, distance="cosine", device=DEV)
    ix2.load_state_dict(ix.state_dict())
    ix2.n_probe, ix2.use_smart_probing = 4, True
    assert ix2.max_id == ix.max_id
    for u, w in zip(a, ix2.search(x, k=10, return_address=True)):
        assert torch.equal(u, w)
    for u, w in zip(b, ix2.search_cells(x, cells, k=10)):
        assert torch.equal(u, w)
    new = torch.from_numpy(rng.standard_normal((24, 30)).astype(np.float32)).to(DEV)
    ids = ix2.add(new)
    assert int(ids.min()) == ix.max_id + 1
    ix2.use_smart_probing = False
    _same(ix2.search(x, k=10, return_address=True), VO.search(VO.state_of(ix2), x.cpu().numpy(), 10, 4))
