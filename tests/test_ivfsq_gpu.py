"""GPU: SQCodec's encode / decode kernels bit for bit against the numpy oracle (oracle/ivfsq_oracle.py), and
IVFSQIndex.search bit for bit against the oracle and against an IVFFlatIndex holding the decoded store, through the
add / remove life cycle, a checkpoint round trip and the edge cases of the probe lists and of the batch."""
import numpy as np
import pytest
import torch

from oracle import ivfsq_oracle as SO

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


def _data(d, n_cells, n, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((d, n_cells)).astype(np.float32) * 3
    return centres[:, rng.integers(0, n_cells, n)] + rng.standard_normal((d, n)).astype(np.float32), rng


def _build(d, n_cells, n, distance, bits=8, seed=0, initial_size=16):
    x, rng = _data(d, n_cells, n, seed)
    ix = _T().IVFSQIndex(d, n_cells, bits=bits, initial_size=initial_size, distance=distance, device=DEV)
    xt = torch.from_numpy(x).to(DEV)
    ix.train(xt, seed=seed)
    ix.add(xt)
    return ix, rng


# ---------------------------------------------------------------- codec
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("mode", ["minmax", "meanstd"])
def test_codec_matches_oracle(bits, mode):
    T = _T()
    rng = np.random.default_rng(bits)
    x = rng.standard_normal((24, 5000)).astype(np.float32) * 4
    x[:, :3] = [7e4, -7e4, 65504]                               # fp16 overflow; outside [lower, upper] for meanstd
    xt = torch.from_numpy(x).to(DEV)
    c = T.codec.SQCodec(bits=bits, mode=mode, alpha=1.5)
    c.train(xt)
    lo, rg = (c.lower.cpu().numpy(), c.range.cpu().numpy()) if bits == 8 else (None, None)
    if bits == 8 and mode == "minmax":
        assert torch.equal(c.lower, torch.amin(xt, dim=-1)) and torch.equal(c.upper, torch.amax(xt, dim=-1))
    x0 = xt.clone()
    code = c.encode(xt)
    want = SO.encode(x, bits, lo, rg)
    assert code.dtype == (torch.uint8 if bits == 8 else torch.float16) and code.shape == (24, 5000)
    assert np.array_equal(code.cpu().numpy().view(np.uint8), want.view(np.uint8))
    code0 = code.clone()
    back = c.decode(code)
    assert np.array_equal(_bits(back.cpu().numpy()), _bits(SO.decode(want, bits, lo, rg)))
    assert torch.equal(xt, x0) and torch.equal(code, code0)    # inputs are never written
    if bits == 8:                                               # every code, and the reference's torch decode on the GPU
        every = torch.arange(256, device=DEV, dtype=torch.uint8)[None].repeat(24, 1)
        ref = every.float().div_(256).mul_(c.range[:, None]).add_(c.lower[:, None])
        assert torch.equal(c.decode(every).view(torch.int32), ref.view(torch.int32))
    c32 = T.codec.SQCodec(bits=32)
    c32.train(xt)
    assert c32.encode(xt) is xt and c32.decode(xt) is xt


# ---------------------------------------------------------------- search
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
@pytest.mark.parametrize("d", [32, 100, 128])
@pytest.mark.parametrize("n_probe", [1, 8, "all"])
def test_search_matches_oracle(bits, distance, d, n_probe):
    C_ = 32
    n_probe = C_ if n_probe == "all" else n_probe
    ix, rng = _build(d, C_, 2500, distance, bits=bits, seed=d + bits)
    ix.n_probe, ix.use_smart_probing = n_probe, False
    st = SO.state_of(ix)
    xq = rng.standard_normal((d, 300)).astype(np.float32)
    want = SO.search(st, xq, 1024, n_probe)
    x = torch.from_numpy(xq).to(DEV)
    for k in (1, 10, 100, 1024):
        for nq in (1, 7, 300):
            got = ix.search(x[:, :nq], k=k, return_address=True)
            _same(got, tuple(w[:nq, :k] for w in want))


def _flat_twin(ix):
    """An IVFFlatIndex with the IVFSQIndex's buffers, its _storage replaced by the decoded fp32 [d, capacity, 1]."""
    T = _T()
    fl = T.IVFFlatIndex(ix.d_vector, ix.n_cells, initial_size=0, distance=ix.distance, device=DEV)
    sd = {k: v for k, v in ix.state_dict().items() if not k.startswith("sq_codec.")}
    cap = ix.capacity
    sd["_storage"] = ix.decode(ix._codes_at(slice(0, cap)).contiguous())[:, :, None].contiguous()
    fl.load_state_dict(sd)
    return fl


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_ivfsq_equals_ivfflat_on_the_decoded_store(bits, distance):
    ix, rng = _build(64, 24, 4000, distance, bits=bits, seed=31)
    ix.remove(ids=torch.arange(0, 4000, 7, device=DEV))
    fl = _flat_twin(ix)
    x = torch.from_numpy(rng.standard_normal((64, 120)).astype(np.float32)).to(DEV)
    for ixx in (ix, fl):
        ixx.n_probe, ixx.use_smart_probing = 6, True
    cells = torch.randint(-2, 26, (120, 6), device=DEV)
    npl = torch.randint(0, 8, (120,), device=DEV)
    for k in (1, 16, 200):
        for u, w in zip(ix.search(x, k=k, return_address=True), fl.search(x, k=k, return_address=True)):
            assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                               w.view(torch.int32) if w.dtype == torch.float32 else w)
        for u, w in zip(ix.search_cells(x, cells, npl, k=k, return_address=True),
                        fl.search_cells(x, cells, npl, k=k, return_address=True)):
            assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                               w.view(torch.int32) if w.dtype == torch.float32 else w)
    assert torch.equal(ix._norm_table(), fl._norm_table())     # the norm table is tpq_flat_norms of the decoded store


def test_search_equals_search_cells_with_smart_probing():
    T = _T()
    ix, rng = _build(48, 64, 4000, "euclidean", seed=7)
    ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature = 12, True, 1.0
    x = torch.from_numpy(rng.standard_normal((48, 200)).astype(np.float32)).to(DEV)
    _, cells, npl = T.fn.coarse_probe(x, ix.vq_codec.codebook, 12, True, ix.smart_probing_temperature)
    assert int(npl.min()) < 12
    a = ix.search(x, k=20, return_address=True)
    b = ix.search_cells(x, cells, npl, k=20, return_address=True)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    _same(b, SO.search_cells(SO.state_of(ix), x.cpu().numpy(), cells.cpu().numpy(), npl.cpu().numpy(), 20))


@pytest.mark.parametrize("bits", [8, 16])
def test_storage_bytes_and_coarse_stage(bits):
    T = _T()
    ix, _ = _build(32, 16, 1000, "euclidean", bits=bits, seed=3)
    assert ix._storage.dtype == torch.uint8
    assert ix._storage.numel() == ix.capacity * 32 * bits // 8          # d (or 2 d) bytes per slot
    fl = T.IVFFlatIndex(32, 16, initial_size=16, device=DEV)
    x, _ = _data(32, 16, 1000, 3)
    fl.train(torch.from_numpy(x).to(DEV), seed=3)
    assert torch.equal(fl.vq_codec.codebook, ix.vq_codec.codebook)     # same data and seed: same coarse codebook


def test_life_cycle_with_expansion_remove_and_refill():
    ix, rng = _build(40, 8, 100, "euclidean", seed=13, initial_size=4)
    ix.n_probe, ix.use_smart_probing = 3, False
    xq = rng.standard_normal((40, 30)).astype(np.float32)
    x = torch.from_numpy(xq).to(DEV)

    def check():
        _same(ix.search(x, k=25, return_address=True), SO.search(SO.state_of(ix), xq, 25, 3))

    check()
    caps = [ix.capacity]
    for n in (50, 300, 7):                                               # adds that expand cells
        new = torch.from_numpy(rng.standard_normal((40, n)).astype(np.float32) * 2).to(DEV)
        ids, adr = ix.add(new, return_address=True)
        assert torch.equal(ix.get_data_by_address(adr), ix.decode(ix.encode(new)))
        caps.append(ix.capacity)
        check()
    assert caps[-1] > caps[0]
    ix.remove(ids=torch.arange(0, ix.max_id + 1, 3, device=DEV))
    assert ix._has_holes
    check()
    cap = ix.capacity
    new = torch.from_numpy(rng.standard_normal((40, 40)).astype(np.float32)).to(DEV)
    _, adr = ix.add(new, return_address=True)                           # fills holes first
    assert ix.capacity == cap and torch.equal(ix.get_data_by_address(adr), ix.decode(ix.encode(new)))
    check()


def test_edge_cases():
    T = _T()
    ix, rng = _build(16, 8, 40, "euclidean", seed=17, initial_size=2)
    ix.n_probe, ix.use_smart_probing = 2, False
    st = SO.state_of(ix)
    xq = rng.standard_normal((16, 5)).astype(np.float32)
    x = torch.from_numpy(xq).to(DEV)
    got = ix.search(x, k=64, return_address=True)
    _same(got, SO.search(st, xq, 64, 2))
    assert (got[1] == -1).any() and torch.isinf(got[0]).any()
    v, i = ix.search(torch.zeros(16, 0, device=DEV), k=5)
    assert v.shape == (0, 5) and i.shape == (0, 5)
    cells = torch.tensor([[3, 3, -1, 9, 5, 3], [0, 1, 2, 3, 4, 5], [7, 100, 7, 6, -5, 7],
                          [2, 2, 2, 2, 2, 2], [4, 5, 6, 7, 0, 1]], dtype=torch.long, device=DEV)
    for npl in ([6, 0, 7, 6, np.iinfo(np.int64).min], [1, 6, 3, 0, 2], [7, 7, 7, 7, 7]):
        npl_t = torch.tensor(npl, dtype=torch.long, device=DEV)
        got = ix.search_cells(x, cells, npl_t, k=30, return_address=True)
        _same(got, SO.search_cells(st, xq, cells.cpu().numpy(), np.array(npl, np.int64), 30))
    a = torch.tensor([-1, 0, ix.capacity, 5], device=DEV)
    data = ix.get_data_by_address(a)
    assert (data[:, [0, 2]] == 0).all() and torch.equal(data[:, 3], ix.decode(ix._codes_at(a[3:]).contiguous())[:, 0])
    ex = T.IVFSQIndex(16, 8, initial_size=0, device=DEV)                # a trained but empty index
    ex.vq_codec.set_codebook(ix.vq_codec.codebook.clone())
    ex.sq_codec.load_state_dict(ix.sq_codec.state_dict())
    ex.n_probe = 8
    v, i, a = ex.search(x, k=7, return_address=True)
    assert torch.isinf(v).all() and (v < 0).all() and (i == -1).all() and (a == -1).all()


@pytest.mark.parametrize("bits", [8, 16])
def test_inputs_unchanged_and_checkpoint_round_trip(bits):
    T = _T()
    ix, rng = _build(24, 16, 2000, "cosine", bits=bits, seed=23)
    ix.n_probe, ix.use_smart_probing = 4, True
    ix.remove(ids=torch.arange(0, 2000, 5, device=DEV))
    x = torch.from_numpy(rng.standard_normal((24, 64)).astype(np.float32)).to(DEV)
    x0 = x.clone()
    cells = torch.randint(0, 16, (64, 4), device=DEV)
    c0 = cells.clone()
    a = ix.search(x, k=10, return_address=True)
    b = ix.search_cells(x, cells, k=10)
    assert torch.equal(x, x0) and torch.equal(cells, c0)
    ix2 = T.IVFSQIndex(24, 16, bits=bits, initial_size=0, distance="cosine", device=DEV)
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
    _same(ix2.search(x, k=10, return_address=True), SO.search(SO.state_of(ix2), x.cpu().numpy(), 10, 4))


@pytest.mark.parametrize("bits,floor", [(16, 0.99), (8, 0.9)])
def test_recall_floor(bits, floor):
    # recall@10 with every cell probed, against exact fp32 search of the original vectors.  The first H100 run measured
    # 1.0000 (fp16) and 0.9745 (SQ8) on this set; the floors keep a margin below that: 0.99 and 0.9.
    T = _T()
    x, rng = _data(64, 16, 20000, 41)
    xt = torch.from_numpy(x).to(DEV)
    ix = T.IVFSQIndex(64, 16, bits=bits, device=DEV)
    ix.train(xt)
    ix.add(xt)
    ix.n_probe, ix.use_smart_probing = 16, False
    q = xt[:, rng.integers(0, 20000, 200)] + torch.from_numpy(rng.standard_normal((64, 200)).astype(np.float32)).to(DEV) * 0.3
    fx = T.FlatIndex(64, device=DEV)
    fx.add(xt)
    _, truth = fx.search(q.contiguous(), k=10)
    _, got = ix.search(q.contiguous(), k=10)
    hits = sum(len(set(a) & set(b)) for a, b in zip(got.cpu().tolist(), truth.cpu().tolist()))
    recall = hits / truth.numel()
    print(f"recall@10 bits={bits}: {recall:.4f}")
    assert recall >= floor
