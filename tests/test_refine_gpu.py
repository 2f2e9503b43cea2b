"""GPU: RefineFlatIndex.refine and .search against the numpy restatement of the exact pass (oracle/refine_oracle.py) bit
for bit, the value against fn.max_sim on the stored vector, every base index family, the store's life cycle,
checkpoints, streams, CUDA graphs and recall."""
import numpy as np
import pytest
import torch

from oracle import refine_oracle as RF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)


def assert_same(got, want):
    v, i, a = (t.cpu().numpy() for t in got)
    ov, oi, oa = want
    assert np.array_equal(v, ov), f"values differ at {np.argwhere(v != ov)[:5]}"
    assert np.array_equal(a, oa) and np.array_equal(i, oi)


def oracle_refine(ix, x, cand, k):
    return RF.refine(x.cpu().numpy(), cand.cpu().numpy(), *RF.state_of(ix), ix.distance, k)


def oracle_search(ix, x, k):
    base = lambda xn, k1: ix.base_index.search(_t(xn), k1)[1].cpu().numpy()
    return RF.search(x.cpu().numpy(), k, ix.k_factor, base, *RF.state_of(ix), ix.distance)


def flat_refine(d, n, distance="euclidean", seed=0, removed=0):
    """A RefineFlatIndex over a FlatIndex of n random vectors under scattered ids, `removed` of them removed again."""
    import torchpq_b200 as T
    rng = np.random.default_rng(seed)
    ix = T.RefineFlatIndex(T.FlatIndex(d, distance=distance, device=DEV))
    ids = torch.from_numpy(rng.permutation(20 * n)[:n]).long().to(DEV)
    ix.add(_t(rng.standard_normal((d, n))), ids)
    gone = ids[torch.from_numpy(rng.permutation(n)[:removed]).to(DEV)]
    ix.remove(gone)
    return ix, ids, gone, rng


# ----------------------------------------------------------------------------------------- refine, bit for bit
def multi_tile_nq():
    """A batch that gives every CTA of refine_kernel's persistent grid at least two tiles of 8 queries, so the tile
    loop's second and later iterations (reused x, keys, lists and cp.async buffers) are checked.  The grid is at most
    SMs x CTAs per SM, and a CTA's 67.6 KB of chunk buffers alone allow at most 3 CTAs in an SM's 228 KB; the odd
    remainder leaves a partial last tile."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * 8 * 3 * sms + 5


@pytest.mark.parametrize("distance,d,k,k1,nq", [
    ("euclidean", 3, 1, 16, 20),
    ("cosine", 3, 4, 40, 9),
    ("euclidean", 37, 10, 10, 20),           # k = k1
    ("cosine", 37, 8, 64, 17),
    ("euclidean", 128, 100, 1024, 12),       # k1 = 1024
    ("cosine", 128, 1, 1024, 8),
    ("euclidean", 256, 1024, 1024, 5),       # k = k1 = 1024
    ("cosine", 256, 30, 200, 11),
    ("euclidean", 37, 5, 8, "tiles"),        # at least two query tiles per CTA (multi_tile_nq)
    ("cosine", 128, 10, 64, "tiles"),
    ("cosine", 128, 50, 400, 0),             # an empty batch
])
def test_refine_matches_oracle(distance, d, k, k1, nq):
    if nq == "tiles":
        nq = multi_tile_nq()
    ix, ids, gone, rng = flat_refine(d, 1500, distance, seed=d + k1, removed=200)
    pool = np.concatenate([ids.cpu().numpy(), gone.cpu().numpy(), [-1, -1, 10 ** 9, 123456789]])
    cand = torch.from_numpy(rng.choice(pool, size=(nq, k1))).long().to(DEV)   # live, removed, -1, unknown, repeats
    if nq > 2:
        cand[1, 3:] = -1                                              # fewer live candidates than k
        cand[2, :] = gone[0]                                          # none live
    x = _t(rng.standard_normal((d, nq)))
    got = ix.refine(x, cand, k, return_address=True)
    torch.cuda.synchronize()
    assert got[0].shape == (nq, k)
    assert_same(got, oracle_refine(ix, x, cand, k))
    if nq > 2:
        assert bool(torch.isinf(got[0][2]).all()) and bool((got[1][2] == -1).all()) and bool((got[2][2] == -1).all())


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_identical_vectors_rank_by_insertion(distance):
    """The same vector under three ids: the one added first has the lowest store address and ranks first."""
    import torchpq_b200 as T
    rng = np.random.default_rng(1)
    d = 24
    ix = T.RefineFlatIndex(T.FlatIndex(d, distance=distance, device=DEV))
    v = rng.standard_normal((d, 1)).astype(np.float32)
    ix.add(_t(rng.standard_normal((d, 50))), torch.arange(100, 150, device=DEV))
    ix.add(_t(v), torch.tensor([900], device=DEV))
    ix.add(_t(rng.standard_normal((d, 20))), torch.arange(200, 220, device=DEV))
    ix.add(_t(np.repeat(v, 2, 1)), torch.tensor([7, 800], device=DEV))
    x = _t(v + 0.01 * rng.standard_normal((d, 1)))
    cand = torch.tensor([[800, 7, 150 - 1, 900, 800, -1]], device=DEV)
    got = ix.refine(x, cand, 5, return_address=True)
    assert_same(got, oracle_refine(ix, x, cand, 5))
    assert got[1][0, :4].tolist() == [900, 7, 800, 800]
    assert got[0][0, 0] == got[0][0, 1] == got[0][0, 2]


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_value_is_max_sim_of_stored_vector(distance):
    import torchpq_b200 as T
    ix, ids, _, rng = flat_refine(96, 2000, distance, seed=5)
    x = _t(rng.standard_normal((96, 6)))
    cand = ids[torch.from_numpy(rng.integers(0, 2000, size=(6, 300))).to(DEV)]
    v, i, a = ix.refine(x, cand, 50, return_address=True)
    xs = T.fn.normalize(x) if distance == "cosine" else x
    for q in range(6):
        y = ix._vectors[a[q]].t().contiguous()
        ref = T.fn.max_sim(y[None], xs[:, q:q + 1][None].contiguous(), distance, exact=True)[0][0]
        assert torch.equal(v[q], ref)


# ----------------------------------------------------------------------------------------- search over every base
def clustered(n, d, n_clusters, seed):
    centers = torch.randn(d, n_clusters, generator=torch.Generator(device="cpu").manual_seed(100)) * 3
    g = torch.Generator(device="cpu").manual_seed(seed)
    lab = torch.randint(0, n_clusters, (n,), generator=g)
    return (centers[:, lab] + torch.randn(d, n, generator=g)).to(DEV)


def make_base(kind, d, n_cells, distance):
    import torchpq_b200 as T
    if kind == "ivfpq":
        b = T.IVFPQIndex(d, 8, n_cells, distance=distance, device=DEV)
    elif kind == "ivfpq_residual":
        b = T.IVFPQIndex(d, 8, n_cells, distance=distance, device=DEV, pq_use_residual=True)
    elif kind == "ivfpqr":
        b = T.IVFPQRIndex(d, 8, 8, n_cells, distance=distance, device=DEV)
    elif kind == "ivfsq":
        b = T.IVFSQIndex(d, n_cells, bits=8, distance=distance, device=DEV)
    elif kind == "ivfflat":
        b = T.IVFFlatIndex(d, n_cells, distance=distance, device=DEV)
    else:
        return T.FlatIndex(d, distance=distance, device=DEV)
    b.n_probe, b.use_smart_probing = 4, False
    return b


@pytest.mark.parametrize("kind,distance,k,k_factor", [
    ("ivfpq", "euclidean", 10, 4),
    ("ivfpq", "cosine", 20, 2),
    ("ivfpq_residual", "euclidean", 10, 3),
    ("ivfsq", "euclidean", 10, 4),
    ("ivfsq", "cosine", 5, 1),
    ("ivfpqr", "euclidean", 10, 4),
])
def test_search_matches_oracle_over_base(kind, distance, k, k_factor):
    import torchpq_b200 as T
    data = clustered(6000, 32, 40, seed=0)
    ix = T.RefineFlatIndex(make_base(kind, 32, 16, distance), k_factor=k_factor)
    ix.train(data[:, :4000])
    ix.add(data)
    x = clustered(40, 32, 40, seed=1)
    got = ix.search(x, k=k, return_address=True)
    torch.cuda.synchronize()
    assert_same(got, oracle_search(ix, x, k))


@pytest.mark.parametrize("kind,distance", [("flat", "euclidean"), ("flat", "cosine"), ("ivfflat", "euclidean"),
                                           ("ivfpq", "cosine")])
def test_search_is_brute_force_when_the_base_returns_everything(kind, distance):
    """k1 >= n and (IVF) n_probe = n_cells: every item is a candidate, so search is the exact top-k of the store."""
    import torchpq_b200 as T
    data = clustered(700, 32, 20, seed=2)
    base = make_base(kind, 32, 8, distance)
    if kind != "flat":
        base.n_probe = 8
    ix = T.RefineFlatIndex(base, k_factor=100)                       # k1 = 1000 >= 700
    ix.train(data)
    ix.add(data)
    ix.remove(torch.arange(0, 700, 7, device=DEV))
    x = clustered(25, 32, 20, seed=3)
    got = ix.search(x, k=10, return_address=True)
    torch.cuda.synchronize()
    assert_same(got, RF.brute_force(x.cpu().numpy(), 10, *RF.state_of(ix), distance))


# ----------------------------------------------------------------------------------------- life cycle, checkpoints
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_life_cycle_from_a_small_capacity(distance):
    import torchpq_b200 as T
    rng = np.random.default_rng(11)
    d = 32
    base = make_base("ivfpq", d, 8, distance)
    base.train(clustered(3000, d, 20, seed=4))
    ix = T.RefineFlatIndex(base)
    rows = {}
    for step in range(10):
        n = int(rng.integers(1, 300))
        x = clustered(n, d, 20, seed=10 + step)
        ids = ix.add(x) if step % 3 == 0 else ix.add(x, torch.from_numpy(rng.permutation(10 ** 6)[:n] + 10 ** 6 * step).long().to(DEV))
        stored = T.fn.normalize(x) if distance == "cosine" else x
        rows.update({int(i): stored[:, j] for j, i in enumerate(ids.tolist())})
        if step % 2:
            gone = rng.choice(sorted(rows), len(rows) // 4, replace=False).tolist()
            assert ix.remove(torch.tensor(gone + [-1, 5 * 10 ** 7], device=DEV)) == len(gone)
            for i in gone:
                del rows[i]
        assert ix.n_items == len(rows)
        assert int((base._address2id >= 0).sum()) == len(rows)
    assert ix.capacity >= ix.n_items and ix.capacity & (ix.capacity - 1) == 0
    for a, i in enumerate(ix._address2id[:ix.n_items].tolist()):
        assert torch.equal(ix._vectors[a], rows[i])
    x = clustered(30, d, 20, seed=99)
    assert_same(ix.search(x, k=10, return_address=True), oracle_search(ix, x, 10))


def test_duplicate_add_raises_and_changes_nothing():
    import torchpq_b200 as T
    base = make_base("ivfpq", 32, 8, "euclidean")
    data = clustered(2000, 32, 20, seed=5)
    ix = T.RefineFlatIndex(base)
    ix.train(data)
    ix.add(data[:, :1000], torch.arange(1000, device=DEV) * 3)
    before = {k: v.clone() for k, v in ix.state_dict().items()}
    for ids in (torch.tensor([1, 2, 1], device=DEV), torch.tensor([1, 2, 300], device=DEV)):
        with pytest.raises(ValueError):
            ix.add(data[:, 1000:1003], ids)
        after = ix.state_dict()
        assert set(after) == set(before) and all(torch.equal(after[k], v) for k, v in before.items())


def test_state_dict_round_trip():
    import torchpq_b200 as T
    data = clustered(4000, 32, 20, seed=6)
    ix = T.RefineFlatIndex(make_base("ivfpq", 32, 16, "cosine"), k_factor=2)
    ix.train(data)
    ix.add(data)
    ix.remove(torch.arange(0, 4000, 5, device=DEV))
    ix2 = T.RefineFlatIndex(make_base("ivfpq", 32, 16, "cosine"), k_factor=2)
    ix2.load_state_dict(ix.state_dict())
    assert ix2.n_items == ix.n_items and ix2.max_id == ix.max_id
    x = clustered(20, 32, 20, seed=7)
    for a, b in zip(ix.search(x, k=10, return_address=True), ix2.search(x, k=10, return_address=True)):
        assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------- streams and graphs
def _stream_index():
    import torchpq_b200 as T
    data = clustered(5000, 32, 20, seed=8)
    ix = T.RefineFlatIndex(make_base("ivfpq", 32, 16, "euclidean"))
    ix.train(data)
    ix.add(data)
    return ix


def test_side_stream_equals_default_stream():
    ix = _stream_index()
    x = clustered(64, 32, 20, seed=9)
    want = ix.search(x, k=10, return_address=True)
    S = torch.cuda.Stream()
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        got = ix.search(x, k=10, return_address=True)
    S.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_captured_graph_equals_eager():
    ix = _stream_index()
    x = clustered(64, 32, 20, seed=10)
    S = torch.cuda.Stream()
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        ix.search(x, k=10, return_address=True)                       # the one warm call
    S.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=S):
        out = ix.search(x, k=10, return_address=True)
    for seed in (11, 12):
        x.copy_(clustered(64, 32, 20, seed=seed))
        g.replay()
        torch.cuda.synchronize()
        want = ix.search(x, k=10, return_address=True)
        for a, b in zip(out, want):
            assert torch.equal(a, b)
        assert_same(out, oracle_search(ix, x, 10))


# ----------------------------------------------------------------------------------------- recall
def test_refine_recall_beats_plain_base():
    import torchpq_b200 as T
    data = clustered(40000, 32, 100, seed=0)
    xq = clustered(500, 32, 100, seed=1)
    plain = T.IVFPQIndex(32, 8, 64, device=DEV)
    plain.n_probe = 8
    ix = T.RefineFlatIndex(plain, k_factor=1)
    ix.train(data[:, :20000], seed=0)
    ix.add(data)
    truth = (data.pow(2).sum(0)[None, :] - 2 * xq.t() @ data).argmin(1)
    r1 = lambda ids: float((ids[:, 0] == truth).float().mean())
    r_plain = r1(plain.search(xq, k=10)[1])
    r_refine = r1(ix.search(xq, k=10)[1])
    print(f"recall@1: IVFPQIndex {r_plain:.4f}, RefineFlatIndex (k_factor 1) {r_refine:.4f}")
    assert r_refine >= r_plain
