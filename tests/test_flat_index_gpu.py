"""GPU: FlatIndex.search (tpq_flat_search) bit for bit against the numpy oracle (flat_oracle.flat_sims + the total order
of the candidate keys), whatever the plan picks; the container driving it; inputs and store left untouched."""
import numpy as np
import pytest
import torch

from oracle.flat_oracle import FlatOracle

pytestmark = pytest.mark.gpu

METRICS = ["euclidean", "cosine", "inner"]


def _pair(base, distance, ids=None, initial_size=None):
    import torchpq_b200 as T
    d, n = base.shape
    ix = T.FlatIndex(d, initial_size=initial_size, device="cuda:0", distance=distance)
    o = FlatOracle(d, initial_size=initial_size, distance=distance)
    if n:
        ix.add(torch.from_numpy(base).cuda(), None if ids is None else torch.from_numpy(ids).cuda())
        o.add(base, ids)
    return ix, o


def _check(ix, o, x, k):
    v, i, a = ix.search(torch.from_numpy(x).cuda(), k=k, return_address=True)
    ov, oi, oa = o.search(x, k)
    assert v.shape == (x.shape[1], k) and v.dtype == torch.float32 and i.dtype == torch.int64
    assert np.array_equal(v.cpu().numpy().view(np.uint32), ov.view(np.uint32)), "values differ"
    assert np.array_equal(a.cpu().numpy(), oa), "addresses differ"
    assert np.array_equal(i.cpu().numpy(), oi), "ids differ"
    return v, i, a


@pytest.mark.parametrize("distance", ["euclidean", "inner"])
def test_integer_data_with_designed_ties(cuda_device, distance):
    """Small integers: every score is exact.  Columns repeat across tiles and slices (copies 1000 and 2176 columns
    apart), so equal scores are everywhere and the address order decides."""
    rng = np.random.default_rng(0)
    d, n = 16, 3500
    base = rng.integers(-3, 4, (d, n)).astype(np.float32)
    base[:, 1000:1300] = base[:, :300]
    base[:, 2176:2476] = base[:, :300]
    base[:, 3300:3500] = base[:, 3000:3200]
    x = rng.integers(-3, 4, (d, 50)).astype(np.float32)
    ix, o = _pair(base, distance, ids=rng.permutation(10 * n)[:n].astype(np.int64))
    for k in (1, 100, 1024):
        _check(ix, o, x, k)


# (d, nq, n, k): every d, nq and k of the issue, n off the 128 grid, n < k, n = 0 and nq = 0
SHAPES = [(1, 7, 300, 10), (3, 129, 1000, 100), (17, 1, 5000, 1024), (128, 1000, 700, 128), (960, 7, 500, 129),
          (128, 129, 50, 100), (17, 7, 0, 10), (3, 0, 300, 10), (128, 1, 2000, 1), (17, 129, 3000, 1024)]


@pytest.mark.parametrize("distance", METRICS)
@pytest.mark.parametrize("d,nq,n,k", SHAPES)
def test_randn_bit_exact(cuda_device, distance, d, nq, n, k):
    rng = np.random.default_rng(d * 7919 + nq * 31 + n + k)
    base = rng.standard_normal((d, n)).astype(np.float32)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    ix, o = _pair(base, distance)
    v, i, a = _check(ix, o, x, k)
    if n < k and nq:
        assert (a[:, n:] == -1).all() and (i[:, n:] == -1).all() and torch.isneginf(v[:, n:]).all()


@pytest.mark.parametrize("distance", METRICS)
@pytest.mark.parametrize("k", [10, 100, 1024])
def test_independent_of_the_plan(cuda_device, distance, k):
    """A query's answer is the same alone (QT 16, many slices) and inside a 1000-query batch (QT up to 64, few slices)."""
    rng = np.random.default_rng(k)
    base = rng.standard_normal((64, 6000)).astype(np.float32)
    x = torch.from_numpy(rng.standard_normal((64, 1000)).astype(np.float32)).cuda()
    ix, _ = _pair(base, distance)
    full = ix.search(x, k=k, return_address=True)
    for sel in (slice(0, 1), slice(500, 507), slice(871, 1000)):
        part = ix.search(x[:, sel].contiguous(), k=k, return_address=True)
        for p, f in zip(part, full):
            assert torch.equal(p, f[sel])


@pytest.mark.parametrize("k", [10, 1024])
def test_worst_to_best_order(cuda_device, k):
    """Base columns sorted from worst to best for every query: each tile raises each query's threshold."""
    rng = np.random.default_rng(5)
    d, n = 32, 4000
    centre = rng.standard_normal(d).astype(np.float32)
    base = (centre[:, None] + rng.standard_normal((d, n)).astype(np.float32) * 3).astype(np.float32)
    base = base[:, np.argsort(-((base - centre[:, None]) ** 2).sum(0))]       # farthest first
    x = (centre[:, None] + 0.01 * rng.standard_normal((d, 40))).astype(np.float32)
    ix, o = _pair(base, "euclidean")
    _check(ix, o, x, k)


@pytest.mark.parametrize("distance", METRICS)
def test_container_then_search(cuda_device, distance):
    rng = np.random.default_rng(11)
    d = 24
    ix, o = _pair(np.zeros((d, 0), np.float32), distance, initial_size=100)
    x = rng.standard_normal((d, 30)).astype(np.float32)
    _check(ix, o, x, 5)                                                  # empty index: all padding
    for n, with_ids in ((150, False), (90, True), (400, False)):
        b = rng.standard_normal((d, n)).astype(np.float32)
        ids = (rng.permutation(100000)[:n] + 1000).astype(np.int64) if with_ids else None
        got = ix.add(torch.from_numpy(b).cuda(), None if ids is None else torch.from_numpy(ids).cuda())
        assert np.array_equal(got.cpu().numpy(), o.add(b, ids)[0])
        _check(ix, o, x, 50)
    assert ix.capacity == o.capacity and ix.max_id == o.max_id
    removed = []
    for sel, by in ((rng.choice(o.address2id[:o.n_items], 60, replace=False), "ids"),
                    (np.arange(o.n_items - 40, o.n_items + 5), "address"),                     # the whole tail
                    (rng.choice(o.n_items, 100, replace=False), "address")):
        removed += list(sel) if by == "ids" else list(o.address2id[sel[sel < o.n_items]])
        t = torch.from_numpy(np.asarray(sel, np.int64)).cuda()
        got = ix.remove(ids=t) if by == "ids" else ix.remove(address=t)
        assert got == (o.remove(ids=sel) if by == "ids" else o.remove(address=sel))
        _, i, _ = _check(ix, o, x, 200)
        assert not np.isin(i.cpu().numpy(), np.asarray(removed)).any()
    adr = rng.choice(o.n_items, 20, replace=False).astype(np.int64)
    new = rng.standard_normal((d, 20)).astype(np.float32)
    ix.set_data_by_address(torch.from_numpy(adr).cuda(), torch.from_numpy(new).cuda())
    o.set_data_by_address(adr, new)
    _check(ix, o, x, 50)                                                 # the norm table follows the store
    live = o.address2id[:o.n_items]
    assert np.array_equal(ix.get_address_by_id(torch.from_numpy(live).cuda()).cpu().numpy(), o.get_address_by_id(live))
    ix.empty()
    o.empty()
    _check(ix, o, x, 5)


@pytest.mark.parametrize("distance", METRICS)
def test_checkpoint_round_trip(cuda_device, distance):
    import torchpq_b200 as T
    rng = np.random.default_rng(3)
    d, n, cap = 20, 700, 1024
    storage = np.zeros((d, cap, 1), np.float32)
    storage[:, :n, 0] = rng.standard_normal((d, n))
    a2i = np.full(cap, -1, np.int64)
    a2i[:n] = rng.permutation(5000)[:n]
    sd = {"_storage": torch.from_numpy(storage).cuda(), "_address2id": torch.from_numpy(a2i).cuda(),
          "_id2address": -torch.ones(1, dtype=torch.long, device="cuda")}     # as the reference saves it
    ix = T.FlatIndex(d, device="cuda:0", distance=distance)
    ix.load_state_dict(sd)
    o = FlatOracle.from_state(storage, a2i, distance=distance)
    assert ix.n_items == n and ix.max_id == o.max_id
    x = rng.standard_normal((d, 33)).astype(np.float32)
    _check(ix, o, x, 64)
    ix2 = T.FlatIndex(d, device="cuda:0", distance=distance)
    ix2.load_state_dict(ix.state_dict())
    _check(ix2, o, x, 64)
    assert ix2.add(torch.zeros(d, 1, device="cuda")).item() == o.max_id + 1


@pytest.mark.parametrize("distance", METRICS)
def test_search_leaves_inputs_and_store_untouched(cuda_device, distance):
    rng = np.random.default_rng(4)
    base = rng.standard_normal((40, 900)).astype(np.float32)
    ix, _ = _pair(base, distance)
    x = torch.from_numpy(rng.standard_normal((40, 77)).astype(np.float32)).cuda()
    x0, s0 = x.clone(), ix._storage.clone()
    ix.search(x, k=10)
    torch.cuda.synchronize()
    assert torch.equal(x.view(torch.int32), x0.view(torch.int32))
    assert torch.equal(ix._storage.view(torch.int32), s0.view(torch.int32))


def test_limits(cuda_device):
    import torchpq_b200 as T
    ix, _ = _pair(np.ones((8, 2000), np.float32), "euclidean")
    with pytest.raises(NotImplementedError):
        ix.search(torch.ones(8, 3, device="cuda"), k=1025)
    for name in ("manhattan", "l1", "nope"):
        with pytest.raises(NotImplementedError):
            T.FlatIndex(8, device="cuda:0", distance=name)
