"""CPU: tpq_refine_flat's argument errors (returned before any launch), RefineFlatIndex's constructor, entry points,
checkpoint keys and store life cycle on a CPU FlatIndex base (no kernel runs there), the shared k1 rule, and the refine
oracle against a float64 evaluation and against itself."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fp32_exact as E
from oracle import ivfpqr_oracle as R
from oracle import refine_oracle as RF

FAKE = C.c_void_p(0x1000)                 # a non-null pointer that is never dereferenced: every case fails its checks


def _refine(lib, d=32, nq=2, k1=8, n=100, metric=0, k=4, ptrs=None, ws=None, ws_bytes=0):
    p = ptrs
    return lib.tpq_refine_flat(p, d, nq, p, k1, p, n, metric, k, p, p, p, p, ws, ws_bytes, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(metric=2), "unsupported metric"),
    (dict(metric=3), "unsupported metric"),
    (dict(k=0), "0 < k <= k1 <= 1024"),
    (dict(k=9, k1=8), "0 < k <= k1 <= 1024"),
    (dict(k=4, k1=1025), "0 < k <= k1 <= 1024"),
    (dict(k=-1, k1=8), "0 < k <= k1 <= 1024"),
    (dict(n=1 << 32), "bad sizes"),
    (dict(n=-1), "bad sizes"),
    (dict(d=0), "bad sizes"),
    (dict(nq=-1), "bad sizes"),
    (dict(), "null pointer"),
    (dict(n=0), "null pointer"),                  # vectors may be NULL with n == 0, the other pointers may not
])
def test_refine_argument_errors(kw, msg):
    import torchpq_b200 as T
    rc = _refine(T._lib.lib, **kw)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and msg in T._lib.last_error()


@pytest.mark.parametrize("ws_bytes", [0, 1, None])
def test_refine_workspace_too_small(ws_bytes):
    import torchpq_b200 as T
    lib = T._lib.lib
    need = lib.tpq_refine_flat_workspace_bytes(32, 2, 4)
    ws_bytes = need - 1 if ws_bytes is None else ws_bytes
    rc = _refine(lib, ptrs=FAKE, ws=FAKE if ws_bytes else None, ws_bytes=ws_bytes)
    assert rc == T._lib.TPQ_ERR_WORKSPACE and "workspace too small" in T._lib.last_error()


def test_refine_shared_memory_limit():
    import torchpq_b200 as T
    lib = T._lib.lib
    d = 1 << 16                                                       # one query's x alone is 256 KB
    rc = _refine(lib, d=d, ptrs=FAKE, ws=FAKE, ws_bytes=lib.tpq_refine_flat_workspace_bytes(d, 2, 4))
    assert rc == T._lib.TPQ_ERR_UNSUPPORTED and "shared memory" in T._lib.last_error()


def test_refine_empty_batch_returns_at_once():
    import torchpq_b200 as T
    lib = T._lib.lib
    assert _refine(lib, nq=0) == T._lib.TPQ_OK
    assert lib.tpq_refine_flat_workspace_bytes(32, 0, 4) == 0
    assert lib.tpq_refine_flat_workspace_bytes(32, 10, 4) == 512 + 1280


def test_k1_rule_is_the_oracles():
    from torchpq_b200.modules import k1_of
    for k in (1, 2, 3, 7, 100, 255, 256, 512, 1000, 1024):
        for kf in (0.5, 1, 1.5, 2, 4, 8, 2.7):
            assert k1_of(k, kf) == R.k1_of(k, kf)


def cpu_base(distance="euclidean", d=8):
    import torchpq_b200 as T
    return T.FlatIndex(d, initial_size=2, expand_step_size=2, distance=distance, device="cpu")


@pytest.mark.parametrize("distance", ["inner", "dot"])
def test_unsupported_distance_raises(distance):
    import torchpq_b200 as T
    with pytest.raises(NotImplementedError):
        T.RefineFlatIndex(cpu_base(distance))
    ix = T.IVFFlatIndex(8, 4, initial_size=2, device="cpu")
    ix.distance = distance                                            # any base: the check reads base.distance
    with pytest.raises(NotImplementedError):
        T.RefineFlatIndex(ix)


def test_constructor_attributes_and_state_dict_keys():
    import torchpq_b200 as T
    base = cpu_base("cosine")
    ix = T.RefineFlatIndex(base, k_factor=2)
    assert (ix.d_vector, ix.distance, ix.k_factor, ix.n_items, ix.capacity) == (8, "cosine", 2, 0, 0)
    assert ix.base_index is base and dict(ix.named_children())["base_index"] is base
    assert ix._vectors.shape == (0, 8) and ix._vectors.dtype == torch.float32
    assert {"_address2id", "_vectors", "base_index._address2id", "base_index._storage"} <= set(ix.state_dict())


def test_entry_points_are_wrapped_for_the_device():
    import torchpq_b200 as T
    for name in ("train", "add", "remove", "search", "refine"):
        assert hasattr(getattr(T.RefineFlatIndex, name), "__wrapped__"), name


def test_life_cycle_on_a_cpu_flat_base():
    """add / remove / growth keep the store a prefix, each id's row what was added, and both indexes in step."""
    import torchpq_b200 as T
    rng = np.random.default_rng(0)
    base = cpu_base()
    ix = T.RefineFlatIndex(base)
    rows = {}
    for step in range(12):
        n = int(rng.integers(0, 6))
        x = torch.from_numpy(rng.standard_normal((8, n)).astype(np.float32))
        if step % 3 == 2:
            ids = ix.add(x)
        else:
            ids = torch.from_numpy(rng.choice(10_000, n, replace=False) + 10_000 * (step + 1)).long()
            assert torch.equal(ix.add(x, ids), ids)
        rows.update({int(i): x[:, j] for j, i in enumerate(ids.tolist())})
        if step % 2 and rows:
            gone = rng.choice(sorted(rows), min(len(rows), 3), replace=False).tolist()
            assert ix.remove(torch.tensor(gone + [-1, 987654321])) == len(gone)
            for i in gone:
                del rows[i]
        assert ix.n_items == len(rows) == base.n_items
        assert ix.capacity >= ix.n_items and ix.capacity & (ix.capacity - 1) == 0 or ix.capacity == 0
        live = ix._address2id[:ix.n_items]
        assert bool((live >= 0).all()) and bool((ix._address2id[ix.n_items:] == -1).all())
        assert bool((ix._vectors[ix.n_items:] == 0).all())
        for a, i in enumerate(live.tolist()):
            assert torch.equal(ix._vectors[a], rows[i])
        assert torch.equal(ix._addresses_of(live), torch.arange(ix.n_items))


def test_duplicate_ids_raise_before_either_index_changes():
    import torchpq_b200 as T
    base = cpu_base()
    ix = T.RefineFlatIndex(base)
    ix.add(torch.ones(8, 3), torch.tensor([5, 6, 7]))
    before = {k: v.clone() for k, v in ix.state_dict().items()}
    for ids in (torch.tensor([1, 2, 1]), torch.tensor([8, 6, 9]), torch.tensor([1, -3, 2])):
        with pytest.raises(ValueError):
            ix.add(torch.zeros(8, 3), ids)
        after = ix.state_dict()
        assert set(after) == set(before) and all(torch.equal(after[k], v) for k, v in before.items())
        assert ix.n_items == base.n_items == 3


def test_state_dict_round_trip_rebuilds_the_id_map():
    import torchpq_b200 as T
    ix = T.RefineFlatIndex(cpu_base())
    ix.add(torch.randn(8, 5), torch.tensor([40, 3, 17, 8, 21]))
    ix.remove(torch.tensor([3]))
    ix2 = T.RefineFlatIndex(cpu_base())
    ix2.load_state_dict(ix.state_dict())
    assert ix2.n_items == ix2.base_index.n_items == 4 and ix2.max_id == 40
    ids = torch.tensor([40, 3, 17, 8, 21, -1, 99])
    assert torch.equal(ix2._addresses_of(ids), ix._addresses_of(ids))
    assert torch.equal(ix2._vectors, ix._vectors)


# ----------------------------------------------------------------------------------------- the oracle
def _store(n, d, rng, distance="euclidean"):
    v = rng.standard_normal((n + 3, d)).astype(np.float32)
    if distance == "cosine":
        v = E.normalize_columns(v.T).T.copy()
    a2i = -np.ones(n + 3, np.int64)
    a2i[:n] = rng.permutation(10 * n)[:n]
    v[n:] = 0
    return v, a2i


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_oracle_batched_scores_equal_the_per_query_chain(distance):
    rng = np.random.default_rng(1)
    d, n, nq, k1 = 13, 40, 5, 9
    v, a2i = _store(n, d, rng, distance)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    addr = rng.integers(0, n, size=(nq, k1))
    got = RF.score_addresses(x, addr, v, distance)
    xs = E.normalize_columns(x) if distance == "cosine" else x
    for q in range(nq):
        assert np.array_equal(got[q], R.scores(xs[:, q], v[addr[q]].T, distance))


@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_oracle_against_float64(distance):
    rng = np.random.default_rng(2)
    d, n, nq, k = 24, 60, 4, 7
    v, a2i = _store(n, d, rng, distance)
    x = rng.standard_normal((d, nq)).astype(np.float32)
    live = a2i[:n]
    cand = np.stack([rng.permutation(live)[:20] for _ in range(nq)])
    cand[1, 9:] = -1                                                  # -1 is dropped
    cand[2, 3:] = 123456                                              # so is an id the store does not hold
    vals, ids, adr = RF.refine(x, cand, v, a2i, n, distance, k)
    x64 = x.astype(np.float64)
    if distance == "cosine":
        x64 = x64 / (np.linalg.norm(x64, axis=0) + 1e-9)
    for q in range(nq):
        c = [a for a in (np.flatnonzero(a2i[:n] == i) for i in cand[q]) if a.size]
        a = np.array([int(t[0]) for t in c], np.int64)
        y = v[a].astype(np.float64).T
        s = -((x64[:, q:q + 1] - y) ** 2).sum(0) if distance == "euclidean" else (x64[:, q:q + 1] * y).sum(0)
        m = min(k, a.shape[0])
        assert np.allclose(vals[q, :m], np.sort(s)[::-1][:m], rtol=1e-5, atol=1e-4)
        assert np.array_equal(ids[q, :m], a2i[adr[q, :m]])
        assert np.all(adr[q, m:] == -1) and np.all(ids[q, m:] == -1) and np.all(np.isneginf(vals[q, m:]))
        assert np.all(np.diff(vals[q, :m]) <= 0)


def test_oracle_duplicates_ties_and_brute_force():
    rng = np.random.default_rng(3)
    d, n = 6, 10
    v, a2i = _store(n, d, rng)
    v[7] = v[2]                                                       # the same vector under two ids
    x = rng.standard_normal((d, 1)).astype(np.float32)
    x[:, 0] = v[2]                                                    # ... and the query itself: both score -0 / +0
    i2, i7 = a2i[2], a2i[7]
    vals, ids, adr = RF.refine(x, np.array([[i7, i2, i7, -1]]), v, a2i, n, "euclidean", 4)
    assert adr[0].tolist() == [2, 7, 7, -1]                           # tie to the lower address; i7 listed twice
    assert ids[0].tolist() == [i2, i7, i7, -1]
    bv, bi, ba = RF.brute_force(x, n + 2, v, a2i, n, "euclidean")
    assert ba[0, :2].tolist() == [2, 7] and np.all(ba[0, n:] == -1)
    assert sorted(ba[0, :n].tolist()) == list(range(n))
    all_ids = np.broadcast_to(a2i[:n], (1, n))
    assert all(np.array_equal(a, b) for a, b in zip(RF.refine(x, all_ids, v, a2i, n, "euclidean", 5),
                                                    RF.brute_force(x, 5, v, a2i, n, "euclidean")))
    ev, ei, ea = RF.brute_force(x, 3, v, a2i, 0, "euclidean")         # an empty store
    assert np.all(np.isneginf(ev)) and np.all(ei == -1) and np.all(ea == -1)


def test_train_on_a_flat_base_trains_nothing():
    import torchpq_b200 as T
    ix = T.RefineFlatIndex(cpu_base())
    ix.train(torch.randn(8, 10))                                      # FlatIndex.train is nn.Module's (mode: bool)
    assert ix.base_index.training and ix.n_items == 0
