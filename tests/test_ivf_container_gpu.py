"""GPU: the add / remove / expand life cycle of the IVF container (build.container_add, build.container_remove,
IdContainer's lookups) against the holes-aware oracle (ivf_container_oracle.py), on IVFPQIndex (plain and residual),
IVFPQRIndex, IVFFlatIndex and IVFSQIndex (8 and 16 bits), in both expand modes, from initial sizes 0, 1 and 3.

Seeded sequences add (default ids, fresh explicit ids, ids of removed items), remove by ids (unknown, negative and
duplicate ids included) and by address (holes and out-of-range addresses included), and round-trip the state_dict into
a fresh index part-way.  Items go through build.container_add, the path every index's add ends in, with codes drawn
on the host, into a few cells of which some are never chosen.  After every operation:
  * _address2id, _is_empty, _cell_start, _cell_size, _cell_capacity and the _storage bytes equal the oracle's, and so
    do capacity, n_items and max_id;
  * get_address_by_id on every id ever issued (plus unknown ones) and get_id_by_address on every address (plus
    out-of-range ones) equal the oracle's lookups;
  * search with every cell probed and smart probing off equals the family's exact oracle on the ORACLE's state --
    fp32_exact.search_fp32, ivfpqr_oracle.search, ivfflat_oracle.search (via the decoded store for IVFSQ) -- values as
    bits, ids and addresses; range_search at one finite threshold equals ivfpq_range_oracle / range_oracle.

Every sequence keeps live ids unique.  Among duplicate live ids the inverse id map's scatter keeps an unspecified slot,
a behaviour these tests do not pin.
"""
import numpy as np
import pytest
import torch

import ivf_container_oracle as CO
import ivfpq_range_oracle as PR
import range_oracle as RGO
from oracle import fp32_exact as X, ivfflat_oracle as VO, ivfpq_oracle as O, ivfpqr_oracle as RO, ivfsq_oracle as SO

pytestmark = pytest.mark.gpu

F32 = np.float32
DEV = "cuda:0"
C = 6
CHOSEN, WEIGHTS = [0, 1, 3, 4], [0.4, 0.3, 0.2, 0.1]                 # cells 2 and 5 never receive an item
STEP = 5                                                            # expand_step_size
NQ, K = 3, 10
FAMILIES = ["ivfpq", "ivfpq_residual", "ivfpqr", "ivfflat", "ivfsq8", "ivfsq16"]


@pytest.fixture(autouse=True)
def _on_gpu(cuda_device):
    """Every test here needs the device (skipped without one)."""


def g(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV)


def h(t):
    return t.detach().cpu().numpy()


class Family:
    """One index type: its constructor, the bytes of random items, and its search / range oracles on a container state."""

    def __init__(self, name, mode, seed=0):
        import torchpq_b200 as T
        self.T, self.name, self.mode = T, name, mode
        rng = np.random.default_rng(seed)
        self.rng = rng
        if name.startswith("ivfpq"):
            self.d, self.M = 16, 8
            self.width = 16 if name == "ivfpqr" else 8
            self.vq = rng.standard_normal((self.d, C)).astype(F32)
            self.pq = rng.standard_normal((self.M, self.d // self.M, 256)).astype(F32)
            self.pqr = rng.standard_normal((8, self.d // 8, 256)).astype(F32)
        else:
            self.d = 8
            self.bits = {"ivfflat": 32, "ivfsq8": 8, "ivfsq16": 16}[name]
            self.width = self.d * self.bits // 8
            self.vq = rng.standard_normal((self.d, C)).astype(F32)
            self.sq_train = rng.standard_normal((self.d, 200)).astype(F32) * 2
        self.xq = rng.standard_normal((self.d, NQ)).astype(F32)

    def make(self, initial_size):
        T, kw = self.T, dict(initial_size=initial_size, expand_step_size=STEP, expand_mode=self.mode, device=DEV)
        if self.name in ("ivfpq", "ivfpq_residual"):
            ix = T.IVFPQIndex(self.d, self.M, C, pq_use_residual=self.name == "ivfpq_residual", **kw)
        elif self.name == "ivfpqr":
            ix = T.IVFPQRIndex(self.d, self.M, 8, C, use_residual=True, **kw)
            ix.pq_rerank_codec.set_codebook(g(self.pqr))
        elif self.name == "ivfflat":
            ix = T.IVFFlatIndex(self.d, C, **kw)
        else:
            ix = T.IVFSQIndex(self.d, C, bits=self.bits, **kw)
            ix.sq_codec.train(g(self.sq_train))
        ix.vq_codec.set_codebook(g(self.vq))
        if self.name.startswith("ivfpq"):
            ix.pq_codec.set_codebook(g(self.pq))
        self.settle(ix)
        return ix

    @staticmethod
    def settle(ix):
        ix.n_probe, ix.use_smart_probing = C, False

    def empty_state(self, initial_size):
        if self.name.startswith("ivfpq"):
            return CO.empty(self.width, C, initial_size, d_vector=self.d, n_subvectors=self.M, vq_codebook=self.vq,
                            pq_codebook=self.pq, n_probe=C, use_smart_probing=False)
        return CO.empty(self.width, C, initial_size, d_vector=self.d, vq_codebook=self.vq)

    def codes(self, n):
        """[width, n] u8: random codes (IVFPQ, IVFPQR, 8-bit SQ), or the bytes of normal fp32 / fp16 columns."""
        rng = self.rng
        if self.name.startswith("ivfpq") or self.name == "ivfsq8":
            return rng.integers(0, 256, (self.width, n)).astype(np.uint8)
        if self.name == "ivfflat":
            return VO.codes_of(rng.standard_normal((self.d, n)).astype(F32))
        x = rng.standard_normal((self.d, n)).astype(np.float16)
        return np.ascontiguousarray(x.view(np.uint8).reshape(self.d, n, 2).transpose(0, 2, 1).reshape(self.width, n))

    def storage_bytes(self, ix):
        return h(ix._storage).view(np.uint8).reshape(self.width // 4, ix.capacity, 4)

    # ------------------------------------------------------------------ oracles on the container state
    def flat_state(self, st, ix):
        """The ivfflat_oracle state of a flat-family container: its fp32 columns (IVFSQ: the decoded codes)."""
        cap = st.capacity
        raw = CO.codes_at(st, np.arange(cap))                          # [width, cap], byte j of each slot
        if self.name == "ivfflat":
            x = np.ascontiguousarray(raw.reshape(self.d, 4, cap).transpose(0, 2, 1)).view(F32).reshape(self.d, cap)
        elif self.bits == 8:
            x = SO.decode(raw, 8, *SO.bounds(ix))
        else:
            f16 = np.ascontiguousarray(raw.reshape(self.d, 2, cap).transpose(0, 2, 1)).view(np.float16)
            x = SO.decode(f16.reshape(self.d, cap), 16)
        vs = VO.empty_state(self.d, C, 0, "euclidean", self.vq)
        vs.storage = np.ascontiguousarray(x, F32).view(np.uint8).reshape(self.d, cap, 4)
        for name in ("is_empty", "cell_start", "cell_size", "cell_capacity", "address2id"):
            setattr(vs, name, getattr(st, name).copy())
        vs.max_id = st.max_id
        return vs

    def search(self, st, ix):
        """-> (values, ids, address) [NQ, K]."""
        if self.name in ("ivfpq", "ivfpq_residual"):
            v, a, _ = X.search_fp32(st, self.xq, K, residual=self.name == "ivfpq_residual")
            return v, O.get_id_by_address(st.address2id, a), a
        if self.name == "ivfpqr":
            return RO.search(st, self.xq, K, self.pqr, True, ix.k_factor)[:3]
        return VO.search(self.flat_state(st, ix), self.xq, K, C)

    def range_search(self, st, ix, t):
        if self.name in ("ivfpq", "ivfpq_residual"):
            return PR.range_search_fp32(st, self.xq, t, residual=self.name == "ivfpq_residual")
        return RGO.ivfflat_range_search(self.flat_state(st, ix), self.xq, t, C)


def same_search(got, want):
    v, i, a = (h(t) for t in got)
    assert np.array_equal(v.view(np.uint32), np.asarray(want[0], F32).view(np.uint32)), "search values differ"
    assert np.array_equal(i, want[1]), "search ids differ"
    assert np.array_equal(a, want[2]), "search addresses differ"


def check(fam, ix, st, issued):
    """Every buffer, count and lookup of the index equals the oracle's, and so do search and range_search."""
    for name in ("address2id", "is_empty", "cell_start", "cell_size", "cell_capacity"):
        assert np.array_equal(h(getattr(ix, "_" + name)), getattr(st, name)), name
    assert np.array_equal(fam.storage_bytes(ix), st.storage), "_storage"
    assert ix.capacity == st.capacity and ix.max_id == st.max_id
    assert ix.n_items == int((st.is_empty == 0).sum())
    top = max(issued) if issued else 0
    ids = np.array(sorted(issued) + [-1, -9, top + 1, top + 77], np.int64)
    assert np.array_equal(h(ix.get_address_by_id(g(ids))), CO.get_address_by_id(st, ids)), "get_address_by_id"
    adr = np.arange(-2, st.capacity + 3, dtype=np.int64)
    assert np.array_equal(h(ix.get_id_by_address(g(adr))), CO.get_id_by_address(st, adr)), "get_id_by_address"
    if st.capacity == 0:                                                # nothing to search yet
        return
    want = fam.search(st, ix)
    same_search(ix.search(g(fam.xq), k=K, return_address=True), want)
    if fam.name == "ivfpqr":                                            # no range search: its scores are not re-ranked
        return
    finite = want[0][:, K // 2][np.isfinite(want[0][:, K // 2])]
    t = float(np.median(finite)) if finite.size else 0.0
    lims, v, i, a = (h(x) for x in ix.range_search(g(fam.xq), t, return_address=True))
    wl, wv, wi, wa = fam.range_search(st, ix, t)
    assert lims.tolist() == wl.tolist(), "range_search lims"
    assert np.array_equal(v.view(np.uint32), wv.view(np.uint32)), "range_search values"
    assert np.array_equal(i, wi) and np.array_equal(a, wa), "range_search ids / addresses"


def add(fam, ix, st, n, ids=None, cells=None):
    from torchpq_b200 import build
    cells = fam.rng.choice(CHOSEN, n, p=WEIGHTS) if cells is None else np.asarray(cells, np.int64)
    codes = fam.codes(n)
    want_ids, want_adr = CO.add(st, codes, cells, ids, expand_mode=fam.mode, expand_step_size=STEP)
    got_ids, got_adr = build.container_add(ix, g(codes), g(cells), None if ids is None else g(ids), return_address=True)
    assert np.array_equal(h(got_ids), want_ids) and np.array_equal(h(got_adr), want_adr), "ids / write addresses"
    return want_ids


def hole_cells(fam, st, n):
    """Up to n cells, one per hole below a cell's high-water mark, shuffled: an add of them needs no expansion."""
    out = []
    for c in range(C):
        s = int(st.cell_start[c])
        out += [c] * int((st.is_empty[s:s + int(st.cell_size[c])] != 0).sum())
    out = np.asarray(out[:n] if len(out) <= n else fam.rng.choice(out, n, replace=False), np.int64)
    fam.rng.shuffle(out)
    return out


def fresh_copy(fam, ix):
    """ix's state_dict loaded into a fresh index of another initial size (the load replaces every buffer)."""
    fresh = fam.make(2)
    fresh.load_state_dict({k: v.clone() for k, v in ix.state_dict().items()})
    fam.settle(fresh)
    return fresh


def round_trip(fam, ix, st):
    return fresh_copy(fam, ix), CO.load(st)


def same_as_rebuilt(fam, ix):
    """The scan layout that an in-place add updated searches exactly as one built from scratch by a fresh index."""
    fresh = fresh_copy(fam, ix)
    a = ix.search(g(fam.xq), k=K, return_address=True)
    b = fresh.search(g(fam.xq), k=K, return_address=True)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


@pytest.mark.parametrize("initial_size", [0, 1, 3])
@pytest.mark.parametrize("mode", ["step", "double"])
@pytest.mark.parametrize("family", FAMILIES)
def test_life_cycle_matches_oracle(family, mode, initial_size):
    fam = Family(family, mode, seed=FAMILIES.index(family) * 10 + initial_size + (mode == "step") * 100)
    rng = fam.rng
    ix, st = fam.make(initial_size), fam.empty_state(initial_size)
    issued, removed = set(), []
    check(fam, ix, st, issued)

    def added(ids):
        issued.update(ids.tolist())
        removed[:] = [r for r in removed if r not in set(ids.tolist())]

    def remove_ids(frac, extra):
        live = np.sort(st.address2id[st.is_empty == 0])
        pick = rng.choice(live, int(frac * live.size), replace=False)
        ids = np.concatenate([pick, pick[:3], extra]).astype(np.int64)
        rng.shuffle(ids)
        gone = CO.remove(st, ids=ids)
        ix.remove(ids=g(ids))
        removed.extend(sorted(set(pick.tolist())))
        assert gone.size == pick.size

    added(add(fam, ix, st, int(rng.integers(60, 200))))                 # default ids
    check(fam, ix, st, issued)
    n = int(rng.integers(50, 150))
    added(add(fam, ix, st, n, ids=max(issued) + 1 + rng.choice(3 * n, n, replace=False)))   # fresh explicit ids
    check(fam, ix, st, issued)
    remove_ids(0.3, [-1, -4, max(issued) + 50])
    check(fam, ix, st, issued)
    reuse = np.asarray(removed[: len(removed) // 2], np.int64)
    cells = hole_cells(fam, st, reuse.size)                             # into holes: no expansion
    lay = ix._layout if family.startswith("ivfpq") else None
    added(add(fam, ix, st, cells.size, ids=reuse[: cells.size], cells=cells))
    if lay is not None:
        assert ix._layout is lay, "the add into holes rebuilt the scan layout"
    check(fam, ix, st, issued)
    if lay is not None:
        same_as_rebuilt(fam, ix)
    live = np.flatnonzero(st.is_empty == 0)
    holes = np.flatnonzero(st.is_empty != 0)
    adr = np.concatenate([rng.choice(live, live.size // 4, replace=False), holes[:5], live[:2],
                          [-1, st.capacity, st.capacity + 5]]).astype(np.int64)
    held = st.address2id.copy()
    gone = CO.remove(st, address=adr)
    removed.extend(held[gone].tolist())
    ix.remove(address=g(adr))
    check(fam, ix, st, issued)
    ix, st = round_trip(fam, ix, st)
    check(fam, ix, st, issued)
    added(add(fam, ix, st, int(rng.integers(100, 250))))                # default ids after the load: from max(address2id)
    check(fam, ix, st, issued)
    if removed:
        added(add(fam, ix, st, len(removed), ids=np.asarray(removed, np.int64)))   # reused ids, anywhere
        check(fam, ix, st, issued)
    remove_ids(0.2, [-2, max(issued) + 1, max(issued) + 1000])
    check(fam, ix, st, issued)
    added(add(fam, ix, st, int(rng.integers(20, 60))))
    check(fam, ix, st, issued)


# ----------------------------------------------------------------------------------------- named regressions
def _stale_map_setup(family):
    """20 items, 5 in each of cells 0..3 (capacity 8: no expansion); ids 2, 7, 11, 16 removed; the inverse map then
    built.  -> (family, index, oracle state, ids, cells of the items)."""
    fam = Family(family, "double", seed=5)
    ix, st = fam.make(8), fam.empty_state(8)
    cells = np.arange(20) % 4
    add(fam, ix, st, 20, cells=cells)
    R = np.array([2, 7, 11, 16], np.int64)
    ix.remove(ids=g(R))
    CO.remove(st, ids=R)
    ix.get_address_by_id(g(np.arange(20)))                              # builds the inverse map after the remove
    return fam, ix, st, R, cells


@pytest.mark.parametrize("family", ["ivfpq", "ivfflat"])
def test_stale_map_explicit_ids(family):
    """Ids re-added into holes by an add that moves no buffer: the lookup must find them and remove(ids=) must remove
    exactly their slots (the kernel writes _address2id through its raw pointer, unseen by its _version)."""
    fam, ix, st, R, cells = _stale_map_setup(family)
    from torchpq_b200 import build
    codes = fam.codes(R.size)
    _, want = CO.add(st, codes, cells[R], R, expand_mode="double", expand_step_size=STEP)
    _, adr = build.container_add(ix, g(codes), g(cells[R]), g(R), return_address=True)
    assert h(adr).tolist() == want.tolist()
    got = h(ix.get_address_by_id(g(R)))
    assert got.tolist() == want.tolist(), f"get_address_by_id(R) = {got.tolist()}, the ids were re-added at {want.tolist()}"
    n = ix.n_items
    ix.remove(ids=g(R))
    assert ix.n_items == n - R.size, f"remove(ids=R) removed {n - ix.n_items} items, not {R.size}"
    assert (h(ix._is_empty)[want] == 1).all()


@pytest.mark.parametrize("family", ["ivfpq", "ivfflat"])
def test_stale_map_default_ids(family):
    """The same with default ids, which lie past the end of the map built before the add."""
    fam, ix, st, R, cells = _stale_map_setup(family)
    new = add(fam, ix, st, R.size, cells=cells[R])
    assert new.tolist() == [20, 21, 22, 23]
    assert np.array_equal(h(ix.get_address_by_id(g(new))), CO.get_address_by_id(st, new))
    check(fam, ix, st, set(range(24)))


@pytest.mark.parametrize("mode", ["step", "double"])
@pytest.mark.parametrize("family", ["ivfpq", "ivfflat"])
def test_zero_capacity_add(family, mode):
    """initial_size=0: every first add into a cell grows it from capacity 0, in both modes."""
    fam = Family(family, mode, seed=9)
    ix, st = fam.make(0), fam.empty_state(0)
    issued = set(add(fam, ix, st, 7, cells=[1, 1, 4, 1, 0, 4, 1]).tolist())
    assert st.cell_capacity.tolist() == [STEP, STEP, 0, 0, STEP, 0]
    check(fam, ix, st, issued)
    issued |= set(add(fam, ix, st, 8, cells=[1] * 8).tolist())         # 12 items: 5 -> 10 -> 20, or 5 -> 10 -> 15
    assert st.cell_capacity[1] == (4 * STEP if mode == "double" else 3 * STEP)
    check(fam, ix, st, issued)


@pytest.mark.parametrize("mode", ["step", "double"])
@pytest.mark.parametrize("family", ["ivfpq_residual", "ivfsq8"])
def test_loaded_state_with_zero_capacity_cells(family, mode):
    """A checkpoint whose cells other than 0 and 3 have capacity 0, loaded into an index of another initial size: adds
    into those cells grow them from 0."""
    fam = Family(family, mode, seed=11)
    ix, st = fam.make(0), fam.empty_state(0)
    issued = set(add(fam, ix, st, 30, cells=np.arange(30) % 2 * 3).tolist())
    ix, st = round_trip(fam, ix, st)
    zero = [c for c in range(C) if st.cell_capacity[c] == 0]
    assert zero == [1, 2, 4, 5]
    check(fam, ix, st, issued)
    issued |= set(add(fam, ix, st, 3 * STEP + 1, cells=np.resize(zero, 3 * STEP + 1)).tolist())
    assert all(st.cell_capacity[c] > 0 for c in zero)
    check(fam, ix, st, issued)


@pytest.mark.parametrize("mode", ["step", "double"])
@pytest.mark.parametrize("family", ["ivfpq", "ivfflat"])
def test_empty_checkpoint_then_add(family, mode):
    """The checkpoint of an index of capacity 0 (initial_size=0, nothing added) loads, and adds into it grow every
    cell from 0 (a loaded index assumes holes: the add must not look for them in a store without a slot)."""
    fam = Family(family, mode, seed=13)
    ix, st = round_trip(fam, fam.make(0), fam.empty_state(0))
    assert ix.capacity == 0 and ix._has_holes
    check(fam, ix, st, set())
    issued = set(add(fam, ix, st, 12).tolist())
    check(fam, ix, st, issued)
