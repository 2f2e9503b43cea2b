"""numpy restatement of the reference's FlatIndex (TEST INFRASTRUCTURE, see ``oracle/__init__.py``).

``FlatOracle`` restates the container of ``torchpq.index.FlatIndex`` (container/FlatContainer.py, BaseContainer.py):
add at [n_items, n_items + n), expand ("double" doubles the step first), the compacting remove, the id/address maps and
empty -- with the reference's bookkeeping defects fixed as ``torchpq_b200.FlatIndex`` fixes them: ``max_id`` advances
with every add (the reference never advances it) and ``n_items`` / ``max_id`` are re-derived from ``address2id`` when
a state is loaded.  ``search`` restates ``FlatIndex.search`` over the live slots only, in the kernel's own arithmetic
(``flat_sims``, built on the restatements of ``fp32_exact``) and total order (score descending, address ascending;
``fp32_exact.probe_select``), padded with (-inf, id -1, address -1).
"""
from __future__ import annotations

import numpy as np

from . import fp32_exact as X

F32 = np.float32
EPS = F32(1e-8)                  # metric.cosine_similarity's `+ 1e-8` (metric.py:14-25), kFlatEps of flat.cu


def col_norm(x):
    """col_norm_kernel (coarse.cu) with eps 1e-8: sqrtf(sum_i fmaf chain of x^2, in col_sumsq's row groups) + 1e-8."""
    return (np.sqrt(X._col_groups(np.asarray(x, F32), fused=True)) + EPS).astype(F32)


def normalize_columns(x):
    """normalize_columns_kernel (coarse.cu) with eps 1e-8: x / col_norm(x), __fdiv_rn."""
    x = np.asarray(x, F32)
    return (x / col_norm(x)[None, :]).astype(F32)


def flat_sims(x, base, distance):
    """The scores of flat_search_kernel (flat.cu), x [d, nq], base [d, n] -> [nq, n]; acc = fmaf chain over i ascending
    from +0 as in fp32_exact.coarse_sims.  euclidean: coarse_sims ((acc * 2 - |x|^2) - |b|^2); cosine:
    acc(normalize_columns(x), b) / col_norm(b) (__fdiv_rn); inner: acc(x, b)."""
    x, base = np.asarray(x, F32), np.asarray(base, F32)
    if distance == "euclidean":
        return X.coarse_sims(x, base)
    if distance == "cosine":
        acc = X.fma_chain(normalize_columns(x)[:, :, None], base[:, None, :])
        return (acc / col_norm(base)[None, :]).astype(F32)
    assert distance == "inner", distance
    return X.fma_chain(x[:, :, None], base[:, None, :])


class FlatOracle:
    def __init__(self, d_vector, initial_size=None, expand_step_size=1024, expand_mode="double", distance="euclidean"):
        self.d_vector, self.distance = d_vector, distance
        self.expand_step_size, self.expand_mode = expand_step_size, expand_mode
        cap = expand_step_size if initial_size is None else initial_size
        self.storage = np.zeros((d_vector, cap), F32)
        self.address2id = np.full(cap, -1, np.int64)
        self.n_items, self.max_id = 0, -1

    @property
    def capacity(self):
        return self.address2id.shape[0]

    @classmethod
    def from_state(cls, storage, address2id, **kw):
        """A loaded state: n_items = the count of address2id >= 0 (a prefix), max_id = max(address2id)."""
        o = cls(storage.shape[0], initial_size=0, **kw)
        o.storage = np.asarray(storage, F32).reshape(storage.shape[0], -1).copy()
        o.address2id = np.asarray(address2id, np.int64).copy()
        o.n_items = int((o.address2id >= 0).sum())
        assert (o.address2id[:o.n_items] >= 0).all()
        o.max_id = int(o.address2id.max()) if o.address2id.size else -1
        return o

    def expand(self):
        if self.expand_mode == "double":
            self.expand_step_size *= 2
        n = self.expand_step_size
        self.storage = np.concatenate([self.storage, np.zeros((self.d_vector, n), F32)], axis=1)
        self.address2id = np.concatenate([self.address2id, np.full(n, -1, np.int64)])

    def add(self, x, ids=None):
        x = np.asarray(x, F32)
        n = x.shape[1]
        ids = np.arange(n, dtype=np.int64) + self.max_id + 1 if ids is None else np.asarray(ids, np.int64)
        while self.capacity - self.n_items < n:
            self.expand()
        adr = np.arange(n, dtype=np.int64) + self.n_items
        self.storage[:, adr] = x
        self.address2id[adr] = ids
        self.n_items += n
        if n:
            self.max_id = max(self.max_id, int(ids.max()))
        return ids, adr

    def get_address_by_id(self, ids):
        ids = np.asarray(ids, np.int64)
        out = np.full(ids.shape, -1, np.int64)
        for i, v in enumerate(ids):
            hit = np.nonzero(self.address2id == v)[0] if v >= 0 else []
            if len(hit):
                out[i] = hit[0]
        return out

    def get_id_by_address(self, address):
        address = np.asarray(address, np.int64)
        ok = (address >= 0) & (address < self.capacity)
        return np.where(ok, self.address2id[np.where(ok, address, 0)], -1)

    def get_data_by_address(self, address):
        address = np.asarray(address, np.int64)
        ok = (address >= 0) & (address < self.capacity)
        return np.where(ok[None, :], self.storage[:, np.where(ok, address, 0)], F32(0))

    def set_data_by_address(self, address, data):
        address = np.asarray(address, np.int64)
        ok = (address >= 0) & (address < self.capacity)
        self.storage[:, address[ok]] = np.asarray(data, F32)[:, ok]

    def remove(self, ids=None, address=None):
        """FlatContainer.remove (FlatContainer.py:160-190) over the live prefix: the surviving items of the last
        n_removed slots fill the removed slots below them, in ascending order."""
        address = self.get_address_by_id(ids) if ids is not None else np.asarray(address, np.int64)
        address = np.unique(address[(address >= 0) & (address < self.n_items)])
        r = address.shape[0]
        if r == 0:
            return 0
        self.address2id[address] = -1
        tail = np.arange(self.n_items - r, self.n_items)
        keep = tail[self.address2id[tail] != -1]
        dst = address[:keep.shape[0]]
        self.storage[:, dst] = self.storage[:, keep]
        self.address2id[dst] = self.address2id[keep]
        self.storage[:, tail] = 0
        self.address2id[tail] = -1
        self.n_items -= r
        return r

    def empty(self):
        self.storage[:] = 0
        self.address2id[:] = -1
        self.n_items = 0

    def search(self, x, k):
        """-> (values [nq, k] f32, ids [nq, k] i64, address [nq, k] i64)."""
        x = np.asarray(x, F32)
        nq, n = x.shape[1], self.n_items
        vals = np.full((nq, k), -np.inf, F32)
        adr = np.full((nq, k), -1, np.int64)
        if n and nq:
            sims = flat_sims(x, self.storage[:, :n], self.distance)
            v, a = X.probe_select(sims, min(k, n))
            vals[:, :v.shape[1]], adr[:, :a.shape[1]] = v, a
        ids = np.where(adr >= 0, self.address2id[np.maximum(adr, 0)], -1)
        return vals, ids, adr
