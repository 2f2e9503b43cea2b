"""RefineFlatIndex: any index of this package, its candidates re-ranked exactly on stored fp32 vectors (Faiss:
``IndexRefineFlat``): FlatIndex, IVFPQIndex, IVFPQRIndex, IVFFlatIndex, IVFSQIndex or IVFPQ4Index.

``search(x, k)`` asks the base index for k1 = min(1024, max(k, ceil(k_factor * k))) candidate ids per query, maps each
to its row of a row-major fp32 store through the id map, scores it exactly (``tpq_refine_flat``, csrc/refine.cu) and
keeps the k best.  A value equals ``fn.max_sim(x_q, stored vector)`` bit for bit: euclidean -||x - y||^2 as one fmaf
chain, cosine <x / (|x| + 1e-9), y> with y stored normalised.  Ties go to the lower store address.

The store keeps its live slots as the prefix [0, n_items): ``add`` appends, ``remove`` compacts by FlatIndex.remove's
rule, the capacity doubles when full.  ``add``, ``remove`` and ``load_state_dict`` rebuild the id map; ``search`` and
``refine`` only read it, so neither synchronises the host and a search can be captured in a CUDA graph.
Not covered: ``range_search`` and ``search_cells`` (Faiss's ``IndexRefine`` has neither), and multi-GPU.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .flat_index import FlatIndex
from .modules import IdContainer, k1_of, live_prefix, on_index_device, prefix_remove


class RefineFlatIndex(IdContainer):
    def __init__(self, base_index, k_factor=4):
        super().__init__()
        if base_index.distance not in ("euclidean", "cosine"):
            raise NotImplementedError(f"RefineFlatIndex supports euclidean and cosine, not {base_index.distance}")
        self.base_index = base_index                                     # a submodule: state_dict carries base_index.*
        self.d_vector, self.distance, self.k_factor = base_index.d_vector, base_index.distance, k_factor
        dev = base_index._address2id.device
        self.device = dev
        self._max_id = -1
        self._n_items = 0
        self._id2address_fp = None
        self.register_buffer("_address2id", -torch.ones(0, dtype=torch.long, device=dev))
        self.register_buffer("_id2address", None)
        self.register_buffer("_vectors", torch.zeros(0, self.d_vector, dtype=torch.float32, device=dev))

    @property
    def n_items(self):
        return self._n_items

    # ------------------------------------------------------------------ id map
    def _rebuild_id_map(self):
        """Rebuild ``_id2address`` from ``_address2id`` now (host-synchronising), so that searches only read it."""
        self._ids_changed()
        self.get_address_by_id(torch.empty(0, dtype=torch.long, device=self._address2id.device))

    def _addresses_of(self, ids):
        """Store address of each id, -1 for -1 and for ids the store does not hold; tensor ops only, no host sync."""
        id2a = self._id2address
        if id2a is None or id2a.shape[0] == 0:
            return torch.full_like(ids, -1)
        m = id2a.shape[0]
        return torch.where((ids >= 0) & (ids < m), id2a[ids.clamp(0, m - 1)], -1)

    def load_state_dict(self, state_dict, strict=True):
        """The buffers and the base index's state, then ``n_items`` = the live slots, which must be a prefix of the
        store (FlatIndex's check), ``max_id`` and the id map."""
        super().load_state_dict(state_dict, strict)
        n = live_prefix(self._address2id)
        assert self._vectors.shape == (self.capacity, self.d_vector)
        self._n_items = n
        self._refresh_max_id()
        self._rebuild_id_map()

    # ------------------------------------------------------------------ build side
    @on_index_device
    def train(self, x, *args, **kwargs):
        """The base index's train.  A FlatIndex base has nothing to train (its ``train`` is nn.Module's)."""
        if not isinstance(self.base_index, FlatIndex):
            self.base_index.train(x, *args, **kwargs)

    def _grow(self, n):
        """Double the capacity until n more items fit."""
        cap = self.capacity
        if cap >= self._n_items + n:
            return
        new = max(1, cap)
        while new < self._n_items + n:
            new *= 2
        dev = self._address2id.device
        a2i = torch.cat([self._address2id, -torch.ones(new - cap, dtype=torch.long, device=dev)])
        vec = torch.cat([self._vectors, torch.zeros(new - cap, self.d_vector, dtype=torch.float32, device=dev)])
        for name, t in (("_address2id", a2i), ("_vectors", vec)):
            delattr(self, name)
            self.register_buffer(name, t)

    @on_index_device
    def add(self, x, ids=None, return_address=False):
        """x [d_vector, n] fp32 into the base index and the refine store, under `ids` (default: continuing after the
        larger max_id of the two).  A repeated, negative or already stored id raises ValueError before either index
        changes.  -> ids[, addresses in the refine store]."""
        assert x.dtype == torch.float32 and x.dim() == 2 and x.shape[0] == self.d_vector
        dev = self._vectors.device
        x, n = x.to(dev), x.shape[1]
        if ids is None:
            ids = torch.arange(n, dtype=torch.long, device=dev) + max(self._max_id, self.base_index.max_id) + 1
        else:
            assert ids.dtype == torch.int64 and ids.shape == (n,)
            ids = ids.to(dev)
        if n:
            if bool((ids < 0).any().item()):
                raise ValueError("RefineFlatIndex.add: ids must be non-negative")
            if ids.unique().shape[0] != n:
                raise ValueError("RefineFlatIndex.add: an id is repeated in the batch")
            if bool((self._addresses_of(ids) >= 0).any().item()):
                raise ValueError("RefineFlatIndex.add: an id is already in the store")
        ids = self.base_index.add(x, ids)
        if n:
            from . import fn
            self._grow(n)
            a0 = self._n_items
            self._vectors[a0:a0 + n] = (fn.normalize(x) if self.distance == "cosine" else x).t()
            self._address2id[a0:a0 + n] = ids
            self._n_items += n
            self._max_id = max(self._max_id, int(ids.max().item()))
        self._rebuild_id_map()
        address = torch.arange(n, dtype=torch.long, device=dev) + self._n_items - n
        return (ids, address) if return_address else ids

    @on_index_device
    def remove(self, ids):
        """Remove `ids` from the base index and the store (FlatIndex.remove's compaction); unknown ids are ignored.
        -> the number removed from the store."""
        assert ids.dtype == torch.int64
        ids = ids.to(self._address2id.device)
        self.base_index.remove(ids=ids)
        n_removed, dst, src, tail = prefix_remove(self._address2id, self._addresses_of(ids), self._n_items)
        if n_removed:
            self._vectors[dst] = self._vectors[src].clone()
            self._vectors[tail] = 0
            self._n_items -= n_removed
        self._rebuild_id_map()
        return n_removed

    # ------------------------------------------------------------------ search
    def _check_query(self, x, k):
        if k > 1024:
            raise NotImplementedError("RefineFlatIndex: k > 1024 is not supported")
        assert x.dim() == 2 and x.shape[0] == self.d_vector and k >= 1
        assert x.dtype == torch.float32 and x.device == self._vectors.device
        assert x.device.type == "cuda", "torchpq_b200 has no CPU path: the index must live on a CUDA device"
        return x.contiguous()

    @on_index_device
    def search(self, x, k=1, return_address=False):
        """x [d_vector, n_query] fp32 -> (values [n_query, k] fp32 descending, ids [n_query, k] i64[, address in the
        refine store]).  The base index's search for k1 = min(1024, max(k, ceil(k_factor * k))) ids, then refine."""
        x = self._check_query(x, k)
        _, cand = self.base_index.search(x, k1_of(k, self.k_factor))
        return self.refine(x, cand, k, return_address)

    @on_index_device
    def refine(self, x, candidate_ids, k, return_address=False):
        """The exact pass alone (tpq_refine_flat): x [d_vector, n_query] fp32, candidate_ids [n_query, k1] i64 (-1 and
        ids the store does not hold are dropped; an id listed twice is scored twice), k <= k1 <= 1024
        -> (values, ids[, address]) [n_query, k], missing slots (-inf, -1, -1)."""
        x = self._check_query(x, k)
        assert candidate_ids.dtype == torch.int64 and candidate_ids.dim() == 2
        assert candidate_ids.shape[0] == x.shape[1]
        cand = self._addresses_of(candidate_ids.to(x.device)).contiguous()
        dev, d, nq = x.device, self.d_vector, x.shape[1]
        values = torch.empty(nq, k, dtype=torch.float32, device=dev)
        ids = torch.empty(nq, k, dtype=torch.long, device=dev)
        address = torch.empty(nq, k, dtype=torch.long, device=dev) if return_address else None
        if nq > 0:
            ws_bytes = lib.tpq_refine_flat_workspace_bytes(d, nq, k)
            ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
            check(lib.tpq_refine_flat(ptr(x), d, nq, ptr(cand), cand.shape[1], ptr(self._vectors), self._n_items,
                                      _lib.METRIC[self.distance], k, ptr(self._address2id), ptr(values), ptr(ids),
                                      ptr(address), ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return (values, ids, address) if return_address else (values, ids)
