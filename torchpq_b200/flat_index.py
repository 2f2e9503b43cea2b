"""Host-side mirror of ``torchpq.index.FlatIndex``: exact brute-force k-NN over a flat fp32 store.

Same constructor arguments, attributes and registered buffers (``_storage [d, capacity, 1]``, ``_address2id``,
``_id2address``, so checkpoints interchange) and the same container operations as the reference
(index/FlatIndex.py, container/FlatContainer.py, container/BaseContainer.py).  ``search`` runs one fused sm_90a kernel
(``tpq_flat_search``) that never stores the score matrix; the container operations are plain tensor indexing.

Decided differently from the reference:
  * search writes neither the queries nor the store (the reference's in-place metric turns both into their absolute
    values for euclidean, metric.py:82-98, and re-rounds them for cosine);
  * only the live slots [0, n_items) are scored; missing results are (-inf, id -1, address -1);
  * ``max_id`` advances with every add and is re-derived on load; ``n_items`` is re-derived on load;
  * ties are broken by the total order (score descending, address ascending);
  * k > 1024 raises NotImplementedError instead of falling back to torch.topk.
"""
from __future__ import annotations

import torch

from . import _lib, _range
from ._lib import lib, check, ptr
from .modules import IdContainer, StreamCache, _fingerprint, live_prefix, on_index_device, prefix_remove

_DISTANCE = {"euclidean": "euclidean", "l2": "euclidean", "cosine": "cosine", "angular": "cosine",
             "inner": "inner", "dot": "inner"}                     # FlatIndex.py:31-40


class FlatIndex(IdContainer):
    def __init__(self, d_vector, initial_size=None, expand_step_size=1024, expand_mode="double", device="cuda:0",
                 distance="euclidean", verbose=0):
        super().__init__()
        if distance in ("manhattan", "l1"):
            raise NotImplementedError("currently manhattan distance is not supported")
        if distance not in _DISTANCE:
            raise NotImplementedError(f"unknown distance metric: {distance}")
        if initial_size is None:
            initial_size = expand_step_size                              # BaseContainer.py:17-18
        assert expand_mode in ("step", "double") and initial_size >= 0 and expand_step_size > 0 and d_vector > 0
        self.d_vector, self.code_size, self.contiguous_size, self.dtype = d_vector, d_vector, 1, torch.float32
        self.distance, self.device, self.device_type, self.verbose = _DISTANCE[distance], device, torch.device(device).type, verbose
        self.initial_size, self.expand_step_size, self.expand_mode = initial_size, expand_step_size, expand_mode
        self.use_inverse_id_mapping = True
        self._max_id = -1
        self._n_items = 0
        self._id2address_fp = None
        self._norms = None                                               # (key, table) of the live columns
        dev = torch.device(device)
        self.register_buffer("_address2id", -torch.ones(initial_size, dtype=torch.long, device=dev))
        self.register_buffer("_id2address", None)
        self.register_buffer("_storage", torch.zeros(d_vector, initial_size, 1, dtype=torch.float32, device=dev))

    @property
    def n_items(self):
        return self._n_items

    def _state_changed(self):
        self._norms = None

    def load_state_dict(self, state_dict, strict=True):
        """Reference semantics (CustomModule.py:14-23), then the state the reference keeps outside its buffers:
        ``n_items`` = the live slots (address2id >= 0), which must be a prefix of the store, and ``max_id``."""
        super().load_state_dict(state_dict, strict)
        n = live_prefix(self._address2id)
        assert self._storage.shape == (self.d_vector, self.capacity, 1)
        self._n_items = n
        self._refresh_max_id()

    # ------------------------------------------------------------------ container (FlatContainer.py)
    def expand(self):
        """BaseContainer.expand + FlatContainer.expand: "double" doubles expand_step_size first, then that many slots
        are appended."""
        if self.expand_mode == "double":
            self.expand_step_size *= 2
        n, dev = self.expand_step_size, self._address2id.device
        a2i = torch.cat([self._address2id, -torch.ones(n, dtype=torch.long, device=dev)])
        storage = torch.cat([self._storage, torch.zeros(self.d_vector, n, 1, dtype=torch.float32, device=dev)], dim=1)
        for name, t in (("_address2id", a2i), ("_storage", storage)):
            delattr(self, name)
            self.register_buffer(name, t)
        self._state_changed()

    def empty(self):
        self._address2id.fill_(-1)
        delattr(self, "_id2address")
        self.register_buffer("_id2address", None)
        self._storage.fill_(0)
        self._n_items = 0
        self._state_changed()

    def get_data_by_address(self, address):
        """[d, n] vectors at `address`; zeros where the address is outside [0, capacity)."""
        assert address.dtype == torch.int64
        address = address.to(self._storage.device)
        mask = (0 <= address) & (address < self.capacity)
        data = self._storage[:, torch.where(mask, address, 0), 0]
        return data * mask.to(data.dtype)[None, :] if data.numel() else data

    def set_data_by_address(self, address, data):
        assert address.dtype == torch.int64 and data.dtype == torch.float32
        assert data.dim() == 2 and data.shape[0] == self.d_vector and data.shape[1] == address.shape[0]
        address, data = address.to(self._storage.device), data.to(self._storage.device)
        mask = (0 <= address) & (address < self.capacity)
        self._storage[:, address[mask], 0] = data[:, mask]
        self._state_changed()

    @on_index_device
    def add(self, x, ids=None, return_address=False):
        """FlatContainer.add (FlatContainer.py:118-158): x [d, n] goes to addresses [n_items, n_items + n); default ids
        continue after max_id."""
        assert x.dtype == torch.float32 and x.dim() == 2 and x.shape[0] == self.d_vector
        dev = self._storage.device
        x, n = x.to(dev), x.shape[1]
        if ids is not None:
            assert ids.dtype == torch.int64 and ids.shape == (n,)
            ids = ids.to(dev)
        else:
            ids = torch.arange(n, dtype=torch.long, device=dev) + self._max_id + 1
        while self.capacity - self._n_items < n:
            self.expand()
        address = torch.arange(n, dtype=torch.long, device=dev) + self._n_items
        self._storage[:, self._n_items:self._n_items + n, 0] = x
        self._address2id[self._n_items:self._n_items + n] = ids
        self._n_items += n
        if n:
            self._max_id = max(self._max_id, int(ids.max().item()))
        self._state_changed()
        return (ids, address) if return_address else ids

    @on_index_device
    def remove(self, ids=None, address=None):
        """FlatContainer.remove (FlatContainer.py:160-190): the store stays a prefix -- the surviving items of the last
        n_removed slots move, in ascending order, into the removed slots below them.  Addresses outside the live
        prefix and unknown ids are ignored.  Returns the number removed."""
        if ids is not None:
            address = self.get_address_by_id(ids)
        elif address is not None:
            assert address.dtype == torch.int64
            address = address.to(self._address2id.device)
        else:
            raise RuntimeError("Need either ids or address")
        n_removed, dst, src, tail = prefix_remove(self._address2id, address, self._n_items)
        if n_removed == 0:
            return 0
        self._storage[:, dst] = self._storage[:, src].clone()
        self._storage[:, tail] = 0
        self._n_items -= n_removed
        self._state_changed()
        return n_removed

    # ------------------------------------------------------------------ search
    def _norm_table(self):
        """tpq_flat_norms of the live columns, kept until the store changes (add / remove / set_data_by_address /
        load_state_dict, or any in-place write to _storage)."""
        key = (_fingerprint(self._storage), self._n_items)
        if self._norms is None or self._norms[0] != key:
            n, dev = self._n_items, self._storage.device
            table = torch.empty(max(1, n), dtype=torch.float32, device=dev)
            check(lib.tpq_flat_norms(ptr(self._storage), self.capacity, self.d_vector, n, _lib.METRIC[self.distance],
                                     ptr(table), _lib.current_stream(dev)))
            self._norms = (key, StreamCache(table, dev))
        return self._norms[1].get()

    def _check_query(self, x):
        assert x.dim() == 2 and x.shape[0] == self.d_vector
        assert x.dtype == torch.float32 and x.device == self._storage.device
        assert x.device.type == "cuda", "torchpq_b200 has no CPU path: the index must live on a CUDA device"
        return x.contiguous()

    @on_index_device
    def search(self, x, k=1, return_address=False):
        """FlatIndex.search (FlatIndex.py:46-101): x [d_vector, n_query] fp32 on the index device
        -> (topk_values [n_query, k] fp32 descending, topk_ids [n_query, k] int64[, topk_address])."""
        x = self._check_query(x)
        assert k >= 1
        dev, nq = x.device, x.shape[1]
        values = torch.empty(nq, k, dtype=torch.float32, device=dev)
        ids = torch.empty(nq, k, dtype=torch.long, device=dev)
        address = torch.empty(nq, k, dtype=torch.long, device=dev) if return_address else None
        out = (values, ids, address) if return_address else (values, ids)
        if nq == 0:                                                      # an empty batch has no storage to point at
            return out
        norms = self._norm_table() if self.distance != "inner" else None
        ws_bytes = lib.tpq_flat_workspace_bytes(self.d_vector, nq, self._n_items, k)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
        check(lib.tpq_flat_search(ptr(x), self.d_vector, nq, ptr(self._storage), self.capacity, self._n_items, ptr(norms),
                                  _lib.METRIC[self.distance], k, ptr(self._address2id), ptr(values), ptr(ids),
                                  ptr(address), ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return out

    @on_index_device
    def range_search(self, x, threshold, return_address=False, max_results=1 << 26):
        """Every live item scoring above `threshold`: x [d_vector, n_query] fp32 on the index device, threshold a float
        or a 0-d tensor (rounded once to fp32; NaN raises ValueError)
        -> (lims [n_query + 1] int64, values [nnz] fp32, ids [nnz] int64[, address [nnz] int64]), Faiss's CSR form:
        query q's matches are [lims[q], lims[q + 1]), by score descending, then address ascending.

        An item matches when search's score for it (the same value, bit for bit) is > threshold, strictly, in fp32; a
        NaN score never matches.  For euclidean the score is -|x - b|^2 (in search's arithmetic), so Faiss's
        ``distance < r^2`` is ``threshold = -r^2``.  More than `max_results` matches raise ValueError (naming the
        total) and return nothing.  Unlike search, this synchronises the stream once, to read the number of matches.
        """
        x = self._check_query(x)
        t = _range.threshold_f32(threshold)
        dev, nq, n = x.device, x.shape[1], self._n_items
        if nq == 0:
            return _range.empty(0, dev, return_address)
        norms = self._norm_table() if self.distance != "inner" else None
        ws_bytes = lib.tpq_flat_range_workspace_bytes(self.d_vector, nq, n)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)

        def run(keys, query, cap, total):
            check(lib.tpq_flat_range_search(ptr(x), self.d_vector, nq, ptr(self._storage), self.capacity, n, ptr(norms),
                                            _lib.METRIC[self.distance], t, ptr(keys), ptr(query), cap, ptr(total),
                                            ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return _range.collect(run, nq, max_results, self._address2id, return_address, dev)
