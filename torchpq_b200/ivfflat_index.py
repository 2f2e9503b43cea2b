"""IVFFlatIndex: inverted-file search with exact fp32 distances (Faiss ``IndexIVFFlat``, cuVS ``ivf_flat``).

The reference ships no such index.  This one is ``IVFPQIndex`` with the PQ code replaced by the vector itself:

  * the container is IVFPQ's, with the same buffer names (``_storage``, ``_is_empty``, ``_cell_start``, ``_cell_size``,
    ``_cell_capacity``, ``_address2id``, ``_id2address``; ``vq_codec``), so ``IdContainer`` and checkpoint tooling apply.
    ``_storage`` is fp32 ``[d, capacity, 1]``, FlatIndex's layout: IVFPQ's placement kernels move 4-byte granules, and
    with ``code_size = 4 d`` bytes granule g of an item is dimension g of its vector;
  * ``train`` is the coarse half of ``IVFPQIndex.train`` (same seed, same data -> same coarse codebook), ``add`` assigns
    cells exactly as ``IVFPQIndex.add`` and stores the caller's vectors (not normalised), ``remove`` leaves holes;
  * ``search`` runs IVFPQ's coarse stage and visiting rule, then scores every live vector of the visited cells exactly,
    with FlatIndex's arithmetic (``tpq_ivfflat_search``, csrc/ivfflat.cu): with every cell probed the values are
    ``FlatIndex.search``'s over the same vectors, bit for bit.  Order: score descending, then address ascending.
"""
from __future__ import annotations

import torch

from . import _lib, _range
from ._lib import lib, check, ptr
from .modules import Codec, IdContainer, StreamCache, _fingerprint, on_index_device


class IVFFlatIndex(IdContainer):
    _SEARCH, _RANGE = "tpq_ivfflat_search", "tpq_ivfflat_range_search"       # the library's entry points

    def __init__(self, d_vector, n_cells=128, initial_size=None, expand_step_size=128, expand_mode="double",
                 distance="euclidean", device="cuda:0", verbose=0):
        super().__init__()
        if distance not in ("euclidean", "cosine"):
            raise NotImplementedError(f"IVFFlatIndex supports euclidean and cosine distance, not {distance!r}")
        if initial_size is None:
            initial_size = expand_step_size
        assert d_vector > 0 and n_cells > 0 and initial_size >= 0
        assert expand_mode in ("step", "double") and expand_step_size > 0
        self.d_vector, self.n_cells = d_vector, n_cells
        self.code_size, self.contiguous_size = 4 * d_vector, 4          # bytes per item, moved in 4-byte granules
        self.distance, self.device, self.verbose = distance, device, verbose
        self.initial_size, self.expand_step_size, self.expand_mode = initial_size, expand_step_size, expand_mode
        self.n_probe = 1
        self.use_smart_probing = True
        self.smart_probing_temperature = 30.0
        self._max_id = -1
        self._has_holes = False
        self._id2address_fp = None
        self._norms = None                                               # (store fingerprint, per-slot norm table)
        dev = torch.device(device)
        cap = n_cells * initial_size
        self.register_buffer("_address2id", -torch.ones(cap, dtype=torch.long, device=dev))
        self.register_buffer("_id2address", None)
        self.register_buffer("_storage", self._empty_store(cap, dev))
        self.register_buffer("_cell_start", torch.arange(n_cells, device=dev) * initial_size)
        self.register_buffer("_cell_size", torch.zeros(n_cells, dtype=torch.long, device=dev))
        self.register_buffer("_cell_capacity", torch.zeros(n_cells, dtype=torch.long, device=dev) + initial_size)
        self.register_buffer("_is_empty", torch.ones(cap, dtype=torch.uint8, device=dev))
        self.vq_codec = Codec()

    @property
    def n_items(self):
        return int((self._is_empty == 0).sum().item())

    def _state_changed(self):
        # tpq_store_codes writes _storage through a raw pointer (its _version does not move), so the norm table is
        # dropped explicitly on every change of the store, not only when its fingerprint moves
        self._norms = None

    def _empty_store(self, cap, dev):
        """A zero store of `cap` slots: fp32 [d, cap, 1]."""
        return torch.zeros(self.d_vector, cap, 1, dtype=torch.float32, device=dev)

    def _store_args(self):
        """The store's arguments of the search entry points, between n_cells and capacity."""
        return (ptr(self._storage),)

    def load_state_dict(self, state_dict, strict=True):
        """As IVFPQIndex.load_state_dict: the buffers, then ``_max_id`` re-derived and holes assumed."""
        super().load_state_dict(state_dict, strict)
        want = self._empty_store(0, "meta")
        assert self._storage.dtype == want.dtype and self._storage.shape == (want.shape[0], self.capacity, want.shape[2])
        self._has_holes = True
        self._refresh_max_id()

    # ------------------------------------------------------------------ build side (build.py, shared with IVFPQIndex)
    @on_index_device
    def train(self, x, force_retrain=False, seed=0):
        """The coarse half of IVFPQIndex.train (build.train_coarse): k-means on x (normalised for cosine)."""
        if self.vq_codec.is_trained and not force_retrain:
            self.print_message("index is already trained", 1)
            return
        from . import build
        _, vq = build.train_coarse(self, x, seed=seed)
        self.vq_codec.set_codebook(vq)
        self._state_changed()

    @on_index_device
    def add(self, x, ids=None, return_address=False, chunk: int = 1 << 20):
        """x [d, n] fp32: cell = exact assignment of x (normalised for cosine, as IVFPQIndex.add); the stored vector is
        x itself.  Placement, holes and expansion are IVFPQIndex's (build.container_add)."""
        assert x.dim() == 2 and x.shape[0] == self.d_vector and x.dtype == torch.float32
        assert self.vq_codec.is_trained, "index is not trained"
        from . import build, fn
        x = x.to(self._storage.device).contiguous()
        cells = []
        for s in range(0, x.shape[1], chunk):
            xc = x[:, s:s + chunk].contiguous()
            if self.distance == "cosine":
                xc = fn.normalize(xc)
            cells.append(build._assign(xc[None], self.vq_codec.codebook[None])[0])
        cells = torch.cat(cells) if cells else torch.empty(0, dtype=torch.long, device=x.device)
        # code byte 4 g + b of item i = byte b of x[g, i]: tpq_store_codes writes it to _storage[g, address] as one word
        codes = x.view(torch.uint8).view(self.d_vector, x.shape[1], 4).permute(0, 2, 1).reshape(self.code_size, x.shape[1])
        return build.container_add(self, codes.contiguous(), cells, ids, return_address)   # calls _state_changed

    @on_index_device
    def remove(self, ids=None, address=None):
        """As IVFPQIndex.remove: removed slots become holes that search skips and the next add fills first;
        ``_cell_size`` is not decremented."""
        from . import build
        build.container_remove(self, ids, address)

    def get_data_by_address(self, address):
        """[d, n] vectors at `address`; zeros where the address is outside [0, capacity)."""
        assert address.dtype == torch.int64
        address = address.to(self._storage.device)
        mask = (0 <= address) & (address < self.capacity)
        data = self._storage[:, torch.where(mask, address, 0), 0]
        return data * mask.to(data.dtype)[None, :] if data.numel() else data

    # ------------------------------------------------------------------ search
    def _norm_table(self):
        """tpq_flat_norms of every slot (|b|^2 or |b| + 1e-8), kept until the store changes."""
        key = _fingerprint(self._storage)
        if self._norms is None or self._norms[0] != key:
            dev, cap = self._storage.device, self.capacity
            table = torch.empty(max(1, cap), dtype=torch.float32, device=dev)
            check(lib.tpq_flat_norms(ptr(self._storage), cap, self.d_vector, cap, _lib.METRIC[self.distance], ptr(table),
                                     _lib.current_stream(dev)))
            self._norms = (key, StreamCache(table, dev))
        return self._norms[1].get()

    def _check_query(self, x, k):
        assert x.dim() == 2 and x.shape[0] == self.d_vector
        assert 0 < k <= 1024
        assert x.dtype == torch.float32 and x.device == self._storage.device
        assert x.device.type == "cuda", "torchpq_b200 has no CPU path: the index must live on a CUDA device"
        return x.contiguous()

    def _search(self, x, k, n_probe, cells, n_probe_list, return_address):
        dev, nq = x.device, x.shape[1]
        values = torch.empty(nq, k, dtype=torch.float32, device=dev)
        ids = torch.empty(nq, k, dtype=torch.long, device=dev)
        address = torch.empty(nq, k, dtype=torch.long, device=dev) if return_address else None
        out = (values, ids, address) if return_address else (values, ids)
        if nq == 0:                                                      # an empty batch has no storage to point at
            return out
        if cells is None:
            assert self.vq_codec.is_trained, "index is not trained"
        norms = self._norm_table()
        ws_bytes = lib.tpq_ivfflat_workspace_bytes(self.d_vector, nq, self.n_cells, n_probe, k)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
        vq = self.vq_codec.kmeans.centroids if cells is None else None
        entry = getattr(lib, self._SEARCH)
        check(entry(ptr(x), self.d_vector, nq, ptr(vq), self.n_cells, *self._store_args(), self.capacity,
                    ptr(self._is_empty), ptr(self._cell_start), ptr(self._cell_size), ptr(norms),
                    _lib.METRIC[self.distance], ptr(cells), ptr(n_probe_list), n_probe,
                    int(bool(self.use_smart_probing)), float(self.smart_probing_temperature), k,
                    ptr(self._address2id), ptr(values), ptr(ids), ptr(address), ptr(ws), ws_bytes,
                    _lib.current_stream(dev)))
        return out

    @on_index_device
    def search(self, x, k=1, return_address=False):
        """x [d_vector, n_query] fp32 on the index device -> (values [n_query, k] fp32 descending, ids [n_query, k]
        int64[, address]).  Probes as IVFPQIndex.search (n_probe, use_smart_probing, smart_probing_temperature)."""
        x = self._check_query(x, k)
        return self._search(x, k, int(self.n_probe), None, None, return_address)

    @on_index_device
    def range_search(self, x, threshold, return_address=False, max_results=1 << 26):
        """Every item that search would score for a query with a score above `threshold`: x [d_vector, n_query] fp32 on
        the index device, threshold a float or a 0-d tensor (rounded once to fp32; NaN raises ValueError)
        -> (lims [n_query + 1] int64, values [nnz] fp32, ids [nnz] int64[, address [nnz] int64]), Faiss's CSR form:
        query q's matches are [lims[q], lims[q + 1]), by score descending, then address ascending.

        The scored items are search's: the live slots of the cells the query visits under n_probe, use_smart_probing
        and smart_probing_temperature; holes left by remove never match.  An item matches when its score (search's
        value, bit for bit) is > threshold, strictly, in fp32; a NaN score never matches.  For euclidean the score is
        -|x - b|^2 (in search's arithmetic), so Faiss's ``distance < r^2`` is ``threshold = -r^2``.  More than
        `max_results` matches raise ValueError (naming the total) and return nothing.  Unlike search, this
        synchronises the stream once, to read the number of matches.
        """
        x = self._check_query(x, 1)
        t = _range.threshold_f32(threshold)
        dev, nq, n_probe = x.device, x.shape[1], int(self.n_probe)
        if nq == 0:
            return _range.empty(0, dev, return_address)
        assert self.vq_codec.is_trained, "index is not trained"
        norms = self._norm_table()
        ws_bytes = lib.tpq_ivfflat_range_workspace_bytes(self.d_vector, nq, self.n_cells, n_probe)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
        entry, store = getattr(lib, self._RANGE), self._store_args()

        def run(keys, query, cap, total):
            check(entry(ptr(x), self.d_vector, nq, ptr(self.vq_codec.kmeans.centroids), self.n_cells, *store,
                        self.capacity, ptr(self._is_empty), ptr(self._cell_start), ptr(self._cell_size), ptr(norms),
                        _lib.METRIC[self.distance], None, None, n_probe, int(bool(self.use_smart_probing)),
                        float(self.smart_probing_temperature), t, ptr(keys), ptr(query), cap, ptr(total), ptr(ws),
                        ws_bytes, _lib.current_stream(dev)))
        return _range.collect(run, nq, max_results, self._address2id, return_address, dev)

    @on_index_device
    def search_cells(self, x, cells, n_probe_list=None, k=1, return_address=False):
        """As IVFPQIndex.search_cells: cells [n_query, n_probe] int64 probe lists, n_probe_list [n_query] int64
        (default n_probe)."""
        x = self._check_query(x, k)
        dev, nq = x.device, x.shape[1]
        assert cells.dtype == torch.int64 and cells.dim() == 2 and cells.shape[0] == nq
        n_probe = cells.shape[1]
        if n_probe_list is None:
            n_probe_list = torch.zeros(nq, dtype=torch.long, device=dev) + n_probe
        assert n_probe_list.shape == (nq,) and n_probe_list.dtype == torch.int64
        return self._search(x, k, n_probe, cells.contiguous(), n_probe_list.contiguous(), return_address)
