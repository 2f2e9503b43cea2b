"""Host-side mirror of ``torchpq.index.IVFPQIndex`` for the search hot path.

Same constructor arguments, attributes, registered buffers (so checkpoints interchange)
and ``search`` / ``search_cells`` signatures and return values as the reference class
(torchpq/index/IVFPQIndex.py:12-87, 407-524; container/CellContainer.py:46-81;
container/BaseContainer.py:32-38).  All computation is the sm_90a library behind
``include/tpq_b200.h``; PyTorch is used for device memory and streams only.

Residual IVFPQ (``pq_use_residual=True``) runs the RES variant of the scan kernel.  Not covered (out of the
hot-path scope, SURVEY.md section 8): ``use_cublas=False`` / tensor-core coarse variants (flags accepted, ignored).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib, _range
from ._lib import lib, check, ptr
from .modules import Codec, IdContainer, StreamCache, _fingerprint, on_index_device


def _codebook_of(codec):
    """The codec's centroid buffer without going through ``is_trained`` (a device->host read in the reference's
    BaseCodec): torchpq_b200 codecs and torchpq codecs both keep it at ``codec.kmeans.centroids``."""
    km = getattr(codec, "kmeans", None)
    cb = getattr(km, "centroids", None) if km is not None else None
    return cb if cb is not None else codec.codebook


class ScanLayout:
    """The scan ("shadow") layout of one index (or of one shard of it) + its ``tpq_index`` struct.

    Built from the reference buffers by ``tpq_relayout_*``; rebuilt whenever any of those
    buffers is replaced or modified in place (``add``, ``expand``, ``load_state_dict``...).
    ``parts`` = (codes_scan, block_valid, cell_block_start, n_blocks) adopts a shard that was laid out elsewhere
    (dist.distribute): the index then needs no ``_storage`` / ``_is_empty`` at all."""

    def __init__(self, index: "IVFPQIndex", shard_rank: int = 0, shard_world: int = 1, parts=None):
        dev = index._address2id.device
        assert dev.type == "cuda", "torchpq_b200 has no CPU path: the index must live on a CUDA device"
        stream = _lib.current_stream(dev)
        M, d, Cn = index.n_subvectors, index.d_vector, index.n_cells
        self.m_pad = (M + 31) // 32 * 32
        self.shard = (shard_rank, shard_world)
        vq, pq = _codebook_of(index.vq_codec), _codebook_of(index.pq_codec)
        self.keep = (index._storage, index._is_empty, index._cell_start, index._cell_size, index._address2id, vq, pq)
        for t in self.keep[2:] if parts is not None else self.keep:
            assert t is not None and t.is_contiguous()
        if parts is None:
            self.cell_block_start = torch.empty(Cn + 1, dtype=torch.int32, device=dev)
            # blocks for every slot of each cell's CAPACITY, so that add() can place new items in the layout in place
            extent = getattr(index, "_cell_capacity", None)
            extent = index._cell_size if extent is None else extent
            check(lib.tpq_relayout_plan(ptr(extent), Cn, shard_rank, shard_world,
                                        ptr(self.cell_block_start), stream))
            self.n_blocks = int(self.cell_block_start[Cn].item())          # one host sync per (re)build
            self.codes_scan = torch.empty(max(1, lib.tpq_codes_scan_bytes(M, self.n_blocks)), dtype=torch.uint8, device=dev)
            self.block_valid = torch.empty(max(1, self.n_blocks), dtype=torch.int32, device=dev)
        else:
            self.codes_scan, self.block_valid, self.cell_block_start, self.n_blocks = parts
            assert self.cell_block_start.shape[0] == Cn + 1 and self.cell_block_start.dtype == torch.int32
            assert self.codes_scan.numel() >= lib.tpq_codes_scan_bytes(M, self.n_blocks)
        self.pq_codebook_t = torch.empty(256 * self.m_pad * (d // M), dtype=torch.float32, device=dev)
        self.pq_norm_t = torch.empty(256 * self.m_pad, dtype=torch.float32, device=dev)
        ix = _lib.TpqIndex()
        ix.d_vector, ix.n_subvectors, ix.n_cells = d, M, Cn
        ix.metric = _lib.METRIC[index.distance]
        ix.capacity = index._address2id.shape[0]
        ix.vq_codebook = vq.data_ptr()
        ix.pq_codebook = pq.data_ptr()
        ix.storage = index._storage.data_ptr() if index._storage is not None else 0
        ix.is_empty = index._is_empty.data_ptr() if index._is_empty is not None else 0
        ix.cell_start = index._cell_start.data_ptr()
        ix.cell_size = index._cell_size.data_ptr()
        ix.address2id = index._address2id.data_ptr()
        ix.m_pad, ix.shard_rank, ix.shard_world = self.m_pad, shard_rank, shard_world
        ix.code_size = getattr(index, "code_size", M)                      # bytes per item in _storage (add writes them all)
        ix.n_blocks = self.n_blocks
        ix.codes_scan = self.codes_scan.data_ptr()
        ix.block_valid = self.block_valid.data_ptr()
        ix.cell_block_start = self.cell_block_start.data_ptr()
        ix.pq_codebook_t = self.pq_codebook_t.data_ptr()
        ix.pq_norm_t = self.pq_norm_t.data_ptr()
        self.part2_scan = None
        if getattr(index, "pq_use_residual", False):
            # IVFPQIndex.precompute_part2 (IVFPQIndex.py:160-170), laid out like the shared-memory LUT
            self.part2_scan = torch.empty(lib.tpq_part2_scan_bytes(M, Cn) // 4, dtype=torch.float32, device=dev)
            check(lib.tpq_relayout_part2(ptr(vq), ptr(pq), d, M, Cn, ptr(self.part2_scan), stream))
            ix.part2_scan = self.part2_scan.data_ptr()
            ix.residual = 1
        self.cindex = ix
        if parts is None:
            check(lib.tpq_relayout_codes(C.byref(ix), ptr(self.codes_scan), ptr(self.block_valid), stream))
        check(lib.tpq_relayout_codebook(ptr(pq), d, M, ix.metric, ptr(self.pq_codebook_t), ptr(self.pq_norm_t), stream))
        # live vectors of this shard = set bits of block_valid; the search picks its scan kernel by the mean per cell
        bits = self.block_valid[:self.n_blocks].view(torch.uint8).long()
        popc = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.long, device=dev)
        self.set_live(int(popc[bits].sum().item()) if self.n_blocks else 0)
        self.fingerprint = _fingerprint(*self.keep)
        self.ready = StreamCache(None, dev)                              # a search on another stream waits for the kernels above

    def set_live(self, n_live: int) -> None:
        self.n_live = n_live
        rank, world = self.shard
        owned = len(range(rank, self.cindex.n_cells, world))
        self.cindex.mean_cell_live = min(n_live // max(1, owned), 2 ** 31 - 1)

    def resident_bytes(self) -> int:
        """Device bytes of the scan layout (what a shard-only rank holds besides the replicated small state)."""
        ts = (self.codes_scan, self.block_valid, self.cell_block_start, self.pq_codebook_t, self.pq_norm_t, self.part2_scan)
        return sum(t.numel() * t.element_size() for t in ts if t is not None)


class IVFPQIndex(IdContainer):
    def __init__(self, d_vector, n_subvectors=8, n_cells=128, initial_size=None, expand_step_size=128,
                 expand_mode="double", distance="euclidean", device="cuda:0", pq_use_residual=False, verbose=0):
        super().__init__()
        assert d_vector % n_subvectors == 0                              # IVFPQIndex.py:30
        assert n_subvectors % 4 == 0, "code_size % contiguous_size(4) == 0"   # CellContainer.py:36, IVFPQIndex.py:41
        assert expand_mode in ("step", "double") and expand_step_size > 0      # BaseContainer.py:19-21
        assert distance in ("euclidean", "cosine"), \
            "the reference can only build/search euclidean and cosine IVFPQ indexes (MultiKMeans.py:82-115,218-223)"
        if pq_use_residual:
            assert distance == "euclidean", "residual IVFPQ is defined on euclidean residuals"
            # IVFPQIndex.py:52-55: the reference precomputes the per-cell half of the LUT when it fits 4 GB and otherwise
            # recomputes it per (query, probe) (precomputed_adc_residual, :382-405) -- a device-memory limit of 2021.  On an
            # 80 GB H100 the table (n_cells * ceil(M/64) * 64 KB in scan layout) is simply kept, up to 32 GB; the two
            # variants differ only in fp32 association, (2xp) + (-2cp - |p|^2) vs (2xp - |p|^2) + (-2cp).
            if n_cells * 256 * ((n_subvectors + 63) // 64 * 64) * 4 > 32 * 1024 ** 3:
                raise NotImplementedError("residual IVFPQ: the precomputed part-2 table would exceed 32 GB")
        if initial_size is None:
            initial_size = expand_step_size                              # CellContainer.py:23-24
        assert initial_size >= 0 and n_cells > 0
        self.d_vector, self.n_subvectors, self.d_subvector = d_vector, n_subvectors, d_vector // n_subvectors
        self.n_cells, self.code_size, self.contiguous_size = n_cells, n_subvectors, 4
        self.distance, self.device, self.verbose = distance, device, verbose
        self.initial_size, self.expand_step_size, self.expand_mode = initial_size, expand_step_size, expand_mode
        self.pq_use_residual = bool(pq_use_residual)
        self._use_precomputed = bool(pq_use_residual)
        self.n_probe = 1                                                 # IVFPQIndex.py:51
        self.use_smart_probing = True                                    # IVFPQIndex.py:58
        self.smart_probing_temperature = 30.0                            # IVFPQIndex.py:59
        self._max_id = -1
        self._has_holes = False                                         # set by remove(): add() then needs the empty-slot prefix
        dev = torch.device(device)
        cap = n_cells * initial_size
        self.register_buffer("_address2id", -torch.ones(cap, dtype=torch.long, device=dev))
        self.register_buffer("_id2address", None)
        self.register_buffer("_storage", torch.zeros(n_subvectors // 4, cap, 4, dtype=torch.uint8, device=dev))
        self.register_buffer("_cell_start", torch.arange(n_cells, device=dev) * initial_size)
        self.register_buffer("_cell_size", torch.zeros(n_cells, dtype=torch.long, device=dev))
        self.register_buffer("_cell_capacity", torch.zeros(n_cells, dtype=torch.long, device=dev) + initial_size)
        self.register_buffer("_is_empty", torch.ones(cap, dtype=torch.uint8, device=dev))
        self.vq_codec = Codec()
        self.pq_codec = Codec()
        self._layout: Optional[ScanLayout] = None
        self._shard = (0, 1)
        self._id2address_fp = None

    # ------------------------------------------------------------------ container properties
    @property
    def n_items(self):
        assert self._is_empty is not None, "shard-only index (dist.distribute) keeps no per-slot state"
        return int((self._is_empty == 0).sum().item())               # live vectors (== _cell_size.sum() until a remove)

    # flags the reference exposes and this path ignores (always the fused fp32 coarse kernel)
    use_cublas = True
    use_tensor_core = False
    fp16_scale_mode = "a"

    def _state_changed(self):
        self._layout = None

    def load_state_dict(self, state_dict, strict=True):
        """Reference semantics (CustomModule.py:14-23) + the one piece of state the reference keeps outside its
        buffers: ``_max_id`` (BaseContainer.py:30,49-51) is re-derived from ``_address2id`` so that ids handed out
        after a load do not restart at 0 and ``get_address_by_id`` sizes its inverse map correctly."""
        super().load_state_dict(state_dict, strict)
        self._has_holes = True                                          # unknown provenance: assume the container may have holes
        self._refresh_max_id()

    # ------------------------------------------------------------------ state import
    def load_state(self, st):
        """Adopt an ``oracle.ivfpq_oracle.IndexState``-shaped object (numpy buffers) -- test/bench helper."""
        dev = torch.device(self.device)

        def T(a):
            return torch.as_tensor(a).to(dev).contiguous()

        assert (st.d_vector, st.n_subvectors, st.n_cells, st.distance) == \
               (self.d_vector, self.n_subvectors, self.n_cells, self.distance)
        for name, val in (("_storage", st.storage), ("_is_empty", st.is_empty), ("_cell_start", st.cell_start),
                          ("_cell_size", st.cell_size), ("_cell_capacity", st.cell_capacity),
                          ("_address2id", st.address2id)):
            delattr(self, name)
            self.register_buffer(name, T(val))
        self.vq_codec.set_codebook(T(st.vq_codebook))
        self.pq_codec.set_codebook(T(st.pq_codebook))
        self._max_id = int(st.max_id)
        self._has_holes = True                                          # as load_state_dict: the state may have holes
        self._ids_changed()                                             # a new _address2id may reuse the old one's memory
        self.n_probe = st.n_probe
        self.use_smart_probing = st.use_smart_probing
        self.smart_probing_temperature = st.smart_probing_temperature
        self._layout = None
        return self

    def set_shard(self, rank: int, world: int):
        """Scan only the cells c with c % world == rank (cell-sharded multi-GPU search, dist.py)."""
        assert 0 <= rank < world
        assert self._storage is not None or (rank, world) == self._shard, "shard-only index: the shard is fixed"
        if (rank, world) != self._shard:
            self._shard = (rank, world)
            self._layout = None

    def adopt_shard(self, shard_rank, shard_world, codes_scan, block_valid, cell_block_start, n_blocks):
        """Become a shard-only index (dist.distribute): the scan layout of this rank's cells was built elsewhere and the
        reference-layout code store (`_storage`, `_is_empty`) is dropped.  Search works; add / remove need the full index."""
        for name in ("_storage", "_is_empty"):
            delattr(self, name)
            self.register_buffer(name, None)
        self._shard = (shard_rank, shard_world)
        self._layout = ScanLayout(self, shard_rank, shard_world, parts=(codes_scan, block_valid, cell_block_start, n_blocks))
        return self

    def drop_reference_layout(self):
        """Search-only deployment on one GPU: keep the scan layout, free `_storage` / `_is_empty` (C3: 0.8 GB of the 1.8 GB
        the index holds).  The index becomes shard-only (shard 0 of 1): add / remove need a reload of the checkpoint."""
        lay = self.layout()
        return self.adopt_shard(lay.shard[0], lay.shard[1], lay.codes_scan, lay.block_valid, lay.cell_block_start, lay.n_blocks)

    def resident_bytes(self) -> int:
        """Device bytes this index object holds (registered buffers, codebooks, scan layout)."""
        n = sum(t.numel() * t.element_size() for t in self.buffers() if t is not None)
        return n + (self._layout.resident_bytes() if self._layout is not None else 0)

    @on_index_device
    def layout(self) -> ScanLayout:
        vq, pq = _codebook_of(self.vq_codec), _codebook_of(self.pq_codec)     # no host sync (is_trained.item()) per search
        fp = _fingerprint(self._storage, self._is_empty, self._cell_start, self._cell_size, self._address2id, vq, pq)
        if self._layout is None or self._layout.fingerprint != fp:
            assert self._storage is not None, "shard-only index: its state cannot change (re-distribute the full index)"
            assert self.vq_codec.is_trained and self.pq_codec.is_trained, "codec is not trained"
            self._layout = ScanLayout(self, *self._shard)
        self._layout.ready.get()
        return self._layout

    # ------------------------------------------------------------------ search
    def _check_query(self, x, k):
        assert len(x.shape) == 2                                          # IVFPQIndex.py:471
        assert x.shape[0] == self.d_vector                                # :472
        assert 0 < k <= 1024                                              # :473
        assert x.dtype == torch.float32 and x.device == self._address2id.device
        return x.contiguous()

    def _search(self, x, k, n_probe, call, outputs=True, return_address=False, return_keys=False):
        """The body of search, search_cells and scan_push: allocates the outputs (values, ids and those the flags ask
        for; none for scan_push) and the workspace tpq_search_workspace_bytes asks for, then runs
        call(index, values, ids, address, keys, ws, ws_bytes, stream) on their pointers."""
        lay = self.layout()
        dev, nq = x.device, x.shape[1]
        new = lambda dtype: torch.empty(nq, k, dtype=dtype, device=dev)
        values, ids = (new(torch.float32), new(torch.long)) if outputs else (None, None)
        address = new(torch.long) if return_address else None
        keys = new(torch.int64) if return_keys else None
        out = ((values, ids) + ((address,) if return_address else ()) + ((keys,) if return_keys else ())) if outputs else None
        if nq == 0 and outputs:                                        # an empty batch has no storage to point at
            return out
        ws_bytes = lib.tpq_search_workspace_bytes(C.byref(lay.cindex), nq, n_probe, k)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
        check(call(C.byref(lay.cindex), ptr(values), ptr(ids), ptr(address), ptr(keys), ptr(ws), ws_bytes,
                   _lib.current_stream(dev)))
        return out

    @on_index_device
    def search(self, x, k=1, return_address=False, return_keys=False):
        """IVFPQIndex.search (IVFPQIndex.py:469-524): x [d_vector, n_query] fp32 on the index device
        -> (topk_values [n_query, k] fp32 descending, topk_ids [n_query, k] int64[, topk_address])."""
        x = self._check_query(x, k)
        n_probe = int(self.n_probe)
        smart, temperature = int(bool(self.use_smart_probing)), float(self.smart_probing_temperature)
        return self._search(x, k, n_probe, lambda ix, *out: lib.tpq_ivfpq_search(ix, ptr(x), x.shape[1], n_probe, k, smart,
                                                                                  temperature, *out),
                            return_address=return_address, return_keys=return_keys)

    @on_index_device
    def range_search(self, x, threshold, return_address=False, max_results=1 << 26):
        """Every item that search would score for a query with a score above `threshold`: x [d_vector, n_query] fp32 on
        the index device, threshold a float or a 0-d tensor (rounded once to fp32; NaN raises ValueError)
        -> (lims [n_query + 1] int64, values [nnz] fp32, ids [nnz] int64[, address [nnz] int64]), Faiss's CSR form:
        query q's matches are [lims[q], lims[q + 1]), by score descending, then address ascending.

        The scored items are search's: the live slots of the cells the query visits under n_probe, use_smart_probing
        and smart_probing_temperature; holes left by remove never match.  An item matches when its score (search's
        value, bit for bit: the ADC score, plus the cell's coarse similarity for a residual index) is > threshold,
        strictly, in fp32; a NaN score never matches.  For euclidean the score approximates -|x - b|^2, so Faiss's
        ``distance < r^2`` is ``threshold = -r^2``.  On a cell shard (set_shard) only the shard's cells are scanned.
        More than `max_results` matches raise ValueError (naming the total) and return nothing.  Unlike search, this
        synchronises the stream once, to read the number of matches.
        """
        x = self._check_query(x, 1)
        t = _range.threshold_f32(threshold)
        dev, nq, n_probe = x.device, x.shape[1], int(self.n_probe)
        if nq == 0 or self._address2id.shape[0] == 0:                   # no queries, or an index without a slot
            return _range.empty(nq, dev, return_address)
        lay = self.layout()
        smart, temperature = int(bool(self.use_smart_probing)), float(self.smart_probing_temperature)
        ws_bytes = lib.tpq_ivfpq_range_workspace_bytes(C.byref(lay.cindex), nq, n_probe)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)

        def run(keys, query, cap, total):
            check(lib.tpq_ivfpq_range_search(C.byref(lay.cindex), ptr(x), None, None, None, nq, n_probe, smart,
                                             temperature, t, ptr(keys), ptr(query), cap, ptr(total), ptr(ws), ws_bytes,
                                             _lib.current_stream(dev)))
        return _range.collect(run, nq, max_results, self._address2id, return_address, dev)

    @on_index_device
    def search_cells(self, x, cells, base_sims=None, n_probe_list=None, k=1, return_address=False, return_keys=False):
        """IVFPQIndex.search_cells, non-residual branch (IVFPQIndex.py:407-467)."""
        x = self._check_query(x, k)
        dev, nq = x.device, x.shape[1]
        assert cells.dtype == torch.int64 and cells.shape[0] == nq and cells.dim() == 2
        n_probe = cells.shape[1]
        if n_probe_list is None:
            n_probe_list = torch.zeros(nq, dtype=torch.long, device=dev) + n_probe
        assert n_probe_list.shape == (nq,) and n_probe_list.dtype == torch.int64     # IVFPQTopkCuda.py:109-110
        cells, n_probe_list = cells.contiguous(), n_probe_list.contiguous()
        if not self.pq_use_residual:
            base_sims = None
        elif nq > 0:
            assert base_sims is not None, "base_sims is required when pq_use_residual is True"   # IVFPQIndex.py:424
            assert base_sims.shape == (nq, n_probe) and base_sims.dtype == torch.float32
            base_sims = base_sims.contiguous()
        return self._search(x, k, n_probe, lambda ix, *out: lib.tpq_ivfpq_search_cells(ix, ptr(x), ptr(cells), ptr(base_sims),
                                                                                        ptr(n_probe_list), nq, n_probe, k, *out),
                            return_address=return_address, return_keys=return_keys)

    def scan_push(self, x, k, peer_ptrs, n_peers, my_slot, cells=None, base_sims=None, n_probe_list=None):
        """The scan of search / search_cells with its output fused into the cross-shard exchange (tpq_ivfpq_scan_push):
        every CTA stores its top-k keys into slot `my_slot` of each rank's gather buffer (`peer_ptrs`: a ctypes array of
        device pointers into peer-mapped memory).  Raises NotImplementedError for batches small enough to be sliced."""
        x = self._check_query(x, k)
        n_probe = int(self.n_probe) if cells is None else cells.shape[1]
        if cells is not None:
            assert cells.dtype == torch.int64 and cells.shape[0] == x.shape[1] and n_probe_list is not None
            cells, n_probe_list = cells.contiguous(), n_probe_list.contiguous()
            base_sims = base_sims.contiguous() if base_sims is not None else None
            assert not self.pq_use_residual or base_sims is not None
        smart, temperature = int(bool(self.use_smart_probing)), float(self.smart_probing_temperature)
        self._search(x, k, n_probe, lambda ix, _v, _i, _a, _k, *ws: lib.tpq_ivfpq_scan_push(
            ix, ptr(x), ptr(cells), ptr(base_sims), ptr(n_probe_list), x.shape[1], n_probe, k, smart, temperature,
            peer_ptrs, n_peers, my_slot, *ws), outputs=False)

    # ------------------------------------------------------------------ build side (see build.py)
    @on_index_device
    def train(self, x, force_retrain=False, seed=0):
        if self.vq_codec.is_trained and self.pq_codec.is_trained and not force_retrain:
            self.print_message("index is already trained", 1)                 # IVFPQIndex.py:235-238
            return
        from . import build
        build.train(self, x, seed=seed)

    @on_index_device
    def add(self, x, ids=None, return_address=False):
        from . import build
        return build.add(self, x, ids, return_address)

    @on_index_device
    def remove(self, ids=None, address=None):
        """CellContainer.remove (CellContainer.py:369-393) as it is documented to behave (README.md:60-66: "virtually
        remove vectors ... ignores ids that don't exist").  The shipped reference returns early whenever fewer items
        are removed than the index holds (CellContainer.py:381-383), i.e. it never removes anything; that bug is not
        reproduced.  Removed slots become holes (is_empty = 1, address2id = -1) that the scan skips and that the next
        `add` into the cell fills first.  `_cell_size` is deliberately NOT decremented: search scans
        [cell_start, cell_start + cell_size) (ivfpq_topk.cu:852-853), so shrinking it -- as the reference's dead code
        would -- hides live vectors at the tail of the cell."""
        from . import build
        build.container_remove(self, ids, address)

    @on_index_device
    def encode(self, x):
        """IVFPQIndex.encode (IVFPQIndex.py:262-287): x [d_vector, n] -> PQ codes [n_subvectors, n] uint8
        (residual index: (pq_code of x - vq centroid, vq_code), IVFPQIndex.py:281-284)."""
        assert len(x.shape) == 2 and x.shape[0] == self.d_vector
        from . import build, fn
        if self.distance == "cosine":
            x = fn.normalize(x.contiguous())
        if self.pq_use_residual:
            cells, codes = build.encode(self, x.contiguous())
            return codes, cells
        sub = x.reshape(self.n_subvectors, self.d_subvector, x.shape[1])
        return build._assign(sub, self.pq_codec.codebook).to(torch.uint8)

    @on_index_device
    def decode(self, code):
        """IVFPQIndex.decode (IVFPQIndex.py:289-314) -> PQCodec.decode (PQCodec.py:113-130): [M, n] u8 -> [d, n] f32
        (residual index: x = (pq_code, vq_code) -> vq centroid + decoded residual)."""
        from . import fn
        if self.pq_use_residual:
            assert len(code) == 2
            pq_code, vq_code = code
            assert pq_code.shape[0] == self.n_subvectors and pq_code.shape[1] == vq_code.shape[0]
            return self.vq_codec.codebook[:, vq_code] + fn.pq_decode(self.pq_codec.codebook, pq_code)
        assert len(code.shape) == 2 and code.shape[0] == self.n_subvectors
        return fn.pq_decode(self.pq_codec.codebook, code)
