"""IVFPQ4Index: inverted-file search over 4-bit PQ codes (Faiss ``IndexIVFPQ`` with ``nbits=4``, cuVS IVF-PQ with
``pq_bits=4``): 16 codewords per sub-quantizer, n_subvectors / 2 bytes per vector.

``IVFPQIndex`` with a 16-word codebook and packed codes:

  * the container is IVFPQ's, buffer for buffer: ``_storage`` is u8 ``[n_subvectors // 8, capacity, 4]``, code m of an
    item is nibble ``m & 1`` of byte ``m >> 1`` (low nibble first), so word g of a slot holds sub-quantizers 8 g .. 8 g + 7;
    add, holes, expansion and remove are ``build.container_add`` / ``build.container_remove`` on the flat store (no scan
    layout); children ``vq_codec`` and ``pq_codec`` (``pq_codec.codebook`` is ``[M, d / M, 16]``);
  * ``train`` is IVFPQIndex's with 16 codewords: the coarse quantizer, then 16-means of the sub-vectors (of the residuals
    x - vq(x) for a residual index); ``encode`` / ``decode`` keep IVFPQIndex's contracts, with codes 0..15 unpacked;
  * ``search`` runs IVFPQ's coarse stage and visiting rule, then scores every live slot of the visited cells on the
    query's [M][16] LUT (``tpq_ivfpq4_search``, csrc/ivfpq4.cu): m ascending from +0, plus the cell's coarse similarity
    for a residual index.  Order: score descending, then address ascending.
Not covered: ``range_search``, ``search_cells``, ``scan_push`` and multi-GPU.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .modules import Codec, IdContainer, StreamCache, _fingerprint, on_index_device

MAX_SUBVECTORS = 256                 # a 16 KB LUT in the scan CTA's shared memory
_PART2_CHUNK_BYTES = 64 << 20        # scratch of one tpq_relayout_part2 call when the residual table is built


def _pack_codes(codes):
    """[M, n] codes 0..15 -> [M / 2, n] u8, byte j = code 2 j | code 2 j + 1 << 4 (tpq_store_codes' input)."""
    c = codes.to(torch.uint8)
    return (c[0::2] | (c[1::2] << 4)).contiguous()


def _unpack_codes(packed):
    """[M / 2, n] u8 -> [M, n] u8 codes 0..15: _pack_codes's inverse."""
    out = torch.stack([packed & 15, packed >> 4], dim=1)            # [M / 2, 2, n]
    return out.reshape(2 * packed.shape[0], packed.shape[1]).contiguous()


class IVFPQ4Index(IdContainer):
    def __init__(self, d_vector, n_subvectors=16, n_cells=128, initial_size=None, expand_step_size=128,
                 expand_mode="double", distance="euclidean", device="cuda:0", pq_use_residual=False, verbose=0):
        super().__init__()
        if distance not in ("euclidean", "cosine"):
            raise NotImplementedError(f"IVFPQ4Index supports euclidean and cosine distance, not {distance!r}")
        if n_subvectors > MAX_SUBVECTORS:
            raise NotImplementedError(f"IVFPQ4Index: n_subvectors={n_subvectors} > {MAX_SUBVECTORS} is not supported")
        assert n_subvectors > 0 and n_subvectors % 8 == 0, \
            f"n_subvectors={n_subvectors} must be a positive multiple of 8 (code_size = n_subvectors / 2 whole words)"
        assert d_vector > 0 and d_vector % n_subvectors == 0, f"d_vector={d_vector} must be a multiple of n_subvectors"
        assert not pq_use_residual or distance == "euclidean", "residual IVFPQ is defined on euclidean residuals"
        assert expand_mode in ("step", "double") and expand_step_size > 0
        if initial_size is None:
            initial_size = expand_step_size
        assert initial_size >= 0 and n_cells > 0
        self.d_vector, self.n_subvectors, self.d_subvector = d_vector, n_subvectors, d_vector // n_subvectors
        self.n_cells, self.code_size, self.contiguous_size = n_cells, n_subvectors // 2, 4
        self.distance, self.device, self.verbose = distance, device, verbose
        self.initial_size, self.expand_step_size, self.expand_mode = initial_size, expand_step_size, expand_mode
        self.pq_use_residual = bool(pq_use_residual)
        self.n_probe = 1
        self.use_smart_probing = True
        self.smart_probing_temperature = 30.0
        self._max_id = -1
        self._has_holes = False
        self._id2address_fp = None
        self._part2 = None                                               # (codebooks' fingerprint, StreamCache of the table)
        dev = torch.device(device)
        cap = n_cells * initial_size
        self.register_buffer("_address2id", -torch.ones(cap, dtype=torch.long, device=dev))
        self.register_buffer("_id2address", None)
        self.register_buffer("_storage", torch.zeros(n_subvectors // 8, cap, 4, dtype=torch.uint8, device=dev))
        self.register_buffer("_cell_start", torch.arange(n_cells, device=dev) * initial_size)
        self.register_buffer("_cell_size", torch.zeros(n_cells, dtype=torch.long, device=dev))
        self.register_buffer("_cell_capacity", torch.zeros(n_cells, dtype=torch.long, device=dev) + initial_size)
        self.register_buffer("_is_empty", torch.ones(cap, dtype=torch.uint8, device=dev))
        self.vq_codec = Codec()
        self.pq_codec = Codec()

    @property
    def n_items(self):
        return int((self._is_empty == 0).sum().item())

    def load_state_dict(self, state_dict, strict=True):
        """As IVFPQIndex.load_state_dict: the buffers, then ``_max_id`` re-derived and holes assumed."""
        super().load_state_dict(state_dict, strict)
        assert self._storage.dtype == torch.uint8 and self._storage.shape == (self.n_subvectors // 8, self.capacity, 4)
        self._has_holes = True
        self._refresh_max_id()

    # ------------------------------------------------------------------ build side
    @on_index_device
    def train(self, x, force_retrain=False, seed=0):
        """IVFPQIndex.train with 16 codewords: build.train_coarse, then 16-means (25 iterations) of the sub-vectors of
        x, or of its residuals x - vq(x) for a residual index."""
        if self.vq_codec.is_trained and self.pq_codec.is_trained and not force_retrain:
            self.print_message("index is already trained", 1)
            return
        from . import build
        x, vq = build.train_coarse(self, x, seed=seed)
        if self.pq_use_residual:
            x = x - vq[:, build._assign(x[None].contiguous(), vq[None])[0]]
        sub = x.reshape(self.n_subvectors, self.d_subvector, x.shape[1]).contiguous()
        pq = build.multi_kmeans(sub, 16, 25, seed=seed + 1, distance=self.distance).contiguous()
        self.vq_codec.set_codebook(vq)
        self.pq_codec.set_codebook(pq)
        self._part2 = None

    @on_index_device
    def encode(self, x):
        """x [d_vector, n] -> codes [n_subvectors, n] u8, values 0..15 (residual index: (pq_code of x - vq centroid,
        vq_code)), as IVFPQIndex.encode."""
        assert x.dim() == 2 and x.shape[0] == self.d_vector
        from . import build, fn
        x = x.contiguous()
        if self.distance == "cosine":
            x = fn.normalize(x)
        cells, codes = build.encode(self, x)
        return (codes, cells) if self.pq_use_residual else codes

    def _codebook256(self):
        """pq_codec's [M, dsub, 16] codebook zero-padded to the [M, dsub, 256] that tpq_pq_decode and
        tpq_relayout_part2 read: codes 0..15 read only the first 16 words, so the results are exact."""
        pq = self.pq_codec.codebook
        out = torch.zeros(self.n_subvectors, self.d_subvector, 256, dtype=torch.float32, device=pq.device)
        out[:, :, :16] = pq
        return out

    @on_index_device
    def decode(self, code):
        """codes [n_subvectors, n] u8 -> [d_vector, n] f32 (residual index: code = (pq_code, vq_code) -> vq centroid +
        decoded residual), as IVFPQIndex.decode."""
        from . import fn
        if self.pq_use_residual:
            assert len(code) == 2
            pq_code, vq_code = code
            assert pq_code.shape[0] == self.n_subvectors and pq_code.shape[1] == vq_code.shape[0]
            return self.vq_codec.codebook[:, vq_code] + fn.pq_decode(self._codebook256(), pq_code)
        assert code.dim() == 2 and code.shape[0] == self.n_subvectors
        return fn.pq_decode(self._codebook256(), code)

    @on_index_device
    def add(self, x, ids=None, return_address=False, chunk: int = 1 << 20):
        """x [d_vector, n] fp32: cell = exact assignment of x (normalised for cosine), code = its 4-bit PQ code, packed
        two per byte.  Placement, holes and expansion are IVFPQIndex's (build.container_add)."""
        assert x.dim() == 2 and x.shape[0] == self.d_vector and x.dtype == torch.float32
        assert self.vq_codec.is_trained and self.pq_codec.is_trained, "index is not trained"
        from . import build, fn
        x = x.to(self._storage.device)
        cells, codes = [], []
        for s in range(0, x.shape[1], chunk):
            xc = x[:, s:s + chunk].contiguous()
            if self.distance == "cosine":
                xc = fn.normalize(xc)
            c, q = build.encode(self, xc)
            cells.append(c)
            codes.append(_pack_codes(q))
        cells = torch.cat(cells) if cells else torch.empty(0, dtype=torch.long, device=x.device)
        codes = torch.cat(codes, 1) if codes else torch.empty(self.code_size, 0, dtype=torch.uint8, device=x.device)
        return build.container_add(self, codes.contiguous(), cells, ids, return_address)

    @on_index_device
    def remove(self, ids=None, address=None):
        """As IVFPQIndex.remove: removed slots become holes that search skips and the next add fills first;
        ``_cell_size`` is not decremented."""
        from . import build
        build.container_remove(self, ids, address)

    def _codes_at(self, address):
        """[M, n] unpacked codes of the slots `address` (an index tensor in [0, capacity))."""
        words = self._storage[:, address, :]                             # [M / 8, n, 4]
        return _unpack_codes(words.permute(0, 2, 1).reshape(self.code_size, -1))

    def get_data_by_address(self, address):
        """[d_vector, n] decoded vectors at `address` (a residual index adds the centroid of the slot's cell); zeros
        where the address is outside [0, capacity)."""
        assert address.dtype == torch.int64
        address = address.to(self._storage.device)
        mask = (0 <= address) & (address < self.capacity)
        if address.numel() == 0 or self.capacity == 0:
            return torch.zeros(self.d_vector, address.numel(), dtype=torch.float32, device=self._storage.device)
        a = torch.where(mask, address, 0)
        codes = self._codes_at(a)
        if self.pq_use_residual:
            cells = torch.searchsorted(self._cell_start, a, right=True) - 1
            data = self.decode((codes, cells))
        else:
            data = self.decode(codes)
        return data * mask.to(data.dtype)[None, :]

    # ------------------------------------------------------------------ search
    def _part2_table(self):
        """Residual: part2 [n_cells, M, 16], the cell half of each cell's LUT, (-2 c_m . p) - |p|^2 in lut.cuh's
        arithmetic.  Built by tpq_relayout_part2 on the zero-padded codebook, a chunk of cells at a time; kept until a
        codebook changes."""
        vq, pq = self.vq_codec.kmeans.centroids, self.pq_codec.kmeans.centroids
        key = _fingerprint(vq, pq)
        if self._part2 is None or self._part2[0] != key:
            M, d, C, dev = self.n_subvectors, self.d_vector, self.n_cells, vq.device
            mg = (M + 63) // 64
            pq256 = self._codebook256()
            table = torch.empty(C, M, 16, dtype=torch.float32, device=dev)
            step = max(1, _PART2_CHUNK_BYTES // lib.tpq_part2_scan_bytes(M, 1))
            st = _lib.current_stream(dev)
            for c0 in range(0, C, step):
                n = min(step, C - c0)
                vqc = vq[:, c0:c0 + n].contiguous()
                scan = torch.empty(lib.tpq_part2_scan_bytes(M, n) // 4, dtype=torch.float32, device=dev)
                check(lib.tpq_relayout_part2(ptr(vqc), ptr(pq256), d, M, n, ptr(scan), st))
                # scan layout [n][MG][256][64] (scan_layout.cuh): entry (m, code) at group m / 64, row code, column m % 64
                table[c0:c0 + n] = scan.view(n, mg, 256, 64)[:, :, :16, :].permute(0, 1, 3, 2).reshape(n, mg * 64, 16)[:, :M]
            self._part2 = (key, StreamCache(table, dev))
        return self._part2[1].get()

    def _check_query(self, x, k):
        assert x.dim() == 2 and x.shape[0] == self.d_vector
        assert 0 < k <= 1024
        assert x.dtype == torch.float32 and x.device == self._storage.device
        assert x.device.type == "cuda", "torchpq_b200 has no CPU path: the index must live on a CUDA device"
        return x.contiguous()

    @on_index_device
    def search(self, x, k=1, return_address=False):
        """x [d_vector, n_query] fp32 on the index device -> (values [n_query, k] fp32 descending, ids [n_query, k]
        int64[, address]), -inf / -1 where fewer than k items were visited.  Probes as IVFPQIndex.search (n_probe,
        use_smart_probing, smart_probing_temperature)."""
        x = self._check_query(x, k)
        dev, nq, n_probe = x.device, x.shape[1], int(self.n_probe)
        values = torch.empty(nq, k, dtype=torch.float32, device=dev)
        ids = torch.empty(nq, k, dtype=torch.long, device=dev)
        address = torch.empty(nq, k, dtype=torch.long, device=dev) if return_address else None
        out = (values, ids, address) if return_address else (values, ids)
        if nq == 0:                                                      # an empty batch has no storage to point at
            return out
        assert self.vq_codec.is_trained and self.pq_codec.is_trained, "index is not trained"
        part2 = self._part2_table() if self.pq_use_residual else None
        d, M, C = self.d_vector, self.n_subvectors, self.n_cells
        ws_bytes = lib.tpq_ivfpq4_workspace_bytes(d, nq, C, n_probe, k)
        ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
        check(lib.tpq_ivfpq4_search(ptr(x), d, M, nq, _lib.METRIC[self.distance], ptr(self._storage),
                                    ptr(self._is_empty), ptr(self._cell_start), ptr(self._cell_size),
                                    ptr(self._address2id), self.capacity, C, ptr(self.vq_codec.kmeans.centroids),
                                    ptr(self.pq_codec.kmeans.centroids), ptr(part2), None, None, None, n_probe,
                                    int(bool(self.use_smart_probing)), float(self.smart_probing_temperature), k,
                                    ptr(values), ptr(ids), ptr(address), ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return out
