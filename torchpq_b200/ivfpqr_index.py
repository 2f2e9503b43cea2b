"""Mirror of ``torchpq.index.IVFPQRIndex``: an IVFPQ index whose items also carry a second, finer PQ code that
re-ranks the first pass's candidates (Faiss: ``IndexIVFPQR``).

Same constructor arguments and defaults, attributes, codecs and registered buffers as the reference
(torchpq/index/IVFPQRIndex.py:7-107), so checkpoints interchange: ``_storage`` is ``[(M + Mr)/4, capacity, 4]``, the
first M/4 word planes an ``IVFPQIndex``'s scanned code and the next Mr/4 the re-rank code.  The container, the add
path and the first pass are ``IVFPQIndex``'s own; the second pass is ``tpq_rerank`` (csrc/rerank.cu).

Departures from the reference, where the class never worked:
  - ``search`` exists (the reference raises NotImplementedError): the IVFPQ scan returns k1 = min(1024, max(k,
    ceil(k_factor * k))) candidates, which are scored exactly on their reconstruction and cut to k;
  - ``k_factor`` (default 4, as in Faiss) is new, with the ``IVFPQIndex`` search attributes ``n_probe``,
    ``use_smart_probing`` and ``smart_probing_temperature``;
  - ``add`` works (the reference calls ``super(IVFPQIndex, self)`` without importing IVFPQIndex); cosine data is
    normalised once, where the reference's add and encode each normalise it;
  - ``train`` fits the re-rank codec (the reference trains ``pq_codec`` a second time), on x - decode_pq(encode_pq(x))
    with ``use_residual``, else on x;
  - ties go to the lower address, as in every top-k of this package.
Not covered, each with an error: ``drop_reference_layout`` / ``dist.distribute`` (the re-rank reads ``_storage``),
``search_cells``, ``scan_push`` and ``patch()``.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .index import IVFPQIndex
from .modules import Codec, k1_of, on_index_device


class IVFPQRIndex(IVFPQIndex):
    def __init__(self, d_vector, n_subvectors=8, n_subvectors_rerank=8, n_cells=128, use_residual=True,
                 initial_size=None, expand_step_size=128, expand_mode="double", distance="euclidean", device="cuda:0",
                 verbose=0):
        assert d_vector % n_subvectors_rerank == 0
        assert n_subvectors_rerank % 4 == 0, "code_size % contiguous_size(4) == 0"
        super().__init__(d_vector, n_subvectors, n_cells, initial_size, expand_step_size, expand_mode, distance, device,
                         pq_use_residual=False, verbose=verbose)
        self.n_subvectors_rerank = n_subvectors_rerank
        self.d_subvector_rerank = d_vector // n_subvectors_rerank
        self.use_residual = bool(use_residual)
        self.code_size = n_subvectors + n_subvectors_rerank              # IVFPQRIndex.py:28
        self.k_factor = 4
        del self._storage
        self.register_buffer("_storage", torch.zeros(self.code_size // 4, self.capacity, 4, dtype=torch.uint8,
                                                     device=torch.device(device)))
        self.pq_rerank_codec = Codec()

    # reference setters (IVFPQRIndex.py:74-99): k-means settings of each codec, read by train
    def set_vq_codec_max_iter(self, value): self.vq_codec.kmeans.max_iter = value
    def set_vq_codec_n_redo(self, value): self.vq_codec.kmeans.n_redo = value
    def set_vq_codec_tolerance(self, value): self.vq_codec.kmeans.tol = value
    def set_pq_codec_max_iter(self, value): self.pq_codec.kmeans.max_iter = value
    def set_pq_codec_n_redo(self, value): self.pq_codec.kmeans.n_redo = value
    def set_pq_codec_tolerance(self, value): self.pq_codec.kmeans.tol = value
    def set_pq_rerank_codec_max_iter(self, value): self.pq_rerank_codec.kmeans.max_iter = value
    def set_pq_rerank_codec_n_redo(self, value): self.pq_rerank_codec.kmeans.n_redo = value
    def set_pq_rerank_codec_tolerance(self, value): self.pq_rerank_codec.kmeans.tol = value

    # ------------------------------------------------------------------ codecs
    def _pq_encode(self, x, codebook, M):
        from . import build
        return build._assign(x.reshape(M, self.d_vector // M, x.shape[1]).contiguous(), codebook).to(torch.uint8)

    def _encode(self, x):
        """x [d, n], already normalised for cosine -> [M + Mr, n] u8 (IVFPQRIndex.py:128-154 after its normalise)."""
        from . import fn
        y1 = self._pq_encode(x, self.pq_codec.codebook, self.n_subvectors)
        if self.use_residual:
            x = x - fn.pq_decode(self.pq_codec.codebook, y1)
        y2 = self._pq_encode(x, self.pq_rerank_codec.codebook, self.n_subvectors_rerank)
        return torch.cat([y1, y2], dim=0)

    @on_index_device
    def encode(self, x):
        """IVFPQRIndex.encode (IVFPQRIndex.py:128-154): x [d_vector, n] -> [M + Mr, n] u8, the PQ code and the re-rank
        code (of the PQ code's residual with use_residual)."""
        assert len(x.shape) == 2 and x.shape[0] == self.d_vector
        from . import fn
        x = x.contiguous()
        if self.distance == "cosine":
            x = fn.normalize(x)
        return self._encode(x)

    @on_index_device
    def decode(self, code):
        """IVFPQRIndex.decode (IVFPQRIndex.py:156-175): [M + Mr, n] u8 -> [d, n] f32, the re-rank decode plus, with
        use_residual, the PQ decode."""
        from . import fn
        assert len(code.shape) == 2 and code.shape[0] == self.code_size
        y = fn.pq_decode(self.pq_rerank_codec.codebook, code[self.n_subvectors:])
        if self.use_residual:
            y = y + fn.pq_decode(self.pq_codec.codebook, code[:self.n_subvectors])
        return y

    # ------------------------------------------------------------------ build side
    @on_index_device
    def train(self, x, force_retrain=False, seed=0):
        """IVFPQRIndex.train (IVFPQRIndex.py:108-126) as meant: VQ and PQ on x (cosine: on the normalised x), then the
        re-rank codec on x - decode_pq(encode_pq(x)) with use_residual, else on x.  Each k-means runs build.fit with its
        codec's max_iter / tol / n_redo (defaults 15 / 1e-4 / 1 for VQ and 25 / 1e-4 / 1 for both PQs, as
        IVFPQIndex.train), from seeds seed, seed + 1 and seed + 2."""
        trained = self.vq_codec.is_trained and self.pq_codec.is_trained and self.pq_rerank_codec.is_trained
        if trained and not force_retrain:
            self.print_message("index is already trained", 1)
            return
        assert x.dim() == 2 and x.shape[0] == self.d_vector
        from . import build, fn

        def fit(data, k, codec, max_iter, seed_, distance):
            km = codec.kmeans
            return build.fit(data.contiguous(), k, getattr(km, "max_iter", max_iter), tol=getattr(km, "tol", 1e-4),
                             n_redo=getattr(km, "n_redo", 1), seed=seed_, distance=distance)[0].contiguous()

        x = x.contiguous()
        if self.distance == "cosine":
            x = fn.normalize(x)
        n, M, Mr = x.shape[1], self.n_subvectors, self.n_subvectors_rerank
        self.vq_codec.set_codebook(fit(x[None], self.n_cells, self.vq_codec, 15, seed, "euclidean")[0].contiguous())
        pq = fit(x.reshape(M, self.d_subvector, n), 256, self.pq_codec, 25, seed + 1, self.distance)
        self.pq_codec.set_codebook(pq)
        if self.use_residual:
            x = x - fn.pq_decode(pq, self._pq_encode(x, pq, M))
        pqr = fit(x.reshape(Mr, self.d_subvector_rerank, n), 256, self.pq_rerank_codec, 25, seed + 2, self.distance)
        self.pq_rerank_codec.set_codebook(pqr)
        self._state_changed()

    @on_index_device
    def add(self, x, ids=None, return_address=False, chunk: int = 1 << 20):
        """IVFPQRIndex.add (IVFPQRIndex.py:177-222): VQ cells and the [M + Mr] code of each column, stored by the
        container add of IVFPQIndex."""
        assert len(x.shape) == 2 and x.shape[0] == self.d_vector
        assert self._storage is not None, "search-only index: add to the full index (reload the checkpoint)"
        from . import build, fn
        cells_l, codes_l = [], []
        for s in range(0, x.shape[1], chunk):
            xc = x[:, s:s + chunk].contiguous()
            if self.distance == "cosine":
                xc = fn.normalize(xc)
            cells_l.append(build._assign(xc[None], self.vq_codec.codebook[None])[0])
            codes_l.append(self._encode(xc))
        return build.container_add(self, torch.cat(codes_l, 1), torch.cat(cells_l, 0), ids, return_address)

    # ------------------------------------------------------------------ search
    @on_index_device
    def search(self, x, k=1, return_address=False):
        """x [d_vector, n_query] fp32 -> (values [n_query, k] fp32 descending, ids [n_query, k] i64[, address]).
        First pass: the IVFPQ scan's k1 = min(1024, max(k, ceil(k_factor * k))) best addresses.  Second pass
        (tpq_rerank): every candidate scored exactly on its reconstruction -- euclidean -||x - y||^2, cosine <x/|x|, y>
        -- the k best kept; a value equals fn.max_sim(x_q, decode(codes)) bit for bit."""
        x = self._check_query(x, k)
        assert self.pq_rerank_codec.is_trained, "codec is not trained"
        k1 = k1_of(k, self.k_factor)
        _, _, cand = IVFPQIndex.search(self, x, k1, return_address=True)
        return self.rerank(x, cand, k, return_address)

    @on_index_device
    def rerank(self, x, candidates, k, return_address=False):
        """The second pass alone (tpq_rerank): x [d_vector, n_query] fp32, candidates [n_query, k1] i64 addresses
        (-1 = none), k <= k1 <= 1024 -> (values, ids[, address]) [n_query, k]."""
        x = self._check_query(x, k)
        assert candidates.dtype == torch.int64 and candidates.dim() == 2 and candidates.shape[0] == x.shape[1]
        cand = candidates.contiguous()
        dev, d, nq = x.device, self.d_vector, x.shape[1]
        values = torch.empty(nq, k, dtype=torch.float32, device=dev)
        ids = torch.empty(nq, k, dtype=torch.long, device=dev)
        address = torch.empty(nq, k, dtype=torch.long, device=dev) if return_address else None
        if nq > 0:
            ws_bytes = lib.tpq_rerank_workspace_bytes(d, nq, k)
            ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
            pq = self.pq_codec.codebook.contiguous()
            pqr = self.pq_rerank_codec.codebook.contiguous()
            check(lib.tpq_rerank(ptr(x), d, nq, ptr(cand), cand.shape[1], ptr(self._storage), self.capacity,
                                 self.n_subvectors, self.n_subvectors_rerank, ptr(pq), ptr(pqr), int(self.use_residual),
                                 _lib.METRIC[self.distance], k, ptr(self._address2id), ptr(values), ptr(ids), ptr(address),
                                 ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return (values, ids, address) if return_address else (values, ids)

    # ------------------------------------------------------------------ not covered
    def search_cells(self, *args, **kwargs):
        raise NotImplementedError("IVFPQRIndex.search_cells is not implemented: use search")

    def range_search(self, *args, **kwargs):
        # IVFPQIndex.range_search would return the first pass's ADC scores, not the re-ranked ones
        raise NotImplementedError("IVFPQRIndex.range_search is not implemented: its scores would not be re-ranked")

    def scan_push(self, *args, **kwargs):
        raise NotImplementedError("IVFPQRIndex has no fused multi-GPU scan: the re-rank pass reads _storage")

    def adopt_shard(self, *args, **kwargs):
        raise NotImplementedError("IVFPQRIndex cannot become shard-only: the re-rank pass reads _storage")

    def drop_reference_layout(self):
        raise NotImplementedError("IVFPQRIndex keeps _storage: the re-rank pass reads the codes from it")
