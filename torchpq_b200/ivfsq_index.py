"""IVFSQIndex: inverted-file search over scalar-quantized vectors (Faiss ``IndexIVFScalarQuantizer``).

``IVFFlatIndex`` with the fp32 column replaced by its ``SQCodec`` code, d bytes per vector for 8 bits and 2 d for 16:

  * the container is IVFPQ's, buffer for buffer: ``_storage`` is u8 ``[code_size // 4, capacity, 4]``, IVFPQ's layout,
    with ``code_size = d`` (8 bits: word g of a slot holds dimensions 4 g .. 4 g + 3) or ``2 d`` (16 bits: dimensions
    2 g, 2 g + 1 as fp16); children ``vq_codec`` and ``sq_codec``;
  * ``train`` is IVFFlatIndex's coarse training (same data and seed -> same coarse codebook), then ``sq_codec.train`` on
    the same x (normalised for cosine); ``add`` assigns cells as IVFFlatIndex.add and stores ``sq_codec.encode`` of x
    (normalised for cosine, as IVFPQIndex encodes); ``remove`` leaves holes;
  * ``search`` is IVFFlatIndex's over the decoded store, bit for bit: the scan (``tpq_ivfsq_search``, csrc/ivfflat.cu)
    decodes each code as the GEMM tile stages it, with the codec's own arithmetic, and the norm table is
    ``tpq_flat_norms`` of the decoded store.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .codec import SQCodec
from .ivfflat_index import IVFFlatIndex
from .modules import StreamCache, _fingerprint, on_index_device

_NORM_CHUNK = 1 << 16            # slots decoded at a time by the norm table's build


class IVFSQIndex(IVFFlatIndex):
    _SEARCH, _RANGE = "tpq_ivfsq_search", "tpq_ivfsq_range_search"

    def __init__(self, d_vector, n_cells=128, bits=8, sq_mode="minmax", sq_alpha=1.0, initial_size=None,
                 expand_step_size=128, expand_mode="double", distance="euclidean", device="cuda:0", verbose=0):
        if bits not in (8, 16):
            raise NotImplementedError(f"IVFSQIndex supports 8 and 16 bits, not {bits}")
        assert d_vector > 0 and d_vector % (4 if bits == 8 else 2) == 0, \
            f"d_vector={d_vector} must be a multiple of {4 if bits == 8 else 2} for {bits}-bit codes"
        self.bits = bits
        super().__init__(d_vector, n_cells, initial_size, expand_step_size, expand_mode, distance, device, verbose)
        self.code_size = d_vector * bits // 8                            # bytes per item, moved in 4-byte granules
        self.sq_codec = SQCodec(bits=bits, alpha=sq_alpha, mode=sq_mode)

    def _empty_store(self, cap, dev):
        """A zero store of `cap` slots: u8 [code_size // 4, cap, 4], IVFPQ's layout."""
        return torch.zeros(self.d_vector * self.bits // 32, cap, 4, dtype=torch.uint8, device=dev)

    # ------------------------------------------------------------------ build side
    @on_index_device
    def train(self, x, force_retrain=False, seed=0):
        """IVFFlatIndex.train (build.train_coarse), then sq_codec.train on the same x (normalised for cosine)."""
        if self.vq_codec.is_trained and not force_retrain:
            self.print_message("index is already trained", 1)
            return
        from . import build
        xt, vq = build.train_coarse(self, x, seed=seed)
        self.vq_codec.set_codebook(vq)
        self.sq_codec.train(xt.contiguous())
        self._state_changed()

    def encode(self, x):
        """sq_codec.encode: x [d, n] fp32 -> [d, n] u8 (8 bits) or fp16 (16 bits)."""
        return self.sq_codec.encode(x)

    def decode(self, code):
        """sq_codec.decode: [d, n] codes -> [d, n] fp32."""
        return self.sq_codec.decode(code)

    @on_index_device
    def add(self, x, ids=None, return_address=False, chunk: int = 1 << 20):
        """x [d, n] fp32: cell = exact assignment of x (normalised for cosine), code = sq_codec.encode of that same x.
        Placement, holes and expansion are IVFPQIndex's (build.container_add)."""
        assert x.dim() == 2 and x.shape[0] == self.d_vector and x.dtype == torch.float32
        assert self.vq_codec.is_trained and self.sq_codec.is_trained, "index is not trained"
        from . import build, fn
        x = x.to(self._storage.device).contiguous()
        cells, codes = [], []
        for s in range(0, x.shape[1], chunk):
            xc = x[:, s:s + chunk].contiguous()
            if self.distance == "cosine":
                xc = fn.normalize(xc)
            cells.append(build._assign(xc[None], self.vq_codec.codebook[None])[0])
            codes.append(self._code_bytes(self.encode(xc)))
        n = x.shape[1]
        cells = torch.cat(cells) if cells else torch.empty(0, dtype=torch.long, device=x.device)
        codes = torch.cat(codes, 1) if codes else torch.empty(self.code_size, 0, dtype=torch.uint8, device=x.device)
        assert codes.shape == (self.code_size, n)
        return build.container_add(self, codes.contiguous(), cells, ids, return_address)   # calls _state_changed

    def _code_bytes(self, code):
        """[d, n] codes -> [code_size, n] u8, byte j of item i = byte j of its code (tpq_store_codes' input)."""
        if self.bits == 8:
            return code
        n = code.shape[1]
        return code.view(torch.uint8).view(self.d_vector, n, 2).permute(0, 2, 1).reshape(self.code_size, n)

    def _codes_at(self, address):
        """[d, n] codes of the slots `address` (an index tensor in [0, capacity), or a slice)."""
        words = self._storage[:, address, :]                             # [code_size // 4, n, 4] u8
        n = words.shape[1]
        if self.bits == 8:
            return words.permute(0, 2, 1).reshape(self.d_vector, n)
        return words.permute(0, 2, 1).reshape(self.d_vector // 2, 2, 2, n).permute(0, 1, 3, 2) \
                    .reshape(self.d_vector, n, 2).contiguous().view(torch.float16).view(self.d_vector, n)

    def get_data_by_address(self, address):
        """[d, n] decoded vectors at `address`; zeros where the address is outside [0, capacity)."""
        assert address.dtype == torch.int64
        address = address.to(self._storage.device)
        mask = (0 <= address) & (address < self.capacity)
        if address.numel() == 0 or self.capacity == 0:
            return torch.zeros(self.d_vector, address.numel(), dtype=torch.float32, device=self._storage.device)
        data = self.decode(self._codes_at(torch.where(mask, address, 0)).contiguous())
        return data * mask.to(data.dtype)[None, :]

    # ------------------------------------------------------------------ search
    def _norm_table(self):
        """tpq_flat_norms of the decoded store, built chunk by chunk (tpq_sq_decode, then tpq_flat_norms on the chunk),
        kept until the store changes."""
        key = _fingerprint(self._storage)
        if self._norms is None or self._norms[0] != key:
            dev, cap, d = self._storage.device, self.capacity, self.d_vector
            table = torch.empty(max(1, cap), dtype=torch.float32, device=dev)
            st = _lib.current_stream(dev)
            for s in range(0, cap, _NORM_CHUNK):
                n = min(_NORM_CHUNK, cap - s)
                x = self.decode(self._codes_at(slice(s, s + n)).contiguous())
                check(lib.tpq_flat_norms(ptr(x), n, d, n, _lib.METRIC[self.distance], ptr(table[s:]), st))
            self._norms = (key, StreamCache(table, dev))
        return self._norms[1].get()

    def _store_args(self):
        lo, rg = self.sq_codec._bounds(self._storage.device)               # None for 16 bits
        self._sq_bounds = (lo, rg)                                       # kept alive past the launch
        return ptr(self._storage), self.bits, ptr(lo), ptr(rg)
