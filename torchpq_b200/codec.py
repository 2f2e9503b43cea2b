"""Codecs (torchpq.codec).  ``SQCodec`` mirrors ``torchpq.codec.SQCodec`` (codec/SQCodec.py): per-dimension scalar
quantization of ``[d_vector, n]`` fp32 data to 8-bit codes, fp16 or fp32.

  * buffers: ``_is_trained``, ``lower``, ``upper``, ``binsize`` (always ``None``, as in the reference) and ``range``,
    so a ``state_dict`` moves between this codec and the reference's in both directions;
  * ``train`` runs the reference's own torch expressions on the caller's device (a one-off reduction, not the hot path):
    minmax ``lower = min, upper = max``, meanstd ``mean -+ alpha * std`` (unbiased std), then
    ``range = upper - lower + 1e-8``; bits 16 and 32 only set the trained flag;
  * ``encode`` / ``decode`` run the library's ``tpq_sq_encode`` / ``tpq_sq_decode`` kernels and are bit-identical to
    the reference's torch expressions (see include/tpq_b200.h and DESIGN.md section 6 for the quirks kept);
  * ``bits = 4`` (the reference packs dimension i with i + d/2 into one byte) is not built: NotImplementedError.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .modules import StateModule, on_device

__all__ = ["SQCodec"]


def _aligned(t):
    """t as a contiguous fp32 tensor whose data is 16-byte aligned (the scan reads lower / range 4 floats at a time)."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class SQCodec(StateModule):
    def __init__(self, bits=8, alpha=1.0, mode="minmax"):
        super().__init__()
        if bits not in (8, 16, 32):
            raise NotImplementedError(f"SQCodec supports 8, 16 and 32 bits, not {bits} (4-bit codes are not built)")
        assert mode in ("minmax", "meanstd"), f"unknown mode {mode!r}"
        self.bits, self.mode, self.alpha = bits, mode, alpha
        self.n_bins = 2 ** bits
        self.register_buffer("_is_trained", torch.tensor(False))
        self.register_buffer("lower", None)
        self.register_buffer("upper", None)
        self.register_buffer("binsize", None)
        self.register_buffer("range", None)

    def _trained(self, value: bool):
        assert type(value) == bool
        self._is_trained.data = torch.tensor(value)

    @property
    def is_trained(self) -> bool:
        return bool(self._is_trained.item())

    # ---------------------------------------------------------------- train: the reference's expressions
    def _train_minmax(self, x):
        self.register_buffer("lower", x.min(dim=-1)[0])
        self.register_buffer("upper", x.max(dim=-1)[0])
        self.register_buffer("range", self.upper - self.lower + 1e-8)

    def _train_meanstd(self, x):
        means = x.mean(dim=-1)
        stds = x.std(dim=-1)
        self.register_buffer("lower", means - self.alpha * stds)
        self.register_buffer("upper", means + self.alpha * stds)
        self.register_buffer("range", self.upper - self.lower + 1e-8)

    def train(self, x):
        """x [d_vector, n] fp32: fit lower / upper / range (bits 8); bits 16 and 32 have nothing to fit."""
        assert x.dim() == 2 and x.dtype == torch.float32
        if self.bits == 8:
            if self.mode == "minmax":
                self._train_minmax(x)
            else:
                self._train_meanstd(x)
        self._trained(True)

    # ---------------------------------------------------------------- encode / decode: library kernels
    def _bounds(self, device):
        """(lower, range) for the kernels: [d] fp32 on `device`, 16-byte aligned (None for bits 16 and 32)."""
        if self.bits != 8:
            return None, None
        lo, rg = self.lower, self.range
        assert lo is not None and rg is not None, "codec is not trained"
        assert lo.dtype == torch.float32 and rg.dtype == torch.float32
        assert lo.device == device and rg.device == device, "the codec's buffers live on another device"
        return _aligned(lo), _aligned(rg)

    @on_device(lambda self, x: x.device)
    def encode(self, x):
        """x [d_vector, n] fp32 CUDA -> [d_vector, n] u8 (bits 8), fp16 (bits 16), or x itself (bits 32)."""
        assert self.is_trained, "codec is not trained"
        if self.bits == 32:
            return x
        assert x.dim() == 2 and x.dtype == torch.float32 and x.device.type == "cuda"
        x = x.contiguous()
        d, n = x.shape
        lo, rg = self._bounds(x.device)
        if lo is not None:
            assert lo.shape == (d,)
        out = torch.empty(d, n, dtype=torch.uint8 if self.bits == 8 else torch.float16, device=x.device)
        check(lib.tpq_sq_encode(ptr(x), d, n, self.bits, ptr(lo), ptr(rg), ptr(out), _lib.current_stream(x.device)))
        return out

    @on_device(lambda self, code: code.device)
    def decode(self, code):
        """code [d_vector, n] u8 (bits 8), fp16 (bits 16) or fp32 (bits 32, returned as is) -> [d_vector, n] fp32."""
        assert self.is_trained, "codec is not trained"
        if self.bits == 32:
            return code
        assert code.dim() == 2 and code.device.type == "cuda"
        assert code.dtype == (torch.uint8 if self.bits == 8 else torch.float16)
        code = code.contiguous()
        d, n = code.shape
        lo, rg = self._bounds(code.device)
        if lo is not None:
            assert lo.shape == (d,)
        out = torch.empty(d, n, dtype=torch.float32, device=code.device)
        check(lib.tpq_sq_decode(ptr(code), d, n, self.bits, ptr(lo), ptr(rg), ptr(out), _lib.current_stream(code.device)))
        return out
