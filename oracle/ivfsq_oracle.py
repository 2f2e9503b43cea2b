"""numpy restatement of ``torchpq_b200.IVFSQIndex`` and ``codec.SQCodec`` (TEST INFRASTRUCTURE, see ``oracle/__init__.py``).

Only the codec is new: ``encode`` / ``decode`` in float32 with each op rounded on its own, as the reference's torch
expressions (``torchpq/codec/SQCodec.py``) and ``tpq_sq_encode`` / ``tpq_sq_decode``:
  8 bits   code = clip(rint(((x - lower) / range) * 256), 0, 255)      x' = ((code / 256) * range) + lower
  16 bits  float16 round to nearest even / widening.
An IVFSQIndex searches as IVFFlatIndex over its decoded store, so ``state_of`` gives the ``ivfflat_oracle`` state
whose fp32 columns are the decoded codes, and ``search`` / ``search_cells`` are ``ivfflat_oracle``'s.
"""
from __future__ import annotations

import numpy as np

from . import ivfflat_oracle as VO

F32 = np.float32


def encode(x, bits, lower=None, range_=None):
    """x [d, n] f32 -> [d, n] u8 (bits 8) or f16 (bits 16)."""
    x = np.asarray(x, F32)
    if bits == 16:
        with np.errstate(over="ignore"):
            return x.astype(np.float16)
    lo, rg = np.asarray(lower, F32)[:, None], np.asarray(range_, F32)[:, None]
    with np.errstate(invalid="ignore"):
        q = np.rint(np.multiply(np.divide(np.subtract(x, lo), rg), F32(256)))
        return np.nan_to_num(np.clip(q, 0, 255), nan=0.0).astype(np.uint8)


def decode(code, bits, lower=None, range_=None):
    """[d, n] u8 (bits 8) or f16 (bits 16) -> [d, n] f32."""
    if bits == 16:
        return np.asarray(code, np.float16).astype(F32)
    lo, rg = np.asarray(lower, F32)[:, None], np.asarray(range_, F32)[:, None]
    q = np.divide(np.asarray(code, np.uint8).astype(F32), F32(256))
    return np.add(np.multiply(q, rg), lo)


def store_codes(index):
    """The [d, capacity] codes of an IVFSQIndex's store (word g of a slot: dimensions 4 g.. (8 bits), 2 g.. (16 bits))."""
    words = index._storage.cpu().numpy()                           # [code_size // 4, capacity, 4] u8
    d, cap = index.d_vector, words.shape[1]
    raw = np.ascontiguousarray(words.transpose(0, 2, 1)).reshape(-1, cap)    # [code_size, capacity], byte j of each slot
    if index.bits == 8:
        return raw
    return np.ascontiguousarray(raw.reshape(d, 2, cap).transpose(0, 2, 1)).view(np.float16).reshape(d, cap)


def bounds(index):
    """(lower, range) of the index's codec as f32 numpy (None for 16 bits)."""
    c = index.sq_codec
    if index.bits != 8:
        return None, None
    return c.lower.cpu().numpy().astype(F32), c.range.cpu().numpy().astype(F32)


def state_of(index):
    """The ivfflat_oracle IndexState of an IVFSQIndex: its buffers, with the decoded vectors as the fp32 store."""
    vq = index.vq_codec.kmeans.centroids
    st = VO.empty_state(index.d_vector, index.n_cells, 0, index.distance, None if vq is None else vq.cpu().numpy())
    lo, rg = bounds(index)
    x = np.ascontiguousarray(decode(store_codes(index), index.bits, lo, rg))
    st.storage = x.view(np.uint8).reshape(index.d_vector, -1, 4).copy()
    st.is_empty = index._is_empty.cpu().numpy().copy()
    st.cell_start = index._cell_start.cpu().numpy().copy()
    st.cell_size = index._cell_size.cpu().numpy().copy()
    st.cell_capacity = index._cell_capacity.cpu().numpy().copy()
    st.address2id = index._address2id.cpu().numpy().copy()
    st.max_id = int(index.max_id)
    return st


search = VO.search
search_cells = VO.search_cells
