"""The host half of range search, shared by FlatIndex and IVFFlatIndex / IVFSQIndex.

The library's range entry points (``tpq_*_range_search``, include/tpq_b200.h) write every match as an unordered
(query, key) pair into a caller-owned buffer of ``cap`` entries and count the exact total on the device.  ``collect``
runs such an entry point, reads the total (the one host synchronisation of a range search), runs it once more with
``cap = total`` when the first buffer was too small, and sorts the pairs into Faiss's CSR form.
"""
from __future__ import annotations

import numpy as np
import torch

_FIRST_CAP_PER_QUERY = 1024      # the first buffer holds this many matches per query ...
_FIRST_CAP_MIN = 1 << 16         # ... but at least this many
_FIRST_CAP_MAX = 1 << 24         # ... and at most this many (12 B each: 192 MB)
_SIGN = -(1 << 63)               # the i64 with only the sign bit set


def threshold_f32(threshold) -> float:
    """A Python float or a 0-d tensor, rounded once to fp32 (to nearest); NaN raises ValueError."""
    if isinstance(threshold, torch.Tensor):
        if threshold.dim() != 0:
            raise ValueError(f"threshold must be a float or a 0-d tensor, got shape {tuple(threshold.shape)}")
        threshold = threshold.detach().to("cpu", torch.float64).item()     # exact for every narrower float
    t = np.float32(threshold)
    if np.isnan(t):
        raise ValueError("threshold is NaN")
    return float(t)


def first_cap(nq: int, max_results: int) -> int:
    return min(max_results, max(_FIRST_CAP_MIN, min(_FIRST_CAP_PER_QUERY * nq, _FIRST_CAP_MAX)))


def empty(nq, dev, return_address):
    lims = torch.zeros(nq + 1, dtype=torch.long, device=dev)
    out = (lims, torch.empty(0, dtype=torch.float32, device=dev), torch.empty(0, dtype=torch.long, device=dev))
    return out + (torch.empty(0, dtype=torch.long, device=dev),) if return_address else out


def collect(run, nq, max_results, address2id, return_address, dev):
    """run(keys, query, cap, total) launches one range pass into keys [cap] i64 (the u64 keys), query [cap] i32 and
    total [1] i64.  -> (lims [nq + 1] i64, values [nnz] f32, ids [nnz] i64[, address [nnz] i64]), each query's matches
    by score descending, then address ascending."""
    if max_results < 0:
        raise ValueError(f"max_results must be >= 0, got {max_results}")
    total = torch.zeros(1, dtype=torch.long, device=dev)
    cap = first_cap(nq, max_results)
    keys = torch.empty(cap, dtype=torch.long, device=dev)
    query = torch.empty(cap, dtype=torch.int32, device=dev)
    run(keys, query, cap, total)
    nnz = int(total.item())
    if nnz > max_results:
        raise ValueError(f"range_search: {nnz} results exceed max_results={max_results}")
    if nnz > cap:                                        # the exact total is known: one more pass writes every match
        keys = torch.empty(nnz, dtype=torch.long, device=dev)
        query = torch.empty(nnz, dtype=torch.int32, device=dev)
        run(keys, query, nnz, total)
    keys, query = keys[:nnz], query[:nnz]
    # CSR order: by key descending (u64 order is i64 order with the sign bit flipped), then, stably, by query
    order = torch.sort(keys ^ _SIGN, descending=True, stable=True).indices
    query = query[order]
    by_query = torch.sort(query, stable=True).indices
    keys, query = keys[order][by_query], query[by_query]
    lims = torch.searchsorted(query, torch.arange(nq + 1, dtype=torch.int32, device=dev)).to(torch.long)
    hi = (keys >> 32) & 0xFFFFFFFF                        # the score's order-preserving image
    bits = torch.where(hi >= 0x80000000, hi - 0x80000000, 0xFFFFFFFF - hi)
    values = torch.where(bits >= 0x80000000, bits - (1 << 32), bits).to(torch.int32).view(torch.float32)
    address = 0xFFFFFFFF - (keys & 0xFFFFFFFF)
    ids = address2id[address]
    return (lims, values, ids, address) if return_address else (lims, values, ids)
