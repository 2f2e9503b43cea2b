"""numpy restatement of range search (TEST INFRASTRUCTURE, in the spirit of ``oracle/``).

``flat_range_search`` is ``FlatIndex.range_search`` over the live prefix, ``ivfflat_range_search`` /
``ivfflat_range_search_cells`` are ``IVFFlatIndex.range_search`` on an ``ivfflat_oracle`` state (an IVFSQIndex's is
``ivfsq_oracle.state_of``, its decoded store).  The scores are ``flat_oracle.flat_sims``; an item matches when its score
is > float32(t); each query's matches are ordered by the key order of every top-k in the package (score descending by
the order-preserving image of the float, then address ascending), and the result is Faiss's CSR form
(lims [nq + 1], values, ids, address).
"""
from __future__ import annotations

import numpy as np

from oracle import fp32_exact as X
from oracle import ivfflat_oracle as VO
from oracle.flat_oracle import flat_sims

F32 = np.float32


def key_order(s, a):
    """Indices that sort scores s / addresses a by score descending (order-preserving image), then address ascending."""
    return np.lexsort((a, -X.score_to_ord(np.asarray(s, F32)).astype(np.int64)))


def csr(parts, address2id):
    """parts: per query (scores, addresses) already selected -> (lims, values, ids, address), each query in key order."""
    lims, vals, adrs = [0], [], []
    for s, a in parts:
        o = key_order(s, a)
        vals.append(np.asarray(s, F32)[o])
        adrs.append(np.asarray(a, np.int64)[o])
        lims.append(lims[-1] + o.size)
    values = np.concatenate(vals) if vals else np.zeros(0, F32)
    address = np.concatenate(adrs) if adrs else np.zeros(0, np.int64)
    ids = np.asarray(address2id, np.int64)[address] if address.size else np.zeros(0, np.int64)
    return np.asarray(lims, np.int64), values.astype(F32), ids, address


def flat_range_search(x, base_live, distance, t, address2id=None, sims=None):
    """x [d, nq], base_live [d, n] (the live prefix) -> CSR of every (q, c) with flat_sims[q, c] > float32(t).
    address2id defaults to the identity; sims: flat_sims(x, base_live, distance) when the caller has it."""
    x, base_live = np.asarray(x, F32), np.asarray(base_live, F32)
    nq, n = x.shape[1], base_live.shape[1]
    t = F32(t)
    a2i = np.arange(n, dtype=np.int64) if address2id is None else address2id
    if n == 0 or nq == 0:
        return csr([(np.zeros(0, F32), np.zeros(0, np.int64))] * nq, a2i)
    sims = flat_sims(x, base_live, distance) if sims is None else sims
    parts = []
    for q in range(nq):
        a = np.nonzero(sims[q] > t)[0].astype(np.int64)
        parts.append((sims[q, a], a))
    return csr(parts, a2i)


def ivfflat_range_search_cells(st, x, cells, n_probe_list, t, sims=None):
    """The IVF range search with the given probe lists: every live visited slot whose flat_sims score is > float32(t).
    sims: flat_sims(x, vectors(st), st.distance) when the caller has it."""
    x = np.asarray(x, F32)
    cells, npl = np.asarray(cells, np.int64), np.asarray(n_probe_list, np.int64)
    nq, n_probe = x.shape[1], cells.shape[1] if cells.ndim == 2 else 0
    t = F32(t)
    if sims is None and nq and st.capacity:
        sims = flat_sims(x, VO.vectors(st), st.distance)
    parts = []
    for q in range(nq):
        a = VO.visited(st, cells[q], npl[q], n_probe) if st.capacity else np.zeros(0, np.int64)
        s = sims[q, a] if a.size else np.zeros(0, F32)
        keep = s > t
        parts.append((s[keep], a[keep]))
    return csr(parts, st.address2id)


def ivfflat_range_search(st, x, t, n_probe, sims=None):
    """IVFFlatIndex.range_search with use_smart_probing = False (ivfflat_oracle.probe's cells)."""
    cells = VO.probe(st, x, n_probe)
    return ivfflat_range_search_cells(st, x, cells, np.full(cells.shape[0], n_probe, np.int64), t, sims)
