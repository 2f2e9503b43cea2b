"""numpy restatement of ``torchpq_b200.IVFFlatIndex`` (TEST INFRASTRUCTURE, see ``oracle/__init__.py``).

The container is ``ivfpq_oracle``'s ``IndexState`` with fp32 columns: ``storage [d, capacity, 4]`` u8 holds the bytes of
the ``[d, capacity]`` f32 store (an item's code is its 4 d bytes, ``n_subvectors = 4 d``), so ``ivfpq_oracle``'s
placement (``container_add``) places vectors exactly as it places PQ codes.  ``search`` is the coarse probe of
``fp32_exact.coarse_probe`` (on ``fp32_exact.normalize_columns(x)`` for cosine), the IVFPQ visiting rule
(``visited``), the scores of ``flat_oracle.flat_sims`` and selection in key order (score descending, address ascending;
``fp32_exact.score_to_ord``), padded with (-inf, id -1, address -1).
"""
from __future__ import annotations

import numpy as np

from . import fp32_exact as X
from . import ivfpq_oracle as IO
from .flat_oracle import flat_sims

F32 = np.float32


def empty_state(d, n_cells, initial_size, distance="euclidean", vq_codebook=None) -> IO.IndexState:
    """A freshly constructed IVFFlatIndex: IVFPQ's container with 4 d code bytes per item."""
    cap = n_cells * initial_size
    vq = np.zeros((d, n_cells), F32) if vq_codebook is None else np.ascontiguousarray(vq_codebook, F32)
    return IO.IndexState(d_vector=d, n_subvectors=4 * d, n_cells=n_cells, distance=distance, vq_codebook=vq,
                         pq_codebook=np.zeros((0, 0, 256), F32), storage=np.zeros((d, cap, 4), np.uint8),
                         is_empty=np.ones(cap, np.uint8), cell_start=np.arange(n_cells, dtype=np.int64) * initial_size,
                         cell_size=np.zeros(n_cells, np.int64), cell_capacity=np.zeros(n_cells, np.int64) + initial_size,
                         address2id=-np.ones(cap, np.int64))


def codes_of(x):
    """x [d, n] f32 -> its [4 d, n] u8 code: byte 4 g + b of item i is byte b of x[g, i]."""
    x = np.ascontiguousarray(x, F32)
    d, n = x.shape
    return np.ascontiguousarray(x.view(np.uint8).reshape(d, n, 4).transpose(0, 2, 1).reshape(4 * d, n))


def add(st, x, cells, ids=None, expand_mode="double", expand_step_size=128):
    """ivfpq_oracle.container_add of x's fp32 columns into the given cells -> (ids, write address)."""
    return IO.container_add(st, codes_of(x), np.asarray(cells, np.int64), ids, expand_mode, expand_step_size)


def vectors(st):
    """The store as [d, capacity] f32."""
    return np.ascontiguousarray(st.storage).view(np.float32).reshape(st.d_vector, -1)


def state_of(index) -> IO.IndexState:
    """The IndexState of a torchpq_b200.IVFFlatIndex (its buffers, copied to the host)."""
    vq = index.vq_codec.kmeans.centroids
    st = empty_state(index.d_vector, index.n_cells, 0, index.distance,
                     None if vq is None else vq.cpu().numpy())
    st.storage = index._storage.cpu().numpy().view(np.uint8).reshape(index.d_vector, -1, 4).copy()
    st.is_empty = index._is_empty.cpu().numpy().copy()
    st.cell_start = index._cell_start.cpu().numpy().copy()
    st.cell_size = index._cell_size.cpu().numpy().copy()
    st.cell_capacity = index._cell_capacity.cpu().numpy().copy()
    st.address2id = index._address2id.cpu().numpy().copy()
    st.max_id = int(index.max_id)
    return st


def visited(st, cells_q, npl_q, n_probe):
    """Live addresses a query scans, in visiting order (a cell listed twice apart appears twice): its first
    probe_count = max(1, min((int32) n_probe_list, n_probe)) entries, skipping a cell outside [0, n_cells) and an entry
    whose cell_start equals the previous entry's (scan_layout.cuh, probe_count and probe_visits)."""
    C = st.n_cells
    P = int(IO.effective_probes(np.array([npl_q], np.int64), n_probe)[0])
    out = []
    for j in range(P):
        c = int(cells_q[j])
        if not 0 <= c < C:
            continue
        if j > 0:
            cp = int(cells_q[j - 1])
            if 0 <= cp < C and st.cell_start[c] == st.cell_start[cp]:
                continue
        s = int(st.cell_start[c])
        a = np.arange(s, s + int(st.cell_size[c]), dtype=np.int64)
        out.append(a[st.is_empty[a] == 0])
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def search_cells(st, x, cells, n_probe_list, k):
    """x [d, nq], cells [nq, n_probe], n_probe_list [nq] -> (values [nq, k] f32, ids, address [nq, k] i64)."""
    x = np.asarray(x, F32)
    cells, npl = np.asarray(cells, np.int64), np.asarray(n_probe_list, np.int64)
    nq, n_probe = x.shape[1], cells.shape[1]
    vals = np.full((nq, k), -np.inf, F32)
    adr = np.full((nq, k), -1, np.int64)
    sims = flat_sims(x, vectors(st), st.distance) if nq and st.capacity else None     # per (query, slot): batch-free
    for q in range(nq):
        a = visited(st, cells[q], npl[q], n_probe)
        if a.size == 0:
            continue
        s = sims[q, a]
        order = np.lexsort((a, -X.score_to_ord(s).astype(np.int64)))[:k]      # score descending, address ascending
        vals[q, :order.size], adr[q, :order.size] = s[order], a[order]
    ids = np.where(adr >= 0, st.address2id[np.maximum(adr, 0)], -1)
    return vals, ids, adr


def probe(st, x, n_probe):
    """The coarse stage of search with smart probing off: cells [nq, n_probe] of fp32_exact.coarse_probe on x
    (normalised as tpq_normalize_columns for cosine)."""
    x = np.asarray(x, F32)
    xp = X.normalize_columns(x) if st.distance == "cosine" else x
    return X.coarse_probe(xp, st.vq_codebook, n_probe)[1]


def search(st, x, k, n_probe):
    """IVFFlatIndex.search with use_smart_probing = False."""
    cells = probe(st, x, n_probe)
    return search_cells(st, x, cells, np.full(cells.shape[0], n_probe, np.int64), k)
