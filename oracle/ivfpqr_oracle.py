"""IVFPQRIndex in numpy (TEST INFRASTRUCTURE, see ``oracle/__init__.py``): the container with a code wider than the
scanned one, the reconstruction, the re-rank score and the selection of ``tpq_rerank`` (csrc/rerank.cu), restated in
the kernel's fp32 arithmetic on ``fp32_exact``'s correctly rounded fma.  The first pass is ``fp32_exact.search_fp32``
on the first M/4 word planes of the store, i.e. the IVFPQ search the index runs.

    reconstruction  y_e = y2_e + y1_e (use_residual) or y2_e
    euclidean       acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0
    cosine          acc = fmaf(x_e, y_e, acc), x normalised by fp32_exact.normalize_columns
    selection       score descending, then address ascending; (-inf, -1) padding
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from . import fp32_exact as E
from . import ivfpq_oracle as O

F32 = np.float32


def empty_state(d, M, Mr, n_cells, initial_size, distance="euclidean", vq_codebook=None, pq_codebook=None):
    """A fresh IVFPQRIndex container: IVFPQIndex's, with (M + Mr)/4 word planes in the store."""
    st = O.empty_state(d, M, n_cells, initial_size, distance, vq_codebook, pq_codebook)
    st.storage = np.zeros(((M + Mr) // 4, st.capacity, 4), np.uint8)
    return st


def container_add(st, codes, cells, ids=None, **kw):
    """O.container_add with [M + Mr, n] codes: placement does not depend on the code width."""
    M = st.n_subvectors
    st.n_subvectors = codes.shape[0]
    try:
        return O.container_add(st, codes, cells, ids, **kw)
    finally:
        st.n_subvectors = M


def state_of(ix):
    """The state of a torchpq_b200.IVFPQRIndex (buffers and first-level codebooks copied to the host; smart probing
    off) and its re-rank codebook."""
    h = lambda t: t.detach().cpu().numpy().copy()
    st = O.IndexState(ix.d_vector, ix.n_subvectors, ix.n_cells, ix.distance, h(ix.vq_codec.codebook),
                      h(ix.pq_codec.codebook), h(ix._storage), h(ix._is_empty), h(ix._cell_start), h(ix._cell_size),
                      h(ix._cell_capacity), h(ix._address2id), ix.max_id, int(ix.n_probe), False, 30.0)
    return st, h(ix.pq_rerank_codec.codebook)


def scanned(st):
    """The state the first pass scans: the first M/4 word planes of the store."""
    return dataclasses.replace(st, storage=np.ascontiguousarray(st.storage[:st.n_subvectors // 4]))


def codes_at(st, address):
    """[M + Mr, n] codes of the given addresses."""
    s = st.storage[:, address, :]
    return s.transpose(0, 2, 1).reshape(st.storage.shape[0] * 4, -1)


def pq_decode(codebook, code):
    """PQDecode: codebook [M, dsub, 256], code [M, n] -> [M * dsub, n] (a gather, no arithmetic)."""
    M, dsub, _ = codebook.shape
    return np.asarray(codebook, F32)[np.arange(M)[:, None, None], np.arange(dsub)[None, :, None],
                                     np.asarray(code, np.int64)[:, None, :]].reshape(M * dsub, -1)


def reconstruct(codes, M, pq, pqr, use_residual):
    """IVFPQRIndex.decode: y2 + y1 in fp32 (use_residual), else y2.  codes [M + Mr, n] -> [d, n]."""
    y = pq_decode(pqr, codes[M:])
    if use_residual:
        y = (y + pq_decode(pq, codes[:M])).astype(F32)
    return y


def scores(xq, y, distance):
    """The kernel's score of one (already normalised for cosine) query xq [d] against columns y [d, n]."""
    xq = np.asarray(xq, F32)[:, None]
    if distance == "euclidean":
        dif = (xq - y).astype(F32)
        return E.fma_chain(-dif, dif)
    return E.fma_chain(np.broadcast_to(xq, y.shape), y)


def rerank(x, cand, st, pq, pqr, use_residual, k):
    """tpq_rerank: x [d, nq], candidates [nq, k1] (-1 = none) -> (values, ids, address) [nq, k]."""
    x = np.asarray(x, F32)
    if st.distance == "cosine":
        x = E.normalize_columns(x)
    nq = x.shape[1]
    vals = np.empty((nq, k), F32)
    adr = np.empty((nq, k), np.int64)
    for q in range(nq):
        a = cand[q][(cand[q] >= 0) & (cand[q] < st.capacity)]
        y = reconstruct(codes_at(st, a), st.n_subvectors, pq, pqr, use_residual)
        vals[q], adr[q] = O.select_topk(scores(x[:, q], y, st.distance), a, k)
    return vals, O.get_id_by_address(st.address2id, adr), adr


def k1_of(k, k_factor):
    """The first pass's depth: min(1024, max(k, ceil(k_factor * k)))."""
    return min(1024, max(k, math.ceil(k_factor * k)))


def search(st, x, k, pqr, use_residual, k_factor=4, n_probe_list=None):
    """IVFPQRIndex.search: the first pass (fp32_exact.search_fp32, no smart probing unless n_probe_list is given) for
    k1 addresses, then rerank.  -> (values, ids, address, first-pass addresses)."""
    k1 = k1_of(k, k_factor)
    _, cand, _ = E.search_fp32(scanned(st), x, k1, n_probe_list=n_probe_list)
    v, i, a = rerank(x, cand, st, st.pq_codebook, pqr, use_residual, k)
    return v, i, a, cand
