"""RefineFlatIndex in numpy (TEST INFRASTRUCTURE, see ``oracle/__init__.py``): the exact pass of ``tpq_refine_flat``
(csrc/refine.cu) and the search on top of a base index's candidate ids, in the kernel's fp32 arithmetic.  The score is
``ivfpqr_oracle.scores`` (the re-rank pass's fmaf chains, here on stored rows instead of reconstructions), the query's
normalisation ``fp32_exact.normalize_columns`` and the selection ``ivfpq_oracle.select_topk``.

    store      vectors [capacity, d] row-major, live slots the prefix [0, n_items), address2id [capacity]
    euclidean  acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0
    cosine     acc = fmaf(x_e, y_e, acc), x normalised by fp32_exact.normalize_columns, y as stored
    selection  score descending, then store address ascending; (-inf, -1, -1) padding
"""
from __future__ import annotations

import numpy as np

from . import fp32_exact as E
from . import ivfpq_oracle as O
from . import ivfpqr_oracle as R

F32 = np.float32


def state_of(ix):
    """(vectors, address2id, n_items) of a torchpq_b200.RefineFlatIndex, copied to the host."""
    h = lambda t: t.detach().cpu().numpy().copy()
    return h(ix._vectors), h(ix._address2id), ix.n_items


def addresses_of(ids, address2id, n_items):
    """The live store address of each id, -1 for -1 and for ids the store does not hold."""
    live = {int(i): a for a, i in enumerate(address2id[:n_items].tolist()) if i >= 0}
    ids = np.asarray(ids, np.int64)
    return np.vectorize(lambda i: live.get(int(i), -1), otypes=[np.int64])(ids) if ids.size else ids.copy()


def score_addresses(x, addr, vectors, distance):
    """Scores of addresses addr [nq, k1] (-1 = none, scored as row 0) for queries x [d, nq] -> [nq, k1] fp32: all
    queries at once through ivfpqr_oracle.scores, on the store rows as columns [d, k1, nq]."""
    x = np.asarray(x, F32)
    if distance == "cosine":
        x = E.normalize_columns(x)
    y = np.asarray(vectors, F32)[np.where(addr >= 0, addr, 0)]          # [nq, k1, d]
    return R.scores(x, np.ascontiguousarray(y.transpose(2, 1, 0)), distance).T


def refine(x, cand_ids, vectors, address2id, n_items, distance, k):
    """tpq_refine_flat behind RefineFlatIndex.refine: x [d, nq], candidate ids [nq, k1] -> (values, ids, address)
    [nq, k].  Ids the store does not hold are dropped; an id listed twice is scored twice."""
    cand_ids = np.asarray(cand_ids, np.int64)
    nq = cand_ids.shape[0]
    addr = addresses_of(cand_ids, address2id, n_items)
    s = score_addresses(x, addr, vectors, distance) if nq and addr.shape[1] else np.zeros(addr.shape, F32)
    vals = np.empty((nq, k), F32)
    adr = np.empty((nq, k), np.int64)
    for q in range(nq):
        ok = addr[q] >= 0
        vals[q], adr[q] = O.select_topk(s[q][ok], addr[q][ok], k)
    return vals, O.get_id_by_address(address2id, adr), adr


def search(x, k, k_factor, base_search, vectors, address2id, n_items, distance):
    """RefineFlatIndex.search: base_search(x, k1) -> candidate ids [nq, k1] with k1 = ivfpqr_oracle.k1_of(k, k_factor),
    then refine."""
    return refine(x, base_search(x, R.k1_of(k, k_factor)), vectors, address2id, n_items, distance, k)


def brute_force(x, k, vectors, address2id, n_items, distance):
    """The exact top-k over every live item: refine with every stored id as a candidate of every query."""
    nq = np.asarray(x).shape[1]
    live_ids = address2id[:n_items]
    return refine(x, np.broadcast_to(live_ids, (nq, n_items)), vectors, address2id, n_items, distance, k)
