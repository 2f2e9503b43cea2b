"""numpy restatement of IVFPQ range search (TEST INFRASTRUCTURE, in the spirit of ``oracle/``).

``range_search_cells_fp32`` / ``range_search_fp32`` are ``fp32_exact.search_cells_fp32`` / ``search_fp32`` with the
top-k replaced by a filter: every live slot of every visited cell whose score -- ``fp32_exact.scan_scores``, the scan
kernels' own arithmetic, plus the cell's coarse similarity for a residual index -- is > float32(t).  The visiting
rules are those restatements' (plain: ``ivfpq_oracle.effective_probes`` / ``probed_addresses``; residual: the first
clip(n_probe_list, 0, n_probe) entries, an entry skipped when its start equals the previous entry's).  The result is
``range_oracle.csr``'s (lims, values, ids, address).
"""
from __future__ import annotations

import numpy as np

from oracle import fp32_exact as X
from oracle import ivfpq_oracle as O
from range_oracle import csr

F32 = np.float32


def visited_scores(st, x, cells, n_probe_list, base_sims=None, residual=False, part2_table=None):
    """Per query, (scores, addresses) of every live slot the scan visits, in visiting order."""
    x = np.asarray(x, F32)
    cells = np.asarray(cells, np.int64)
    nq, n_probe = cells.shape
    npl = np.asarray(n_probe_list)
    luts = X.lut_scan(x, st.pq_codebook, st.distance, residual)
    live = st.is_empty == 0
    out = []
    if not residual:
        P = O.effective_probes(npl, n_probe)
        for q in range(nq):
            a = O.probed_addresses(st.cell_start[cells[q]], st.cell_size[cells[q]], int(P[q]))
            a = a[live[a]]
            out.append((X.scan_scores(st, luts[q], a, X._cell_lanes(st, a)), a))
        return out
    p2 = X.part2(st.vq_codebook, st.pq_codebook) if part2_table is None else part2_table
    base = np.asarray(base_sims, F32)
    P = np.clip(npl.astype(np.int64).astype(np.int32).astype(np.int64), 0, n_probe)
    for q in range(nq):
        sc, ad = [np.zeros(0, F32)], [np.zeros(0, np.int64)]
        prev = None
        for j in range(int(P[q])):
            c = int(cells[q, j])
            s, n = int(st.cell_start[c]), int(st.cell_size[c])
            if j > 0 and s == prev:
                continue
            prev = s
            a = np.arange(s, s + n, dtype=np.int64)
            a = a[live[a]]
            lut = (luts[q] + p2[c]).astype(F32)
            sc.append(X.scan_scores(st, lut, a, (a - s) & 31, base[q, j]))
            ad.append(a)
        out.append((np.concatenate(sc), np.concatenate(ad)))
    return out


def range_search_cells_fp32(st, x, cells, n_probe_list, t, base_sims=None, residual=False, part2_table=None):
    """tpq_ivfpq_range_search with the probe lists given: x [d, nq] used as given -> CSR (lims, values, ids, address)."""
    t = F32(t)
    parts = []
    for s, a in visited_scores(st, x, cells, n_probe_list, base_sims, residual, part2_table):
        keep = s > t
        parts.append((s[keep], a[keep]))
    return csr(parts, st.address2id)


def range_search_fp32(st, x, t, residual=False, n_probe_list=None):
    """IVFPQIndex.range_search in the kernels' arithmetic (cosine normalisation and the coarse probe of
    fp32_exact.search_fp32).  n_probe_list: as there (None without smart probing)."""
    x = np.asarray(x, F32)
    if st.distance == "cosine":
        x = X.normalize_columns(x)
    sims, cells = X.coarse_probe(x, st.vq_codebook, st.n_probe)
    if n_probe_list is None:
        assert not (st.use_smart_probing and st.n_probe > 1), "pass the GPU's n_probe_list to pin smart probing"
        n_probe_list = np.full(x.shape[1], st.n_probe, np.int64)
    return range_search_cells_fp32(st, x, cells, n_probe_list, t, base_sims=sims, residual=residual)
