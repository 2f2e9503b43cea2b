"""numpy restatement of ``torchpq_b200.IVFPQ4Index.search`` (TEST INFRASTRUCTURE, see ``oracle/__init__.py``).

Built on the existing pieces: the state is an ``ivfpq_oracle.IndexState`` whose ``pq_codebook`` is ``[M, dsub, 16]``
and whose ``storage`` is ``[M / 8, capacity, 4]`` u8 of packed codes (code m in nibble m & 1, low first, of byte m >> 1);
the probe is ``fp32_exact.coarse_probe``; the LUT is ``fp32_exact.lut_entries`` (any codeword count) and, residual,
``fp32_exact.part2`` on the codebook zero-padded to 256 words; the visiting rule and the top-k are ``ivfpq_oracle``'s.

The kernel's arithmetic (csrc/ivfpq4.cu): acc = fp32 sum of LUT[m][code_m] over m ascending from +0, one rounding per
add; score = base + acc, base = the cell's coarse similarity (residual) or +0; residual LUT = part1 + part2[cell], one
fp32 add per entry.  Keys: score descending, then address ascending; padding (-inf, -1).
"""
from __future__ import annotations

import numpy as np

from . import fp32_exact as FX
from . import ivfpq_oracle as O

F32 = np.float32


# ----------------------------------------------------------------------------------------- packing
def pack(codes):
    """[M, n] codes 0..15 -> [M / 2, n] u8: byte j = code 2 j | code 2 j + 1 << 4."""
    c = np.asarray(codes, np.uint8)
    return (c[0::2] | (c[1::2] << 4)).astype(np.uint8)


def unpack(packed):
    """[M / 2, n] u8 -> [M, n] u8: pack's inverse."""
    p = np.asarray(packed, np.uint8)
    return np.stack([p & 15, p >> 4], axis=1).reshape(2 * p.shape[0], p.shape[1])


def storage_words(codes):
    """[M, n] codes -> the [M / 8, n, 4] u8 a store holds for these items (word g = sub-quantizers 8 g .. 8 g + 7)."""
    b = pack(codes)                                              # [M / 2, n]
    return np.ascontiguousarray(b.reshape(b.shape[0] // 4, 4, b.shape[1]).transpose(0, 2, 1))


def codes_at(st, address):
    """[M, n] unpacked codes of the slots `address`."""
    w = st.storage[:, np.asarray(address, np.int64), :]             # [M / 8, n, 4]
    return unpack(w.transpose(0, 2, 1).reshape(st.n_subvectors // 2, -1))


def state_of(index):
    """The IndexState of a torchpq_b200.IVFPQ4Index (numpy copies of its buffers)."""
    cpu = lambda t: t.detach().cpu().numpy().copy()
    return O.IndexState(
        d_vector=index.d_vector, n_subvectors=index.n_subvectors, n_cells=index.n_cells, distance=index.distance,
        vq_codebook=cpu(index.vq_codec.codebook), pq_codebook=cpu(index.pq_codec.codebook), storage=cpu(index._storage),
        is_empty=cpu(index._is_empty), cell_start=cpu(index._cell_start), cell_size=cpu(index._cell_size),
        cell_capacity=cpu(index._cell_capacity), address2id=cpu(index._address2id), max_id=index.max_id,
        n_probe=int(index.n_probe), use_smart_probing=bool(index.use_smart_probing),
        smart_probing_temperature=float(index.smart_probing_temperature))


# ----------------------------------------------------------------------------------------- LUT
def luts(x, pq, distance, residual=False):
    """[nq, M, 16]: lut.cuh's entries (fp32_exact.lut_entries) of x [d, nq] against pq [M, dsub, 16]; residual: the
    query half 2 dot."""
    return np.ascontiguousarray(np.moveaxis(FX.lut_entries(x, pq, "part1" if residual else distance), 1, 0))


def part2_table(vq, pq):
    """[C, M, 16]: the cell half of the residual LUT (fp32_exact.part2 on the codebook zero-padded to 256 words)."""
    pq = np.asarray(pq, F32)
    M = pq.shape[0]
    pq256 = np.zeros(pq.shape[:2] + (256,), F32)
    pq256[:, :, :16] = pq
    return np.ascontiguousarray(FX.part2(vq, pq256)[:, :M, :16])


def scores(codes, lut, base=F32(0)):
    """base + (sum over m ascending from +0 of lut[m, codes[m]]), fp32.  codes [M, n], lut [M, 16]."""
    acc = np.zeros(codes.shape[1], F32)
    for m in range(codes.shape[0]):
        acc = acc + lut[m, codes[m]]
    return (F32(base) + acc).astype(F32)


# ----------------------------------------------------------------------------------------- search
def search_cells(st, x, cells, n_probe_list, k, base_sims=None, residual=False, part2=None):
    """The scan of given probe lists (tpq_ivfpq4_search with cells): x [d, nq] used as given.  Visiting rule: plain
    O.effective_probes + O.probed_addresses; residual P = clip((int) n_probe_list, 0, n_probe) with an entry skipped
    when its start equals the previous entry's.  -> (values [nq, k] f32, address [nq, k] i64)."""
    x = np.asarray(x, F32)
    cells = np.asarray(cells, np.int64)
    nq, n_probe = cells.shape
    npl = np.asarray(n_probe_list)
    L = luts(x, st.pq_codebook, st.distance, residual)
    vals, adr = np.empty((nq, k), F32), np.empty((nq, k), np.int64)
    live = st.is_empty == 0
    if not residual:
        P = O.effective_probes(npl, n_probe)
        for q in range(nq):
            a = O.probed_addresses(st.cell_start[cells[q]], st.cell_size[cells[q]], int(P[q]))
            a = a[live[a]]
            vals[q], adr[q] = O.select_topk(scores(codes_at(st, a), L[q]), a, k)
        return vals, adr
    p2 = part2_table(st.vq_codebook, st.pq_codebook) if part2 is None else part2
    base = np.asarray(base_sims, F32)
    P = np.clip(npl.astype(np.int64).astype(np.int32).astype(np.int64), 0, n_probe)
    for q in range(nq):
        sc, ad = [np.zeros(0, F32)], [np.zeros(0, np.int64)]
        for j in range(int(P[q])):
            c = int(cells[q, j])
            s, n = int(st.cell_start[c]), int(st.cell_size[c])
            if j > 0 and s == int(st.cell_start[cells[q, j - 1]]):
                continue
            a = np.arange(s, s + n, dtype=np.int64)
            a = a[live[a]]
            sc.append(scores(codes_at(st, a), (L[q] + p2[c]).astype(F32), base[q, j]))
            ad.append(a)
        vals[q], adr[q] = O.select_topk(np.concatenate(sc), np.concatenate(ad), k)
    return vals, adr


def search(st, x, k, residual=False, n_probe_list=None):
    """tpq_ivfpq4_search with the coarse stage inside: cosine queries normalised (fp32_exact.normalize_columns), the
    coarse probe (fp32_exact.coarse_probe), then search_cells with the probe similarities as the residual base.
    n_probe_list: the per-query list lengths (None: n_probe, i.e. no smart probing; pass the GPU's own list to pin
    smart probing).  -> (values, ids, address)."""
    x = np.asarray(x, F32)
    if st.distance == "cosine":
        x = FX.normalize_columns(x)
    sims, cells = FX.coarse_probe(x, st.vq_codebook, st.n_probe)
    if n_probe_list is None:
        n_probe_list = np.full(x.shape[1], st.n_probe, np.int64)
    v, a = search_cells(st, x, cells, n_probe_list, k, base_sims=sims, residual=residual)
    return v, O.get_id_by_address(st.address2id, a), a


def adc_float64(st, x, address, cells=None):
    """Plain float64 ADC of the items at `address` for the query columns x [d, nq] -> [nq, n]: euclidean
    -|x - y|^2, cosine x . y, where y is the decoded item (residual, `cells` given: its cell's centroid + the decoded
    residual; the LUT halves and the coarse similarity add up to exactly that)."""
    x = np.asarray(x, np.float64)
    pq = np.asarray(st.pq_codebook, np.float64)
    codes = codes_at(st, address)
    y = np.concatenate([pq[m][:, codes[m]] for m in range(pq.shape[0])], axis=0)        # [d, n]
    if cells is not None:
        y = y + np.asarray(st.vq_codebook, np.float64)[:, np.asarray(cells, np.int64)]
    if st.distance == "cosine":
        return x.T @ y
    return -((x[:, :, None] - y[:, None, :]) ** 2).sum(0)
