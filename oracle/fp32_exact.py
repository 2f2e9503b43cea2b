"""Bit-exact fp32 restatements of the search path's own kernels (TEST INFRASTRUCTURE, see ``oracle/__init__.py``).

``ivfpq_oracle`` restates the *reference* (torch fp32, sub-quantizers summed in ascending m); the tuned kernels sum
and multiply in other, fully determined orders, so on real-valued data they agree with it only to a tolerance.  The
functions here restate each query-side kernel of ``torchpq_b200/csrc`` operation for operation -- the same
``fmaf`` chains, the same separately rounded products and sums, the same summation order -- so that a GPU result
must equal them bit for bit on any input, not just on integer-valued states.  Each docstring cites the kernel lines
it restates.  Every value is float32; every float32 operation is a single IEEE round-to-nearest-even step (numpy's
float32 add / mul / div / sqrt are), and ``fma32`` is a correctly rounded fused multiply-add.

Smart probing (``expf`` / ``log2f`` and shuffle-order sums) has no bit-exact restatement; ``smart_probing_check``
bounds the GPU's result against a float64 evaluation instead.
"""
from __future__ import annotations

import math

import numpy as np

from . import ivfpq_oracle as O

F32 = np.float32
_TWO = F32(2.0)
_MINUS_TWO = F32(-2.0)
_EPS_NORM = F32(1e-9)            # util.normalize's `+ 1e-9`, as the float literal 1e-9f of coarse.cu:51


# ----------------------------------------------------------------------------------------- correctly rounded fma
def fma32(a, b, c):
    """fp32 fused multiply-add a * b + c with ONE rounding (round to nearest, ties to even), vectorised.

    The product of two fp32 values is exact in float64, so only the sum s = p + c is rounded there; rounding s to
    fp32 afterwards is a second rounding that is wrong exactly when s lands on an fp32 tie (the midpoint of two
    neighbouring fp32 values) while p + c itself does not.  TwoSum gives the exact error e of s (p + c == s + e); on
    such a tie the correct result is the neighbour on the side of e.  Subnormal results, signed zeros, overflow to
    infinity and NaN/inf operands follow IEEE 754 (an fp32 tie is a float64 value in every range, and e is exact
    because p and c are finite float64 values far from float64's own overflow)."""
    a, b, c = (np.asarray(v, F32) for v in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    c64 = c.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)                             # TwoSum: p + c == s + e exactly
        r = s.astype(F32)
        fin = np.isfinite(s)
        r64 = np.where(np.isinf(r) & fin, np.copysign(2.0 ** 128, s), r.astype(np.float64))
        d = s - r64                                                 # exact (Sterbenz): r is s's fp32 neighbour
        toward = np.where(d > 0, F32(np.inf), F32(-np.inf))
        nb = np.nextafter(r, toward)
        nb64 = np.where(np.isinf(nb), np.copysign(2.0 ** 128, nb.astype(np.float64)), nb.astype(np.float64))
        tie = fin & (d != 0) & (2.0 * d == nb64 - r64)
        fix = tie & (e != 0) & ((e > 0) == (d > 0))                 # the exact value lies beyond the midpoint
    out = np.where(fix, nb, r)
    return out.astype(F32) if out.ndim else F32(out)


def fma_chain(x, y, acc=None):
    """acc = fmaf(x[i], y[i], acc) for i ascending along axis 0, from +0 (or `acc`)."""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    shape = np.broadcast_shapes(x.shape[1:], y.shape[1:])
    acc = np.zeros(shape, F32) if acc is None else np.asarray(acc, F32)
    for i in range(x.shape[0]):
        acc = fma32(x[i], y[i], acc)
    return acc


def sum_sq_rounded(v):
    """s = __fadd_rn(s, __fmul_rn(v[i], v[i])) for i ascending along axis 0, from +0: every square rounded."""
    v = np.asarray(v, F32)
    s = np.zeros(v.shape[1:], F32)
    for i in range(v.shape[0]):
        s = s + v[i] * v[i]
    return s


# ----------------------------------------------------------------------------------------- coarse stage (coarse.cu)
_CR_G = 32


def _col_groups(x, fused):
    """col_sumsq (coarse.cu:19-33): row group g sums rows i = g, g + 32, ... ascending from +0 (fmaf(v, v, s) when
    `fused`, else __fadd_rn(s, __fmul_rn(v, v))); the 32 partials are then added in ascending group order from +0."""
    x = np.asarray(x, F32)
    d, n = x.shape
    t = np.zeros(n, F32)
    for g in range(_CR_G):
        rows = x[g::_CR_G]
        s = fma_chain(rows, rows, np.zeros(n, F32)) if fused else sum_sq_rounded(rows)
        t = t + s
    return t


def col_sqnorm(x):
    """col_sqnorm_kernel (coarse.cu:36-42): out[j] = sum_i x[i, j]^2 over [d, n], squares separately rounded."""
    return _col_groups(x, fused=False)


def normalize_columns(x):
    """normalize_columns_kernel (coarse.cu:45-53): x / (sqrtf(sum_i fmaf chain of x^2) + 1e-9f), __fdiv_rn."""
    x = np.asarray(x, F32)
    nrm = np.sqrt(_col_groups(x, fused=True)) + _EPS_NORM
    return (x / nrm[None, :]).astype(F32)


def coarse_sims(x, cb):
    """coarse_gemm_kernel (coarse.cu:59-138): sims[q, c] = ((acc * 2) - xn[q]) - cn[c], acc = fmaf chain over i
    ascending from +0 (:110, zero-padded K slabs add nothing), xn / cn from col_sqnorm (:253-254), epilogue :129-131.
    x [d, nq], cb [d, C] -> [nq, C]."""
    x, cb = np.asarray(x, F32), np.asarray(cb, F32)
    acc = fma_chain(x[:, :, None], cb[:, None, :])
    y = acc * _TWO
    y = y - col_sqnorm(x)[:, None]
    return (y - col_sqnorm(cb)[None, :]).astype(F32)


def score_to_ord(v):
    """common.cuh:34-41: the order-preserving uint32 image of an fp32 score (so +0 ranks above -0)."""
    b = np.asarray(v, F32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def probe_select(sims, n_probe):
    """probe_select_kernel (coarse.cu:142-179): per row the n_probe largest keys (score_to_ord(score) << 32 | ~cell),
    i.e. descending in the key order of common.cuh, ties to the lower cell.  -> (probe_sims [nq, n_probe] f32,
    cells [nq, n_probe] i64)."""
    sims = np.asarray(sims, F32)
    nq, C = sims.shape
    ords = score_to_ord(sims).astype(np.int64)
    order = np.argsort(-ords, axis=1, kind="stable")[:, :n_probe]   # stable: equal keys keep ascending cell order
    return np.take_along_axis(sims, order, axis=1), order.astype(np.int64)


def coarse_probe(x, cb, n_probe):
    """tpq_coarse_probe (coarse.cu:235-266) without smart probing: (probe_sims, cells)."""
    return probe_select(coarse_sims(x, cb), n_probe)


# ----------------------------------------------------------------------------------------- LUT builders
def _split(x, M):
    """x [d, nq] -> [M, dsub, nq] (sub-vector m = rows m * dsub .. m * dsub + dsub - 1)."""
    x = np.asarray(x, F32)
    return x.reshape(M, x.shape[0] // M, x.shape[1])


def lut_entries(x, pq, kind):
    """One LUT entry per (m, q, code), the arithmetic of lut.cuh:23-35 that lut_kernel (lut.cu:18-68), build_lut
    (lut.cuh:40-79) and so cell_lut_kernel (scan.cu:654-659) share: dot = fmaf chain of
    x_m[i] * p_m[i][code] over i ascending from +0; |x_m|^2 and |p|^2 are sums of separately rounded squares;
    kind "euclidean": ((dot * 2) - |x_m|^2) - |p|^2; "cosine": dot; "part1" (residual query half): dot * 2.
    x [d, nq], pq [M, dsub, 256] -> [M, nq, 256]."""
    pq = np.asarray(pq, F32)
    M, dsub, _ = pq.shape
    xs = _split(x, M)                                           # [M, dsub, nq]
    dot = fma_chain(np.moveaxis(xs, 1, 0)[:, :, :, None], np.moveaxis(pq, 1, 0)[:, :, None, :])   # [M, nq, 256]
    if kind == "cosine":
        return dot
    if kind == "part1":
        return (dot * _TWO).astype(F32)
    assert kind == "euclidean", kind
    a2 = sum_sq_rounded(np.moveaxis(xs, 1, 0))                  # [M, nq]
    b2 = sum_sq_rounded(np.moveaxis(pq, 1, 0))                  # [M, 256]
    return ((dot * _TWO - a2[:, :, None]) - b2[:, None, :]).astype(F32)


def build_lut(x, pq, distance):
    """lut_kernel in the reference layout (lut.cu:65), the LUT of tpq_build_lut / fn.precompute_adc: [M, nq, 256]."""
    return lut_entries(x, pq, distance)


def lut_scan(x, pq, distance, residual=False):
    """The LUT in scan layout (scan_layout.cuh:17-18), per query and sub-quantizer: [nq, m_pad, 256], the rows of
    padding sub-quantizers m >= M +0 (lut_kernel, lut.cu:64-65; build_lut reads zero sub-vectors and a zero-padded
    codebook, relayout.cu:76).  residual: the query half part1 = dot * 2 (lut.cuh:32)."""
    pq = np.asarray(pq, F32)
    M = pq.shape[0]
    mp = (M + 31) // 32 * 32
    v = lut_entries(x, pq, "part1" if residual else distance)  # [M, nq, 256]
    out = np.zeros((v.shape[1], mp, 256), F32)
    out[:, :M] = np.moveaxis(v, 1, 0)
    return out


def part2(vq, pq):
    """tpq_relayout_part2 (relayout.cu:91-101: lut_kernel, kind part 2, lut.cuh:27, :33): part2[c, m, code] =
    (dot * -2) - nrm * nrm, dot = fmaf chain of vq[m * dsub + i, c] * pq[m, i, code], nrm = sqrtf(fmaf chain of
    pq[m, i, code]^2), i ascending from +0;
    padding sub-quantizers +0.  vq [d, C], pq [M, dsub, 256] -> [C, m_pad, 256]."""
    pq = np.asarray(pq, F32)
    M, dsub, _ = pq.shape
    C = np.asarray(vq).shape[1]
    mp = (M + 31) // 32 * 32
    vs = np.moveaxis(_split(vq, M), 1, 0)                       # [dsub, M, C]
    pt = np.moveaxis(pq, 1, 0)                                  # [dsub, M, 256]
    dot = fma_chain(vs[:, :, :, None], pt[:, :, None, :])       # [M, C, 256]
    nrm = np.sqrt(fma_chain(pt, pt))                            # [M, 256]
    y = (dot * _MINUS_TWO - (nrm * nrm)[:, None, :]).astype(F32)
    out = np.zeros((C, mp, 256), F32)
    out[:, :M] = np.moveaxis(y, 1, 0)
    return out


# ----------------------------------------------------------------------------------------- the scan
def rot_subq(t, lane):
    """scan_layout.cuh:31: the sub-quantizer in record byte t of lane `lane`."""
    return (t & ~31) + ((lane + t) & 31)


def scan_scores(st, lut, addr, lane, base=F32(0)):
    """The score one scan lane forms for each address (adc_unit scan.cu:73-82, process_block :123-127,
    key_of_block :140-147, the cell-major kernel :614-616): record byte t of lane l holds sub-quantizer rot_subq(t, l)
    (code 0 for padding); acc[J] sums the LUT entries of record bytes t = J, J + 4, ... in ascending t from +0 (a
    64-sub-quantizer unit at a time; at m_pad 96 the last unit is 32 bytes, the same ascending t);
    score = base + ((acc0 + acc1) + (acc2 + acc3)).
    lut [m_pad, 256] fp32; addr, lane [n]; base: scalar (residual: the cell's coarse similarity; else +0)."""
    mp = lut.shape[0]
    M = st.n_subvectors
    codes = O.codes_at(st, addr)                                # [M, n]
    acc = [np.zeros(addr.shape[0], F32) for _ in range(4)]
    cols = np.arange(addr.shape[0])
    for t in range(mp):
        m = rot_subq(t, lane)                                   # [n]
        live = m < M
        code = np.where(live, codes[np.minimum(m, M - 1), cols], 0)
        acc[t & 3] = acc[t & 3] + lut[m, code]
    return (F32(base) + ((acc[0] + acc[1]) + (acc[2] + acc[3]))).astype(F32)


def _cell_lanes(st, addr):
    """The lane of each address: its offset from the start of its cell, mod 32 (blocks of 32 start at cell_start)."""
    cell = np.searchsorted(st.cell_start, addr, side="right") - 1
    return ((addr - st.cell_start[cell]) & 31).astype(np.int64)


def search_cells_fp32(st, x, cells, n_probe_list, k, base_sims=None, residual=False, part2_table=None):
    """tpq_ivfpq_search_cells (scan.cu:1100-1110): the scan of caller-supplied probe lists, in the kernels' own
    arithmetic.  x [d, nq] is used as given (no cosine normalisation, as there); the visiting rule is the oracle's
    (plain: O.effective_probes / O.probed_addresses; residual: P = clip((int) n_probe_list, 0, n_probe), entries whose
    start equals the previous entry's skipped, ivfpq_topk.cu:1080-1104), the selection O.select_topk.
    -> (values [nq, k] f32, address [nq, k] i64)."""
    x = np.asarray(x, F32)
    cells = np.asarray(cells, np.int64)
    nq, n_probe = cells.shape
    npl = np.asarray(n_probe_list)
    luts = lut_scan(x, st.pq_codebook, st.distance, residual)
    vals = np.empty((nq, k), F32)
    adr = np.empty((nq, k), np.int64)
    live = st.is_empty == 0
    if not residual:
        P = O.effective_probes(npl, n_probe)
        for q in range(nq):
            a = O.probed_addresses(st.cell_start[cells[q]], st.cell_size[cells[q]], int(P[q]))
            a = a[live[a]]
            vals[q], adr[q] = O.select_topk(scan_scores(st, luts[q], a, _cell_lanes(st, a)), a, k)
        return vals, adr
    p2 = part2(st.vq_codebook, st.pq_codebook) if part2_table is None else part2_table
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
            lut = (luts[q] + p2[c]).astype(F32)                 # store_precomputed_to_smem: part1 + part2 (scan.cu:343-346)
            sc.append(scan_scores(st, lut, a, (a - s) & 31, base[q, j]))
            ad.append(a)
        vals[q], adr[q] = O.select_topk(np.concatenate(sc), np.concatenate(ad), k)
    return vals, adr


def search_fp32(st, x, k, residual=False, n_probe_list=None):
    """tpq_ivfpq_search (scan.cu:1112-1122) in the kernels' arithmetic: cosine queries normalised (normalize_columns),
    coarse probe (coarse_sims + probe_select), then search_cells_fp32 with the probe similarities as the residual
    base.  n_probe_list: the per-query list lengths; None = n_probe without smart probing, else the oracle's smart
    probing of the restated probe similarities (not bit-exact: pass the GPU's own list to pin bits).
    -> (values, address, (x_used, probe_sims, cells, n_probe_list))."""
    x = np.asarray(x, F32)
    if st.distance == "cosine":
        x = normalize_columns(x)
    sims, cells = coarse_probe(x, st.vq_codebook, st.n_probe)
    if n_probe_list is None:
        if st.use_smart_probing and st.n_probe > 1:
            import torch
            n_probe_list = O.smart_probing(torch.from_numpy(sims), st.n_probe, st.smart_probing_temperature).numpy()
        else:
            n_probe_list = np.full(x.shape[1], st.n_probe, np.int64)
    v, a = search_cells_fp32(st, x, cells, n_probe_list, k, base_sims=sims, residual=residual)
    return v, a, (x, sims, cells, np.asarray(n_probe_list))


# ----------------------------------------------------------------------------------------- float64 error bounds
U32 = 2.0 ** -24                 # unit roundoff of fp32


def coarse_bound(x, cb):
    """A bound on |coarse_sims - exact| per entry: every fp32 operation of the restatement is one rounding, so the
    fma chain, both norm sums and the epilogue each err by at most (their length) * u * (sum of magnitudes)."""
    x, cb = np.asarray(x, np.float64), np.asarray(cb, np.float64)
    d = x.shape[0]
    mag = 2 * np.abs(x).T @ np.abs(cb) + (x * x).sum(0)[:, None] + (cb * cb).sum(0)[None, :]
    return (d + 4) * U32 * mag * (1 + 1e-6)


def smart_probing_check(probe_sims, npl_gpu, n_probe, temperature, safety=2.0):
    """Smart probing (coarse.cu:180-215) against float64: H * n_probe from the GPU's own probe similarities, with a
    margin derived from the error of each fp32 step -- the z values (sqrtf, __fdiv_rn: 2u relative, then z - max),
    expf (2 ulp), the n-term sums (n u), __fdiv_rn for p, log2f (1 ulp), the products and the final * n -- times
    `safety`.
    Returns a dict of row masks and counts; the caller asserts:
      ordinary rows (no p near 2^-150): exactly ceil(v) outside the margin, floor or ceil inside it;
      NaN rows: min p < 2^-152 (the fp32 p is 0, so p * log2f(p) is NaN) -> INT64_MIN; min p > 2^-147 -> not."""
    s = np.abs(np.asarray(probe_sims, np.float64))
    n = n_probe
    u = U32
    z = -np.sqrt(s) / temperature
    mx = z.max(axis=1, keepdims=True)
    w = z - mx
    with np.errstate(under="ignore", divide="ignore", invalid="ignore"):
        e = np.exp(w)
        tot = e.sum(axis=1, keepdims=True)
        p = e / tot
        lg = math.log2(n)
        t = np.where(p > 0, p * np.log2(p), 0.0)
    H = -t.sum(axis=1) / lg
    v = H * n
    dz = 2 * u * (np.abs(z) + np.abs(mx)) + u * np.abs(w)
    de = dz + 4 * u
    dsum = de.max(axis=1, keepdims=True) + n * u
    dp = de + dsum + u
    err = (np.abs(t) * (dp + 5 * u) + p * dp / math.log(2)).sum(axis=1) + n * u * np.abs(t).sum(axis=1)
    margin = safety * (n / lg * err + 3 * u * np.abs(v))
    pmin = p.min(axis=1)
    npl = np.asarray(npl_gpu, np.int64)
    nan_rows = pmin < 2.0 ** -152
    num_rows = pmin > 2.0 ** -147
    amb_rows = ~(nan_rows | num_rows)
    frac = v - np.floor(v)
    dist = np.minimum(frac, 1 - frac)
    inside = num_rows & (dist <= margin)
    lo, hi = np.ceil(v - margin).astype(np.int64), np.ceil(v + margin).astype(np.int64)
    in_range = (npl >= lo) & (npl <= hi)
    return dict(v=v, margin=margin, pmin=pmin, nan_rows=nan_rows, num_rows=num_rows, amb_rows=amb_rows,
                inside=inside, exact_ok=np.where(num_rows & ~inside, npl == np.ceil(v).astype(np.int64), True),
                range_ok=np.where(num_rows, in_range, True),
                nan_ok=np.where(nan_rows, npl == O.INT64_MIN, True) & np.where(num_rows, npl != O.INT64_MIN, True),
                amb_ok=np.where(amb_rows, in_range | (npl == O.INT64_MIN), True))
