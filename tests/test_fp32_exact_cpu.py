"""CPU: oracle/fp32_exact.py -- a correctly rounded fp32 FMA, and fp32 restatements of the query-side kernels that
equal the reference oracle bit for bit where every value is an integer, and the exact result within a derived bound
on real-valued data.  Its GPU counterpart, tests/test_fp32_exact_gpu.py, requires the kernels to equal them bit for
bit."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import build_state as B, fp32_exact as X, ivfpq_oracle as O

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)


# ----------------------------------------------------------------------------------------- fma32
def _f32_of(fr: Fraction, zero_sign: float) -> F32:
    """The exact rational fr rounded to fp32, nearest, ties to even; `zero_sign` signs an exact zero."""
    if fr == 0:
        return F32(math_copysign0(zero_sign))
    neg, a = fr < 0, abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)                     # the fp32 quantum at this magnitude (subnormal below 2^-126)
    m = a / q
    r = m.numerator // m.denominator
    rem = m - r
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and r % 2 == 1):
        r += 1
    v = r * q
    out = np.inf if v >= Fraction(2) ** 128 else float(v)
    if out == 0:
        return F32(-0.0 if neg else 0.0)
    return F32(-out if neg else out)


def math_copysign0(s):
    return -0.0 if np.signbit(s) else 0.0


def fma_ref(a, b, c) -> F32:
    """fmaf by exact rational arithmetic: a * b + c, one rounding.  An exact zero is -0 only when both the product and
    c are -0 (IEEE 754 round to nearest)."""
    a, b, c = F32(a), F32(b), F32(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        with np.errstate(invalid="ignore", over="ignore"):
            return F32(float(a) * float(b) + float(c))
    p_neg = np.signbit(a) != np.signbit(b)
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    both_neg_zero = p_neg and (a == 0 or b == 0) and c == 0 and np.signbit(c)
    return _f32_of(exact, -0.0 if both_neg_zero else 0.0)


def _same(x, y):
    """Equal as fp32 bit patterns (so +0 != -0), NaN equal to NaN."""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    return np.array_equal(x.view(np.uint32), y.view(np.uint32)) or (np.isnan(x).all() and np.isnan(y).all())


def _check_all(a, b, c):
    got = X.fma32(a, b, c)
    bad = [i for i in range(len(a)) if not _same(got[i], fma_ref(a[i], b[i], c[i]))]
    assert not bad, [(a[i], b[i], c[i], got[i], fma_ref(a[i], b[i], c[i])) for i in bad[:5]]


def test_fma32_counterexample_of_float64_emulation():
    """a = b = 1 + 2^-12, c = 2^-60: the exact result lies just above the midpoint between 1 + 2^-11 and its fp32
    successor.  float64-then-fp32 rounds twice and lands on 1 + 2^-11; the correct answer is the successor."""
    a = F32(1 + 2.0 ** -12)
    c = F32(2.0 ** -60)
    twice = F32(float(a) * float(a) + float(c))                 # the former emulator
    assert twice == F32(1 + 2.0 ** -11)
    want = F32(1 + 2.0 ** -11 + 2.0 ** -23)
    assert fma_ref(a, a, c) == want
    assert X.fma32(a, a, c) == want
    assert X.fma32(a, a, -c) == F32(1 + 2.0 ** -11)             # just below the midpoint: the lower neighbour
    assert X.fma32(a, a, F32(0)) == F32(1 + 2.0 ** -11)         # exactly the midpoint: ties to even


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    n = 6000
    for lo, hi in ((-3, 3), (-40, 40), (-75, -55), (50, 64)):  # ordinary, wide, subnormal products, overflow
        a = (rng.standard_normal(n) * 2.0 ** rng.integers(lo, hi, n)).astype(F32)
        b = (rng.standard_normal(n) * 2.0 ** rng.integers(lo, hi, n)).astype(F32)
        p = a.astype(np.float64) * b.astype(np.float64)
        c = (-p * (1 + rng.standard_normal(n) * 2.0 ** rng.integers(-30, 0, n))).astype(F32)   # near-cancellation
        with np.errstate(over="ignore"):
            c[::3] = (rng.standard_normal(n) * 2.0 ** rng.integers(2 * lo, 2 * hi, n))[::3].astype(F32)
        _check_all(a, b, c)


def test_fma32_constructed_double_rounding():
    """Products that are exactly an fp32 midpoint (odd 13-bit mantissas whose product has 25 significant bits),
    nudged by a c far below float64's half-ulp so that the float64 sum rounds back onto the midpoint: the fp32 result
    must follow the sign of c.  Scaled into the normal and the subnormal range, with both signs."""
    rng = np.random.default_rng(1)
    i = rng.integers(0, 2 ** 11, 4000) * 2 + 1
    j = rng.integers(0, 2 ** 11, 4000) * 2 + 1
    mi, mj = (2 ** 12 + i), (2 ** 12 + j)
    keep = np.array([(int(x) * int(y)).bit_length() == 25 for x, y in zip(mi, mj)])
    mi, mj = mi[keep][:600], mj[keep][:600]
    n = mi.shape[0]
    assert n >= 300
    hits = 0
    for scale in (0, 40, -60, -75):                            # p near 2^0, 2^80, 2^-120, 2^-150 (subnormal results)
        a = (mi * 2.0 ** (-12 + scale)).astype(F32)
        b = (mj * 2.0 ** -12).astype(F32)
        b[1::2] = -b[1::2]
        p = a.astype(np.float64) * b.astype(np.float64)
        for rel in (2.0 ** -36, 2.0 ** -60):
            c = (np.abs(p) * rel * np.where(np.arange(n) % 4 < 2, 1, -1)).astype(F32)
            _check_all(a, b, c)
            old = (p + c.astype(np.float64)).astype(F32)
            hits += int((old != X.fma32(a, b, c)).sum())
    assert hits > 0                                            # the cases really do break float64-then-fp32 rounding


def test_fma32_signed_zeros_subnormals_overflow():
    t = 2.0 ** -100
    cases = [
        (0.0, 1.0, -0.0), (-0.0, 1.0, -0.0), (-1.0, 0.0, -0.0), (-1.0, 0.0, 0.0), (1.0, 1.0, -1.0), (-1.0, 1.0, 1.0),
        (t, t, 0.0), (-t, t, 0.0), (-t, t, -0.0), (t, t, -0.0),                           # underflow to a signed zero
        (2.0 ** -75, 2.0 ** -74, 0.0), (2.0 ** -75, 3 * 2.0 ** -75, 0.0),                 # 2^-149 and its midpoints
        (2.0 ** -75, 2.0 ** -75, 2.0 ** -149), (1.5 * 2.0 ** -75, 2.0 ** -75, -2.0 ** -149),
        (2.0 ** -70, 2.0 ** -60, -2.0 ** -126), (1e-20, 1e-20, 1e-45),
        (2.0 ** 127, 2.0, 0.0), (-2.0 ** 127, 2.0, 0.0), (FLT_MAX, 1.0, FLT_MAX), (FLT_MAX, 2.0, -FLT_MAX),
        (FLT_MAX, 1.0, 2.0 ** 103), (FLT_MAX, 1.0, 2.0 ** 102), (FLT_MAX, -1.0, -2.0 ** 103),
        (1 + 2.0 ** -23, FLT_MAX, -2.0 ** 104), (2.0 ** 64, 2.0 ** 64, -FLT_MAX),
        (np.inf, 0.0, 1.0), (np.inf, 1.0, -np.inf), (1.0, 1.0, np.inf), (np.nan, 1.0, 1.0),
    ]
    a, b, c = (np.array(v, F32) for v in zip(*cases))
    _check_all(a, b, c)
    assert np.signbit(X.fma32(F32(-t), F32(t), F32(0))) and not np.signbit(X.fma32(F32(1), F32(1), F32(-1)))
    assert np.isinf(X.fma32(F32(FLT_MAX), F32(1), F32(2.0 ** 103)))
    assert X.fma32(F32(FLT_MAX), F32(1), F32(2.0 ** 102)) == F32(FLT_MAX)


# ----------------------------------------------------------------------------------------- integer states: == oracle
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_integer_state_coarse_and_lut_equal_oracle(distance):
    st, queries = B.integer_state(48, 12, 37, 2000, seed=4, distance=distance)
    x = queries(45).numpy()
    sims = X.coarse_sims(x, st.vq_codebook)
    osims = O.negative_squared_l2(torch.from_numpy(x), torch.from_numpy(st.vq_codebook)).numpy()
    assert _same(sims, osims)
    ps, cells = X.probe_select(sims, 37)
    ops, ocells = O.topk_desc(torch.from_numpy(osims), 37)
    assert _same(ps, ops.numpy()) and np.array_equal(cells, ocells.numpy())
    lut = X.build_lut(x, st.pq_codebook, distance)
    assert _same(lut, O.precompute_adc(torch.from_numpy(x), torch.from_numpy(st.pq_codebook), distance).numpy())
    assert _same(X.col_sqnorm(x), (x.astype(np.float64) ** 2).sum(0).astype(F32))
    p1, p2 = O.residual_parts(torch.from_numpy(x), torch.from_numpy(st.vq_codebook), torch.from_numpy(st.pq_codebook))
    assert _same(X.lut_scan(x, st.pq_codebook, distance, residual=True)[:, :12], p1.numpy())
    assert _same(X.part2(st.vq_codebook, st.pq_codebook)[:, :12], p2.numpy())


@pytest.mark.parametrize("M,d,smart", [(8, 32, True), (16, 48, False), (96, 96, True), (40, 80, True)])
def test_integer_state_search_equals_oracle(M, d, smart):
    st, queries = B.integer_state(d, M, 16, 3000, seed=M)
    st.n_probe, st.use_smart_probing = 5, smart
    x = queries(20)
    ov, oi, oa = O.search(st, x, k=30, return_address=True)
    v, a, _ = X.search_fp32(st, x.numpy(), 30)
    assert _same(v, ov) and np.array_equal(a, oa)


def test_integer_state_residual_search_equals_oracle():
    st, queries = B.integer_state(16, 16, 16, 3000, seed=2)    # d/M = 1: sqrt(p^2)^2 == p^2, every score is an integer
    st.n_probe, st.use_smart_probing = 6, True
    x = queries(24)
    p2 = X.part2(st.vq_codebook, st.pq_codebook)
    assert _same(np.round(p2), p2)
    ov, oi, oa = O.search_residual(st, x, k=25, return_address=True)
    v, a, _ = X.search_fp32(st, x.numpy(), 25, residual=True)
    assert _same(v, ov) and np.array_equal(a, oa)


# ----------------------------------------------------------------------------------------- randn: within fp32 bounds
def test_randn_coarse_and_lut_within_float64_bound():
    """The restated coarse sims and LUT entries are the mathematical quantities up to a derived fp32 error bound:
    a restatement that computed something else (a wrong sign, a missing term) could not pass."""
    rng = np.random.default_rng(3)
    d, C, nq, M = 96, 70, 33, 24
    x = rng.standard_normal((d, nq)).astype(F32)
    cb = (rng.standard_normal((d, C)) * 0.7).astype(F32)
    x64, cb64 = x.astype(np.float64), cb.astype(np.float64)
    exact = 2 * x64.T @ cb64 - (x64 ** 2).sum(0)[:, None] - (cb64 ** 2).sum(0)[None, :]
    err = np.abs(X.coarse_sims(x, cb) - exact)
    assert (err <= X.coarse_bound(x, cb)).all()
    assert err.max() > 0                                       # the bound is not vacuous: fp32 really rounds here
    pq = rng.standard_normal((M, d // M, 256)).astype(F32)
    xs, p64 = x64.reshape(M, d // M, nq), pq.astype(np.float64)
    dot = np.einsum("miq,mic->mqc", xs, p64)
    mag = np.einsum("miq,mic->mqc", np.abs(xs), np.abs(p64))
    a2, b2 = (xs ** 2).sum(1)[:, :, None], (p64 ** 2).sum(1)[:, None, :]
    dsub = d // M
    u = X.U32
    eu = np.abs(X.build_lut(x, pq, "euclidean") - (2 * dot - a2 - b2))
    assert (eu <= (dsub + 3) * u * (2 * mag + a2 + b2) * (1 + 1e-6)).all()
    co = np.abs(X.build_lut(x, pq, "cosine") - dot)
    assert (co <= dsub * u * mag * (1 + 1e-6)).all()
    vq = rng.standard_normal((d, 5)).astype(F32)
    vs = vq.astype(np.float64).reshape(M, dsub, 5)
    p2 = X.part2(vq, pq)[:, :M]                                # [C, M, 256]
    want = -2 * np.einsum("mic,mik->cmk", vs, p64) - (p64 ** 2).sum(1)[None]
    bound = (dsub + 4) * u * (2 * np.einsum("mic,mik->cmk", np.abs(vs), np.abs(p64)) + (p64 ** 2).sum(1)[None]) * 1.01
    assert (np.abs(p2 - want) <= bound).all()


def _term_magnitudes(st, x, cells_q, residual):
    """[len(cells_q), M, 256] float64: for each probed cell, the sum of |terms| of every LUT entry (the quantities whose
    fp32 evaluation it is), for the re-association bound."""
    pq = np.abs(st.pq_codebook.astype(np.float64))
    M, dsub, _ = pq.shape
    xs = np.abs(np.asarray(x, np.float64)).reshape(M, dsub)
    dot = np.einsum("mi,mic->mc", xs, pq)
    if st.distance == "cosine":
        return np.broadcast_to(dot, (len(cells_q), M, 256))
    p2 = (pq ** 2).sum(1)
    if not residual:
        return np.broadcast_to(2 * dot + (xs ** 2).sum(1)[:, None] + p2, (len(cells_q), M, 256))
    vq = np.abs(st.vq_codebook.astype(np.float64)).reshape(M, dsub, -1)[:, :, cells_q]
    return 2 * dot[None] + 2 * np.einsum("mij,mic->jmc", vq, pq) + p2[None]


@pytest.mark.parametrize("kind", ["euclidean", "cosine", "residual"])
def test_randn_search_within_reordering_bound(kind):
    """search_cells_fp32 against the reference oracle on the same probe lists: each score differs from the oracle's
    by at most the fp32 error of its two evaluations (n = M + d/M + 6 roundings on any path: about n 2^-24 sum |terms|),
    so the k-th largest scores of a row differ by at most the largest such bound among the row's candidates.  A
    relative tolerance would not do: cosine sums cancel."""
    M, d = (24, 96) if kind != "residual" else (16, 64)
    rng = np.random.default_rng(4)
    distance = "cosine" if kind == "cosine" else "euclidean"
    st = B.randn_state(d, M, 12, 4000, seed=5, distance=distance)
    st.n_probe, st.use_smart_probing = 4, False
    x = torch.from_numpy(rng.standard_normal((d, 16)).astype(F32))
    xx, sims, cells, npl = O.coarse_probe(st, x)
    cn, s = cells.numpy(), sims.numpy()
    res = kind == "residual"
    if res:
        ov, oi = O.search_residual(st, x, k=40)
        v, _ = X.search_cells_fp32(st, xx.numpy(), cn, npl.numpy(), 40, base_sims=s, residual=True)
    else:
        ov, oi = O.search(st, x, k=40)
        v, _ = X.search_cells_fp32(st, xx.numpy(), cn, npl.numpy(), 40)
    n_terms = M + d // M + 6
    for q in range(x.shape[1]):
        mag = _term_magnitudes(st, xx.numpy()[:, q], cn[q], res)
        worst = 0.0
        for j in range(int(npl[q])):
            a0, n = int(st.cell_start[cn[q, j]]), int(st.cell_size[cn[q, j]])
            a = np.arange(a0, a0 + n)[st.is_empty[a0:a0 + n] == 0]
            tot = mag[j][np.arange(M)[:, None], O.codes_at(st, a)].sum(0) + (abs(s[q, j]) if res else 0.0)
            worst = max(worst, tot.max(initial=0.0))
        assert np.abs(v[q].astype(np.float64) - ov[q]).max() <= 2 * n_terms * X.U32 * worst, q
