"""CPU: an executable specification of the packed arg-max in the epilogue of assign_tc_kernel
(torchpq_b200/csrc/assign_tc.cu: argmax_key / argmax_key_column and the loop around them).  The functions below
transliterate, in fp32 bit arithmetic, the key packing of every accumulator column, the per-thread fmaxf over its
columns chunk by chunk, the quad shuffle (xor 1, then xor 2, "all lanes at once") and the decode; they are checked
against a plain arg-max with the lowest index winning ties, which is what the exact kernel and the oracle return.
The GPU tests check the kernel's labels; this file pins the packing where no GPU is needed."""
import numpy as np
import pytest

F32, U32, I32 = np.float32, np.uint32, np.int32
INIT = F32(-3.0e38)                        # b0 / cb0 before the first column
PAD = F32(-1e30)                           # score of a padded column (j >= k)


def _bits(x):
    return np.asarray(x, F32).view(U32)


def _float(u):
    return np.asarray(u, U32).view(F32)


def argmax_key(score, rcol):
    """argmax_key(score, rcol = 255 ^ j): prmt.b32 u, score, 0, 0x321B (bytes 3..1 of the score, byte 0 = its sign bit
    replicated), then u ^ rcol."""
    u = _bits(score)
    prmt = (u & U32(0xFFFFFF00)) | np.where(u >> U32(31), U32(0xFF), U32(0)).astype(U32)
    return _float(prmt ^ U32(rcol))


def argmax_key_column(key):
    u = _bits(key)
    return 255 - ((u ^ (u.view(I32) >> 31).view(U32)) & U32(0xFF)).astype(np.int64)


def _thread_columns(tq, ch):
    """Columns of chunk ch held by quad thread tq, in the order the epilogue visits them: (8 i + 2 tq, + 1), i = 0..7."""
    return [(64 * ch + 8 * i + 2 * tq, 64 * ch + 8 * i + 2 * tq + 1) for i in range(8)]


def _padded(scores, nch):
    s = np.full(64 * nch, PAD, F32)
    s[:len(scores)] = scores
    return s


def packed_argmax(scores):
    """Label of one row (one of r0 / r1), k = len(scores) <= 256 columns, as the kernel computes it."""
    nch = (len(scores) + 63) // 64
    s = _padded(np.asarray(scores, F32), nch)
    b = [INIT] * 4                                        # per quad thread tq
    for tq in range(4):
        base = 255 ^ (2 * tq)
        for ch in range(nch):
            cb = INIT
            for i, (j0, j1) in enumerate(_thread_columns(tq, ch)):
                i0 = base ^ (64 * ch + 8 * i)
                assert (i0, i0 ^ 1) == (255 - j0, 255 - j1)
                cb = np.fmax(cb, np.fmax(argmax_key(s[j0], i0), argmax_key(s[j1], i0 ^ 1)))
            b[tq] = np.fmax(b[tq], cb)
    for o in (1, 2):                                      # __shfl_xor_sync: every lane reads the pre-stage value
        b = [np.fmax(b[tq], b[tq ^ o]) for tq in range(4)]
    assert all(_bits(x) == _bits(b[0]) for x in b)        # the four threads agree on the row's key
    return int(argmax_key_column(b[0])), b[0]


def packed_argmax_old(scores):
    """The packing before the sign-aware index field: 63 - (j mod 64) OR-ed in, chunks merged by a strict compare of
    the packed keys.  Kept to show what the specification catches."""
    nch = (len(scores) + 63) // 64
    s = _padded(np.asarray(scores, F32), nch)
    b, bi = [INIT] * 4, [0] * 4
    for ch in range(nch):
        cb = [INIT] * 4
        for tq in range(4):
            base = 63 - 2 * tq
            for i, (j0, j1) in enumerate(_thread_columns(tq, ch)):
                i0 = base - 8 * i
                k0 = _float((_bits(s[j0]) & U32(0xFFFFFF00)) | U32(i0))
                k1 = _float((_bits(s[j1]) & U32(0xFFFFFF00)) | U32(i0 - 1))
                cb[tq] = np.fmax(cb[tq], np.fmax(k0, k1))
        for o in (1, 2):
            cb = [np.fmax(cb[tq], cb[tq ^ o]) for tq in range(4)]
        for tq in range(4):
            if cb[tq] > b[tq]:
                b[tq], bi[tq] = cb[tq], 64 * ch + 63 - int(_bits(cb[tq]) & U32(0xFF))
    return bi[0]


def reference_argmax(scores):
    """Plain arg-max, lowest index among equal maxima; +0 == -0 as in the exact kernel's > / == compares."""
    s = np.asarray(scores, np.float64)
    return int(np.flatnonzero(s == s.max())[0])


def _check(scores):
    got, _ = packed_argmax(scores)
    assert got == reference_argmax(scores), (got, reference_argmax(scores), scores)


@pytest.mark.parametrize("k", [8, 60, 64, 100, 128, 132, 192, 196, 252, 256])
@pytest.mark.parametrize("sign", [1, -1, 0])
def test_random_ties_lowest_index(k, sign):
    """Half-integer scores from a small set: many exact ties inside a chunk and across chunks.  sign 0 mixes signs."""
    rng = np.random.default_rng(k * 3 + sign + 1)
    for _ in range(12):
        v = rng.integers(0, 12, k).astype(np.float64) * 0.5 + 1.0
        if sign == -1:
            v = -v
        elif sign == 0:
            v = v - 4.0                                    # negative, zero and positive
        _check(v.astype(F32))


@pytest.mark.parametrize("value", [5.5, -5.5, 0.0, -0.0, 1e-40, -1e-40, 3.0e38, -2.9e38, 2.0 ** 13 - 0.5, -(2.0 ** 13 - 0.5)])
@pytest.mark.parametrize("cols", [(3, 10), (10, 67), (3, 74), (0, 255), (130, 131), (1, 2, 65, 129, 193)])
def test_planted_ties(value, cols):
    """Equal best scores at the given columns, everything else lower: the lowest of them wins for every sign."""
    k = 256
    s = np.full(k, -1e4 if value > -1e4 else -3.0e38, F32)
    s[list(cols)] = F32(value)
    _check(s)
    if value > PAD:                                        # (scores below the padding's are outside the kernel's range)
        for kk in (max(cols) + 1, 64 * ((max(cols) + 64) // 64)):   # fewer columns: padding behind them
            _check(s[:kk])


@pytest.mark.parametrize("c_neg,c_pos", [(3, 10), (10, 3), (3, 74), (74, 3)])
def test_signed_zeros(c_neg, c_pos):
    """The key ranks -0 just below +0 (a zero-magnitude score keeps its sign bit), so +0 and -0 would not tie.  The
    kernel relies on its accumulator never holding -0: the last MMA of every column adds +0 products from the bias
    K-block, and the GPU test test_max_sim_tensor_core_signed_zero_ties checks that an exact-zero score built from -0
    products comes out as +0.  Ties among zeros of one sign go to the lowest column."""
    s = np.full(128, -1.0, F32)
    s[c_neg], s[c_pos] = F32(-0.0), F32(0.0)
    assert packed_argmax(s)[0] == c_pos
    s[c_neg] = F32(0.0)
    assert packed_argmax(s)[0] == min(c_neg, c_pos)
    s[c_neg], s[c_pos] = F32(-0.0), F32(-0.0)
    assert packed_argmax(s)[0] == min(c_neg, c_pos)


@pytest.mark.parametrize("k", [8, 60, 64, 100, 255])
def test_padding_and_initial_value_never_win(k):
    """Padded columns (score -1e30) lose to any real score above it, however negative; the -3.0e38 start value loses
    to every key, so a row of equal scores far below zero still decodes to column 0."""
    for v in (-1e29, -9.9e29, -1.0, 0.0):
        s = np.full(k, v, F32)
        assert packed_argmax(s)[0] == 0
        s[k - 1] = F32(v) / F32(2) if v else F32(1)        # a unique, larger last column
        assert packed_argmax(s)[0] == k - 1
    s = np.full(k, -2.9e38, F32)                           # real scores below the padding's, no padding column wins
    if k % 64 == 0:
        assert packed_argmax(s)[0] == 0


def test_key_is_close_to_the_score_and_ordered():
    """|key - score| < 2^-15 |score| (the TF32-derived-value bound rests on it), and for |score| < 2^13 two scores
    at least 2^-3 apart keep their order after the 8 low bits are replaced."""
    rng = np.random.default_rng(7)
    s = (rng.standard_normal(20000) * np.exp(rng.uniform(-20, 20, 20000))).astype(F32)
    for r in (0, 1, 128, 255):
        key = argmax_key(s, r).astype(np.float64)
        assert (np.abs(key - s.astype(np.float64)) < 2.0 ** -15 * np.abs(s.astype(np.float64))).all()
    a = (rng.integers(-2 ** 16, 2 ** 16, 20000) * 0.125).astype(F32)
    b = (a + F32(0.125)).astype(F32)
    for ra, rb in ((0, 255), (255, 0), (17, 200)):
        assert (argmax_key(b, rb) > argmax_key(a, ra)).all()


def test_decode_inverts_every_column():
    for v in (7.25, -7.25, 0.0, -0.0, 1e-42, -1e-42, -1e30):
        for j in range(256):
            assert argmax_key_column(argmax_key(F32(v), 255 ^ j)) == j


def test_old_rule_breaks_ties_by_sign_and_chunk_offset():
    """The packing this specification replaced: highest column among tied negative scores, and across chunks the
    column with the lower offset inside its chunk; the specification above returns the lowest column."""
    def with_tie(v, cols, k=128):
        s = np.full(k, -1e4, F32)
        s[list(cols)] = F32(v)
        return s
    assert packed_argmax_old(with_tie(5.5, (3, 10))) == 3
    assert packed_argmax_old(with_tie(-5.5, (3, 10))) == 10
    assert packed_argmax_old(with_tie(-0.0, (3, 10))) == 10
    assert packed_argmax_old(with_tie(5.5, (10, 67))) == 67
    assert packed_argmax_old(with_tie(-5.5, (3, 74))) == 74
    for v, cols in ((5.5, (3, 10)), (-5.5, (3, 10)), (-0.0, (3, 10)), (5.5, (10, 67)), (-5.5, (3, 74))):
        assert packed_argmax(with_tie(v, cols))[0] == min(cols)
