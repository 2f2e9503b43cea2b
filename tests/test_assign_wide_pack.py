"""CPU model of the arg-max in assign_wide_kernel (csrc/assign_wide.cu), checked against a plain lowest-index arg-max.

Per 128-column N tile, a thread of the quad tq holds the columns 8 i + 2 tq + {0, 1}, i < 16, packs each score with
its in-tile column (argmax_key, tc_common.cuh) and keeps the fmaxf of the keys.  Across N tiles it keeps (key, tile),
replaced only when the new key's truncated score (index field cleared) is STRICTLY greater.  Finally the quad merges by
(truncated score desc, global column asc).  Result: the lowest index among the columns whose truncated score is the
maximum, for every sign of the score -- and the plain lowest-index arg-max whenever distinct scores differ by more
than the 8 truncated mantissa bits (always for integer-valued scores |s| < 2^13, at half-integer resolution).
"""
import numpy as np
import pytest

N_TILE = 128


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _float(u):
    return np.asarray(u, np.uint32).view(np.float32)


def argmax_key(score, col):
    """PRMT (bytes 3..1 of the score, byte 0 = sign replicated) then XOR with 255 ^ col."""
    u = _bits(score)
    sign_byte = np.where(u >> 31, np.uint32(0xFF), np.uint32(0))
    return _float(((u & np.uint32(0xFFFFFF00)) | sign_byte) ^ (np.uint32(255) ^ np.uint32(col)))


def key_column(key):
    u = _bits(key)
    return 255 - int((u ^ (np.uint32(0xFFFFFFFF) if u >> 31 else np.uint32(0))) & np.uint32(0xFF))


def key_score(key):
    return _float(_bits(key) & np.uint32(0xFFFFFF00))


def wide_argmax(scores):
    """The kernel's arg-max of one row of scores [k] (fp32), padded columns at -1e30 as in the pre-pass."""
    k = len(scores)
    kpad = (k + N_TILE - 1) // N_TILE * N_TILE
    s = np.full(kpad, -1e30, np.float32)
    s[:k] = scores
    per_thread = []
    for tq in range(4):
        best, bs, bt = np.float32(-3e38), np.float32(-3e38), 0
        for nt in range(kpad // N_TILE):
            cb = np.float32(-3e38)
            for i in range(16):
                for b in range(2):
                    jt = 8 * i + 2 * tq + b
                    cb = np.fmax(cb, argmax_key(s[nt * N_TILE + jt], jt))
            ts = key_score(cb)
            if ts > bs:                                        # strictly greater: the earlier tile keeps ties
                best, bs, bt = cb, ts, nt
        per_thread.append((bs, bt * N_TILE + key_column(best)))
    for o in (1, 2):                                           # shuffle-xor butterfly over the quad
        merged = []
        for tq in range(4):
            (s0, g0), (s1, g1) = per_thread[tq], per_thread[tq ^ o]
            merged.append((s1, g1) if (s1 > s0 or (s1 == s0 and g1 < g0)) else (s0, g0))
        per_thread = merged
    assert len({(float(s), int(g)) for s, g in per_thread}) == 1   # every thread of the quad agrees
    return per_thread[0][1]


def lowest_index_argmax_truncated(scores):
    t = key_score(np.asarray(scores, np.float32))
    return int(np.flatnonzero(t == t.max())[0])


@pytest.mark.parametrize("sign", [1.0, 0.0, -1.0])
@pytest.mark.parametrize("k", [8, 130, 257, 600])
def test_ties_across_tile_boundaries(sign, k):
    """Equal best scores at j, j + 128, j + 256, ... and inside one tile -> the lowest of them, for every sign."""
    rng = np.random.default_rng(k)
    for trial in range(20):
        s = (sign * 50 - rng.integers(1, 40, k)).astype(np.float32) if sign <= 0 else rng.integers(-40, 40, k).astype(np.float32)
        best = np.float32(sign * 100.0)
        js = sorted(set(int(j) for j in rng.integers(0, k, 4)) | {int(rng.integers(0, k)) % N_TILE})
        for j in js:
            s[j] = best
        s[s > best] = best - 1                                 # `best` is the maximum
        assert wide_argmax(s) == min(js) == int(np.argmax(s))


def test_zero_ties_across_tiles():
    s = np.full(3 * N_TILE + 5, -7.0, np.float32)
    s[[N_TILE + 3, 3, 2 * N_TILE]] = 0.0
    assert wide_argmax(s) == 3


@pytest.mark.parametrize("seed", range(6))
def test_random_integer_scores_match_plain_argmax(seed):
    """Half-integer scores |s| < 2^13 (what integer data gives): the truncation loses nothing."""
    rng = np.random.default_rng(seed)
    k = int(rng.integers(8, 1200))
    s = (rng.integers(-2 ** 14 + 1, 2 ** 14, k) / 2.0).astype(np.float32)
    s[rng.integers(0, k, 5)] = s.max()                         # plus ties at the top
    assert wide_argmax(s) == int(np.argmax(s))


@pytest.mark.parametrize("seed", range(6))
def test_random_real_scores_lowest_index_of_truncated_max(seed):
    rng = np.random.default_rng(100 + seed)
    k = int(rng.integers(8, 1000))
    s = (rng.standard_normal(k) * 10 ** rng.uniform(-3, 3)).astype(np.float32)
    got = wide_argmax(s)
    assert got == lowest_index_argmax_truncated(s)
    assert key_score(s[got]) == key_score(s.max())            # within the 8 truncated bits of the true maximum
