"""CPU: an executable specification of the register bitonic networks and the top-k selection protocol of
torchpq_b200/csrc/common.cuh (reg_sort / reg_merge / warp_bitonic_merge_desc / warp_merge_run / warp_merge_runs, and
CtaTopK / WarpTopK).  The functions below are line-by-line transliterations of the index arithmetic of those
routines (element r*32 + lane of a warp's run, shuffle distance j, direction bit k, run regions 64 keys apart, the
gap-closing copy for 32-key runs) with "all lanes at once" semantics for a shuffle stage; they are checked against
`sorted`.  The product library bootstraps the scan's threshold with CtaTopK::cta_quickstart, specified below together
with push / flush / merge_staged / merge_capped / merge_locked / cta_drain under a seeded scheduler of warps and lock
contention.
CtaTopK::cta_bootstrap, the merge tree, is compiled only into the -DTPQ_DEBUG_KNOBS build, where it is the default; it
is specified here too.  The GPU tests check the kernels' results; this file pins the protocol where no GPU is
needed."""
import random

import pytest


def _cswap(x, a, b, lane, desc):
    hi, lo = max(x[a][lane], x[b][lane]), min(x[a][lane], x[b][lane])
    x[a][lane], x[b][lane] = (hi, lo) if desc else (lo, hi)


def _shuffle_stage(x, R, j, k, asc, merge):
    new = [[0] * 32 for _ in range(R)]
    for lane in range(32):
        up = (lane & j) != 0
        for r in range(R):
            y = x[r][lane ^ j]                                   # __shfl_xor_sync(x[r], j)
            if merge:
                new[r][lane] = min(x[r][lane], y) if (up != asc) else max(x[r][lane], y)
            else:
                desc = ((((r * 32) | lane) & k) == 0) != asc
                new[r][lane] = max(x[r][lane], y) if (desc != up) else min(x[r][lane], y)
    for r in range(R):
        x[r] = new[r]


def reg_merge(x, R, asc=False):
    for lane in range(32):
        if R == 4:
            _cswap(x, 0, 2, lane, not asc); _cswap(x, 1, 3, lane, not asc)
        if R >= 2:
            for r in range(0, R, 2):
                _cswap(x, r, r + 1, lane, not asc)
    j = 16
    while j > 0:
        _shuffle_stage(x, R, j, 0, asc, True)
        j >>= 1


def reg_sort(x, R, asc=False):
    k = 2
    while k <= 32 * R:
        j = k >> 1
        if R == 4 and k == 128:
            for lane in range(32):
                _cswap(x, 0, 2, lane, not asc); _cswap(x, 1, 3, lane, not asc)
            j = 32
        if R >= 2 and j == 32:
            for lane in range(32):
                for r in range(0, R, 2):
                    _cswap(x, r, r + 1, lane, (((r * 32) & k) == 0) != asc)
            j = 16
        while j > 0:
            _shuffle_stage(x, R, j, k, asc, False)
            j >>= 1
        k <<= 1


def _flat(x, R):
    return [x[r][l] for r in range(R) for l in range(32)]


def _regs(v, R):
    return [[v[r * 32 + l] for l in range(32)] for r in range(R)]


def bitonic_merge_desc(a, off, n):
    j = n >> 1
    while j >= 64:
        for t in range(n >> 1):
            lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)); hi = lo + j
            if a[off + lo] < a[off + hi]:
                a[off + lo], a[off + hi] = a[off + hi], a[off + lo]
        j >>= 1
    if n == 32:
        x = _regs(a[off:off + 32], 1); reg_merge(x, 1); a[off:off + 32] = _flat(x, 1)
    else:
        for c in range(0, n, 64):
            x = _regs(a[off + c:off + c + 64], 2); reg_merge(x, 2); a[off + c:off + c + 64] = _flat(x, 2)


def merge_run(A, n, x, R):
    tail = n - 32 * R
    if n == 32 * R:
        y = [[max(A[tail + r * 32 + l], x[r][l]) for l in range(32)] for r in range(R)]
        reg_merge(y, R)
        A[tail:] = _flat(y, R)
        return
    for r in range(R):
        for l in range(32):
            A[tail + r * 32 + l] = max(A[tail + r * 32 + l], x[r][l])
    bitonic_merge_desc(A, 0, n)


def merge_runs(buf, a, b, ln, top_only):
    for t in range(ln):
        x, y = buf[a + t], buf[b + ln - 1 - t]
        buf[a + t] = max(x, y)
        if not top_only:
            buf[b + ln - 1 - t] = min(x, y)
    bitonic_merge_desc(buf, a, ln)
    if not top_only:
        bitonic_merge_desc(buf, b, ln)


def cta_bootstrap(keys_per_warp, nw, R, kp):
    scratch = [0] * (nw * 64)
    ln = 32 if (R == 1 or kp < 64) else 64
    for w in range(nw):
        x = _regs(keys_per_warp[w] + [0] * (64 - 32 * R), 2) if R == 2 else _regs(keys_per_warp[w], 1)
        reg_sort(x, 2 if R == 2 else 1)
        scratch[w * 64:w * 64 + ln] = _flat(x, 2 if R == 2 else 1)[:ln]
    s = 1
    while s < nw:
        top_only = 2 * ln > kp
        for w in range(nw):
            if (w & (2 * s - 1)) == 0 and w + s < nw:
                a, b = w * 64, (w + s) * 64
                merge_runs(scratch, a, b, ln, top_only)
                if not top_only and b != a + ln:
                    scratch[a + ln:a + 2 * ln] = scratch[b:b + ln]
        if not top_only:
            ln <<= 1
        s <<= 1
    lst = [0] * kp
    for t in range(ln):                                        # warp_merge_desc(list, kp, scratch, len)
        i = kp - ln + t
        lst[i] = max(lst[i], scratch[ln - 1 - t])
    bitonic_merge_desc(lst, 0, kp)
    return lst


@pytest.mark.parametrize("R", [1, 2, 4])
@pytest.mark.parametrize("asc", [False, True])
def test_register_sort_and_merge(R, asc):
    rng = random.Random(R * 2 + asc)
    for _ in range(25):
        v = [rng.randrange(0, 60) for _ in range(32 * R)]         # many ties
        x = _regs(v, R)
        reg_sort(x, R, asc)
        assert _flat(x, R) == sorted(v, reverse=not asc)
        h = 16 * R
        x = _regs(sorted(v[:h], reverse=True) + sorted(v[h:]), R)  # a bitonic sequence
        reg_merge(x, R, asc)
        assert _flat(x, R) == sorted(v, reverse=not asc)


@pytest.mark.parametrize("kp", [32, 64, 128, 256, 1024])
@pytest.mark.parametrize("R", [1, 2, 4])
def test_merge_run_into_list(kp, R):
    if 32 * R > kp:
        pytest.skip("the run is capped to the list length before the merge (merge_capped)")
    rng = random.Random(kp + R)
    for _ in range(8):
        lst = sorted([rng.randrange(0, 1000) for _ in range(kp)], reverse=True)
        run = sorted(rng.randrange(0, 1000) for _ in range(32 * R))
        A = lst[:]
        merge_run(A, kp, _regs(run, R), R)
        assert A == sorted(lst + run, reverse=True)[:kp]


@pytest.mark.parametrize("nw", [4, 8, 16])
@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("kp", [32, 64, 128, 256, 1024])
def test_merge_tree_bootstrap(nw, R, kp):
    rng = random.Random(nw * 100 + R * 10 + kp)
    for _ in range(3):
        keys = [[rng.randrange(1, 10 ** 6) for _ in range(32 * R)] for _ in range(nw)]
        got = cta_bootstrap(keys, nw, R, kp)
        expect = sorted((k for w in keys for k in w), reverse=True)[:kp]
        assert got == expect + [0] * (kp - len(expect))


# ----------------------------------------------------------------------------------------------- the shipped protocol
# CtaTopK as the product build runs it in ivfpq_scan_kernel (scan.cu): cta_quickstart on the first R blocks of every
# warp, then push / flush (try-lock above 32 staged keys, forced above 64) / merge_staged / merge_capped / merge_locked (with its
# early return) while the warps take blocks from a shared cursor, then cta_drain; and WarpTopK as cell_select_kernel runs
# it.  A seeded scheduler picks which warp takes the next block, whether the lock is busy at each try, and whether a
# warp's copy of the threshold is stale; the networks are the transliterations above.
K_STAGE = 96                    # CtaTopK staging entries per warp (kStage)


def list_capacity(k):
    p = 1
    while p < max(k, 32):
        p <<= 1
    return p


def _run(keys, R, asc=True):
    """a warp's staged keys (missing ones 0) sorted in registers: load_sorted_run<R>, reg_sort<R, ASC>"""
    x = _regs(list(keys) + [0] * (32 * R - len(keys)), R)
    reg_sort(x, R, asc)
    return x


class CtaSim:
    def __init__(self, k, nw, rng, p_busy):
        self.k, self.nw, self.kp = k, nw, list_capacity(k)
        self.lst, self.thr = [0] * self.kp, 0
        self.buf = [[] for _ in range(nw)]
        self.rng, self.p_busy = rng, p_busy
        self.paths = set()

    def _merged(self):
        assert self.lst == sorted(self.lst, reverse=True), "the shared list is sorted after every merge"

    def merge_locked(self, x, R):
        top = x[R - 1][31]
        if top < self.thr:                                     # nothing staged can still be in the top k
            self.paths.add("early return")
            return
        if top > self.lst[self.k - 1]:
            merge_run(self.lst, self.kp, x, R)
            self._merged()
            self.thr = max(self.thr, self.lst[self.k - 1])

    def merge_capped(self, x, R):
        """merge_capped with merge = merge_locked: only the run's kp largest, its last registers, can matter"""
        if R > 1 and self.kp == 32:
            self.paths.add(f"capped R={R} kp=32")
            self.merge_locked([x[R - 1]], 1)
        elif R > 2 and self.kp == 64:
            self.paths.add(f"capped R={R} kp=64")
            self.merge_locked([x[R - 2], x[R - 1]], 2)
        else:
            self.merge_locked(x, R)

    def flush(self, w, force):
        b = self.buf[w]
        if not b:
            return
        if not force and self.rng.random() < self.p_busy:      # another warp holds the lock: keep scanning
            self.paths.add("lock busy")
            return
        if len(b) <= 32:                                       # merge_staged<4>
            self.merge_locked(_run(b, 1), 1)
        elif len(b) <= 64:
            self.merge_capped(_run(b, 2), 2)
        else:
            self.paths.add("forced 65-96")
            self.merge_capped(_run(b, 4), 4)
        b.clear()

    def push(self, w, keys):
        b = self.buf[w]
        b.extend(keys)
        assert len(b) <= K_STAGE, "a warp stages at most kStage keys"
        if len(b) > 32:
            self.flush(w, len(b) > K_STAGE - 32)

    def quickstart(self, staged, R):
        """staged[w]: the 32 R keys of warp w's bootstrap blocks (0 for missing vectors)"""
        runs = []
        for w in range(self.nw):
            x = _regs(list(staged[w]) + [0] * (64 - 32 * R), 2)
            reg_sort(x, 2)                                     # descending: ranks 0..63
            runs.append(_flat(x, 2))
        q = (self.k + self.nw - 1) // self.nw
        bound = min(r[q - 1] if q <= 32 * R else 0 for r in runs)
        if bound == 0:
            self.paths.add("no bound")
        self.thr = max(self.thr, bound)
        for w, r in enumerate(runs):
            kept = [i for i, v in enumerate(r) if v != 0 and v >= bound]
            assert kept == list(range(len(kept))), "the kept keys are a prefix of the sorted run"
            self.buf[w] = r[:len(kept)]

    def drain(self):
        t = self.thr
        left = [v for b in self.buf for v in b[:K_STAGE] if v != 0 and v >= t]
        if any(v == t for v in left):
            self.paths.add("drain keeps the bound")
        for c0 in range(0, len(left), 64):                     # merge_staged<2> with merge = warp_merge_run
            chunk = left[c0:c0 + 64]
            if len(chunk) <= 32:
                merge_run(self.lst, self.kp, _run(chunk, 1), 1)
            elif self.kp == 32:
                merge_run(self.lst, self.kp, [_run(chunk, 2)[1]], 1)
            else:
                merge_run(self.lst, self.kp, _run(chunk, 2), 2)
            self._merged()
        self.buf = [[] for _ in range(self.nw)]


def simulate_scan(blocks, k, nw, seed, R=2, p_busy=0.5, p_stale=0.3):
    """ivfpq_scan_kernel's selection over `blocks` (lists of 32 keys, 0 = not live) -> (the CTA's list, paths seen)"""
    rng = random.Random(seed)
    cta = CtaSim(k, nw, rng, p_busy)
    n = len(blocks)
    staged = [[key for r in range(R) for key in (blocks[w + r * nw] if w + r * nw < n else [0] * 32)]
              for w in range(nw)]
    cta.quickstart(staged, R)
    cursor, thr_seen, active = R * nw, [cta.thr] * nw, list(range(nw))
    while active:
        w = rng.choice(active)
        if cursor >= n:
            active.remove(w)
            continue
        b = blocks[cursor]
        cursor += 1
        if rng.random() >= p_stale:
            thr_seen[w] = cta.thr                              # the running k-th best, read at most once per block
        cta.push(w, [key for key in b if key != 0 and key > thr_seen[w]])
    cta.drain()
    return cta.lst, cta.paths


def warp_select(start, cand, k):
    """cell_select_kernel: WarpTopK seeded with a sorted list of k keys (the pass-1 list), pushed 32 candidates at a
    time against its own k-th best, flushed above 32 staged keys and at the end (flush: merge_staged<2> with merge =
    warp_merge_run)"""
    kp = list_capacity(k)
    lst = list(start) + [0] * (kp - len(start))
    buf = []

    def flush():
        if not buf:
            return
        if len(buf) <= 32:
            merge_run(lst, kp, _run(buf, 1), 1)
        else:
            x = _run(buf, 2)
            if kp == 32:
                merge_run(lst, kp, [x[1]], 1)
            else:
                merge_run(lst, kp, x, 2)
        assert lst == sorted(lst, reverse=True)
        buf.clear()

    for i0 in range(0, len(cand), 32):
        th = lst[k - 1]
        buf.extend(v for v in cand[i0:i0 + 32] if v > th)
        assert len(buf) <= 64
        if len(buf) > 32:
            flush()
    flush()
    return lst


def pattern_keys(pattern, n_blocks, k, nw, seed, R=2):
    """keys of n_blocks blocks in visit order for one of the designed score patterns (tests/designed_state.py);
    key = score << 20 | ~position: distinct, larger is better, 0 is empty"""
    rng = random.Random(seed)
    n = 32 * n_blocks
    if pattern == "ascending":
        s = list(range(1, n + 1))
    elif pattern == "descending":
        s = list(range(n, 0, -1))
    elif pattern == "equal":
        s = [7] * n
    elif pattern == "needle":
        s = rng.sample(range(1, n + 1), n)
        s[n - 5] = n + 1
    elif pattern == "random":
        s = rng.sample(range(1, n + 1), n)
    elif pattern == "plateau":
        lead = min(k - 1, n // 4)
        s = [1 + rng.randrange(n) for _ in range(n)]
        for i in range(n):
            if i % 3 == 1:
                s[i] = n + 1
        for i in rng.sample([i for i in range(n) if i % 3 != 1], lead):
            s[i] = n + 2 + rng.randrange(n)
    elif pattern == "bound":
        s = [1 + rng.randrange(n) for _ in range(n)]
        for r in range(1, min(k, 64 * nw) + 1):
            w, idx = (r - 1) % nw, (r - 1) // nw
            s[(w + nw * (idx // 32)) * 32 + idx % 32] = 2 * n - r
    else:
        raise ValueError(pattern)
    keys = [(v << 20) | ((1 << 20) - 1 - i) for i, v in enumerate(s)]
    if pattern in ("equal", "needle", "random"):                # holes: partly live blocks, the last one too
        for i in range(0, n, 7 if pattern == "equal" else 11):
            keys[i] = 0
        keys[n - 2] = 0
    return [keys[b * 32:(b + 1) * 32] for b in range(n_blocks)]


SCAN_CASES = [(nw, k) for nw in (4, 8) for k in (1, 31, 32, 33, 64, 65, 100, 128, 300)] + [(8, 513)]


@pytest.mark.parametrize("nw, k", SCAN_CASES)
@pytest.mark.parametrize("pattern", ["ascending", "descending", "equal", "needle", "random", "plateau", "bound"])
def test_shipped_scan_selection(pattern, nw, k):
    """The exact top k of every pattern under two seeded schedules; k = 300 at 4 warps and 513 at 8 exceed the quick
    start's limit 32 * 2 * NW, so it gives no bound there."""
    n_blocks = 2 * nw + 24
    blocks = pattern_keys(pattern, n_blocks, k, nw, seed=k)
    every = sorted((v for b in blocks for v in b if v), reverse=True)[:k]
    for seed in (1, 2):
        lst, _ = simulate_scan(blocks, k, nw, seed=seed * 1000 + k)
        assert lst[:k] == every + [0] * (k - len(every))


def test_shipped_scan_reaches_every_path():
    """The schedules above are not idle: over a handful of runs the simulation takes every branch the GPU reaches
    only by chance -- forced 65-96-key flushes, both capped merges, the early return, no bound, and a drain that keeps
    a key equal to the bound."""
    seen = set()
    for pattern, nw, k, n in (("ascending", 8, 32, 40), ("ascending", 8, 100, 40), ("ascending", 4, 1, 32),
                              ("bound", 8, 64, 40), ("random", 4, 300, 32), ("descending", 8, 256, 40),
                              ("ascending", 8, 33, 40), ("random", 8, 1, 400)):
        for seed in range(3):
            seen |= simulate_scan(pattern_keys(pattern, n, k, nw, seed), k, nw, seed=seed, p_busy=0.7, p_stale=0.9)[1]
    for p in ("forced 65-96", "capped R=4 kp=32", "capped R=4 kp=64", "capped R=2 kp=32", "early return", "lock busy",
              "no bound", "drain keeps the bound"):
        assert p in seen, p


@pytest.mark.parametrize("k", [1, 31, 32, 33, 64, 100, 128, 1024])
def test_warp_select(k):
    rng = random.Random(k)
    for pattern in ("ascending", "descending", "equal", "random"):
        pool = pattern_keys(pattern, 40, k, 8, seed=k)
        flat = [v for b in pool for v in b if v]
        start = sorted(flat[:k], reverse=True)
        cand = sorted(flat[k:], reverse=(pattern == "descending")) if pattern != "random" else flat[k:]
        if pattern == "equal":
            rng.shuffle(cand)
        got = warp_select(start, cand, k)
        every = sorted(flat, reverse=True)[:k]
        assert got[:k] == every + [0] * (k - len(every))
