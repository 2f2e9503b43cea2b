"""Designed-score index states: every live slot's score is an integer the test chooses, exact in fp32 whatever order
the scan sums it in, so a test can lay out any pattern of scores along the scan's visit order and know the exact
answer (score descending, address ascending) without floating-point slack.

Euclidean (d/M >= 4): queries are 0, so the LUT entry of sub-quantizer m and code j is ((0 * 2) - 0) - |c_mj|^2 =
-|c_mj|^2, |c|^2 a sum of separately rounded squares (lut.cuh).  The three "digit" sub-quantizers m = 0, 1, 2 give code
j four integer coordinates (a, b, c, d) * s_m with a^2 + b^2 + c^2 + d^2 = j (Lagrange; every j < 256 has them below
16) and s = 1, 16, 256, so |c_mj|^2 = j * 256^m exactly.  A slot with digit codes (c0, c1, c2) scores
-(c0 + 256 c1 + 65536 c2): any score in [-(2^24 - 1), -1].  Every other sub-quantizer has code 0 and a zero entry, and
every partial sum is an integer below 2^24, so any association of the sum is exact.

Cosine: the query is +-1/2 on the first coordinate of sub-quantizers 0..3 (the normalised form of four +-1 entries),
so the LUT entry is the codebook's first coordinate / 2 (sign +).  Digit m's entry j has first coordinate
2 (j - 128) 256^m, so a slot scores (c0 - 128) + 256 (c1 - 128) + 65536 (c2 - 128): signed scores in
[-8421504, 8421503].  Sub-quantizer 3 carries the query's fourth entry (-1/2) against a zero codebook.

The visit order of a query-major scan: the probe entries in order (an entry whose cell starts where the previous
entry's does is skipped), each cell's slots [cell_start, cell_start + cell_size) ascending in blocks of 32.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ivfpq_oracle as O

F32 = np.float32
EUC_MAX = 2 ** 24 - 1                        # euclidean scores lie in [-EUC_MAX, -1]
COS_OFF = 128 * (1 + 256 + 65536)            # cosine scores lie in [-COS_OFF, 2^24 - 1 - COS_OFF]


def _four_squares():
    out = {}
    for a in range(16):
        for b in range(a, 16):
            for c in range(b, 16):
                for d in range(c, 16):
                    n = a * a + b * b + c * c + d * d
                    if n < 256 and n not in out:
                        out[n] = (d, c, b, a)
    assert len(out) == 256
    return np.array([out[j] for j in range(256)], np.float32)       # [256, 4]


FOUR = _four_squares()


def score_range(distance):
    return (-EUC_MAX, -1) if distance == "euclidean" else (-COS_OFF, 2 ** 24 - 1 - COS_OFF)


class Designed:
    """An IndexState whose live slots carry chosen integer scores.

    sizes: live-slot count of each cell (cells are filled from their first slot); dsub >= 4; initial_size: slots per
    cell (default: the largest size).  Every live slot starts at the lowest score; set_scores writes others."""

    def __init__(self, sizes, M=8, dsub=4, distance="euclidean", initial_size=None):
        assert dsub >= 4 and M >= 4 and M % 4 == 0
        sizes = np.asarray(sizes, np.int64)
        C, d = len(sizes), M * dsub
        pq = np.zeros((M, dsub, 256), F32)
        j = np.arange(256)
        for m in range(3):
            if distance == "euclidean":
                pq[m, :4, :] = FOUR.T * F32(16 ** m)
            else:
                pq[m, 0, :] = 2 * (j - 128) * 256 ** m
        st = O.empty_state(d, M, C, int(initial_size or max(1, sizes.max())), distance,
                           np.zeros((d, C), F32), pq)
        n = int(sizes.sum())
        O.container_add(st, np.zeros((M, n), np.uint8), np.repeat(np.arange(C), sizes))
        st.use_smart_probing = False
        self.st, self.distance, self.M, self.dsub = st, distance, M, dsub
        self.score = np.full(st.capacity, score_range(distance)[0], np.int64)
        self.set_scores(np.flatnonzero(st.is_empty == 0), self.score[st.is_empty == 0])

    def set_scores(self, addr, scores):
        addr, scores = np.asarray(addr, np.int64), np.asarray(scores, np.int64)
        lo, hi = score_range(self.distance)
        assert scores.shape == addr.shape and (scores >= lo).all() and (scores <= hi).all()
        self.score[addr] = scores
        u = -scores if self.distance == "euclidean" else scores + COS_OFF
        for m in range(3):
            self.st.storage[0, addr, m] = (u >> (8 * m)) & 255

    def queries(self, nq):
        """[d, nq] queries as the scan uses them (search_cells takes them as given)"""
        x = torch.zeros(self.st.d_vector, nq)
        if self.distance == "cosine":
            x[[0, self.dsub, 2 * self.dsub], :] = 0.5
            x[3 * self.dsub, :] = -0.5
        return x

    def cell_slots(self, c):
        s = int(self.st.cell_start[c])
        return np.arange(s, s + int(self.st.cell_size[c]), dtype=np.int64)

    def visit(self, row, n=None):
        """addresses of every slot (live or not) the query-major scan visits for probe list `row`, in visit order"""
        row = np.asarray(row, np.int64)
        n = len(row) if n is None else n
        return O.probed_addresses(self.st.cell_start[row], self.st.cell_size[row], n)

    def live(self, addr):
        return addr[self.st.is_empty[addr] == 0]

    def expected(self, cells, npl, k):
        """(values [nq, k] f32, address [nq, k], ids [nq, k]) from the designed table: the probed live slots of every
        query, ordered (score desc, address asc), padded with (-inf, -1).  Identical rows are computed once."""
        cells, npl = np.asarray(cells, np.int64), np.asarray(npl, np.int64)
        nq, n_probe = cells.shape
        P = O.effective_probes(npl, n_probe)
        vals, adr = np.empty((nq, k), F32), np.empty((nq, k), np.int64)
        memo = {}
        for q in range(nq):
            key = tuple(cells[q, :P[q]])
            if key not in memo:
                a = self.live(self.visit(cells[q], int(P[q])))
                memo[key] = O.select_topk(self.score[a].astype(F32), a, k)
            vals[q], adr[q] = memo[key]
        return vals, adr, O.get_id_by_address(self.st.address2id, adr)


def visit_blocks(D, row):
    """(address, block, first) of every slot the query-major scan visits for `row`, in visit order: block = its index in
    the concatenated probe list (what the kernel's bootstrap and block cursor count); first = its first visit (a cell
    listed twice apart is scanned twice)"""
    addr, blk, b0, prev = [], [], 0, None
    for c in np.asarray(row, np.int64):
        s, n = int(D.st.cell_start[c]), int(D.st.cell_size[c])
        if s == prev:
            continue
        prev = s
        addr.append(np.arange(s, s + n, dtype=np.int64))
        blk.append(b0 + np.arange(n) // 32)
        b0 += (n + 31) // 32
    addr, blk = np.concatenate(addr), np.concatenate(blk)
    first = np.zeros(addr.shape[0], bool)
    first[np.unique(addr, return_index=True)[1]] = True
    return addr, blk, first


PATTERNS = ("ascending", "descending", "equal", "needle", "random", "plateau", "bound")


def design(D, row, pattern, rng, k=None, nw=None, leaders=None):
    """Give the live slots that probe list `row` visits the scores of `pattern`, stated along the visit order:
      ascending / descending  strictly rising / falling;
      equal                   one score for all;
      needle                  the best slot is the last live slot of the last probe entry, the rest random below it;
      random                  a random permutation of distinct ranks;
      plateau                 `leaders` distinct leaders, then every third slot tied at one score, the rest below it;
      bound                   the k best in the quick start's blocks (warp w of nw holds blocks w and w + nw), answer
                              rank r (1-based) in warp (r - 1) % nw: the minimum over warps of the ceil(k / nw)-th best
                              is a non-answer (k % nw != 0) or the k-th answer itself (k % nw == 0), while with
                              floor(k / nw) it would lie above answers k - (k % nw) + 1 .. k.
    Scores of slots visited twice are set once, by their first visit."""
    addr, blk, first = visit_blocks(D, row)
    keep = first & (D.st.is_empty[addr] == 0)
    a, b = addr[keep], blk[keep]
    n = a.shape[0]
    top = score_range(D.distance)[1]
    if pattern == "ascending":
        s = top - (n - 1) + np.arange(n)
    elif pattern == "descending":
        s = top - np.arange(n)
    elif pattern == "equal":
        s = np.full(n, top - 7)
    elif pattern == "needle":
        s = top - 1 - rng.permutation(n)
        s[-1] = top
    elif pattern == "random":
        s = top - 3 * rng.permutation(n)
    elif pattern == "plateau":
        s = top - leaders - 10 - rng.permutation(n)
        tied = np.flatnonzero(np.arange(n) % 3 == 1)
        lead = rng.choice(np.setdiff1d(np.arange(n), tied), leaders, replace=False)
        s[tied] = top - leaders
        s[lead] = top - rng.permutation(leaders)
    elif pattern == "bound":
        s = top - k - 10 - rng.permutation(n)
        pos = {}
        for i, bi in enumerate(b):
            pos.setdefault(int(bi), []).append(i)
        for r in range(1, k + 1):
            w, idx = (r - 1) % nw, (r - 1) // nw
            slots = pos[w + nw * (idx // 32)]
            assert len(slots) == 32, "the quick start's blocks must be fully live"
            s[slots[idx % 32]] = top - r
    else:
        raise ValueError(pattern)
    D.set_scores(a, s)
