"""GPU: the scans' top-k selection on designed, rank-adversarial scores (tests/designed_state.py).

Random codes settle the running k-th best within a few blocks, after which almost nothing beats the threshold, so the
rare paths of the selection protocol (common.cuh: CtaTopK's try-lock and forced flushes, merge_capped, the quick
start's bound and the drain that keeps keys equal to it; scan.cu: the cell-major survivor reservation at exactly its
capacity, multi-item cells, the 16 384-query chunk; merge_topk_kernel over empty slices and shards) are reached seldom
or never.  Here every slot's score is an exact integer laid out along the scan's visit order -- ascending, descending,
all equal, a needle in the last partly live block, plateaus of ties at the k-th value, the k best placed so that the
quick start's bound is the k-th answer -- and every row of every result must equal the designed answer bit for bit
(score descending, address ascending: there are no ties the order leaves open)."""
import numpy as np
import pytest
import torch

from designed_state import Designed, design, score_range, visit_blocks
from helpers import make_index
from test_scan_plan_gpu import launched

pytestmark = pytest.mark.gpu

KS = (1, 31, 32, 33, 64, 65, 100, 128, 512, 513, 1000, 1024)
NQ = 600                                   # > 4 x 132 SMs: unsliced


def assert_exact(D, out, cells, npl, k):
    v, i, a = (t.cpu().numpy() for t in out[:3])
    ev, ea, ei = D.expected(cells, npl, k)
    bad = np.flatnonzero((v.view(np.uint32) != ev.view(np.uint32)).any(1) | (a != ea).any(1) | (i != ei).any(1))
    assert bad.size == 0, f"k={k}: {bad.size} rows differ, first {bad[0]}: row {cells[bad[0]].tolist()}"


def query_major_state(M, dsub, distance="euclidean", initial_size=None, nw=8):
    """One index, one group of cells per pattern; group g is scanned by probe list rows[g].  The bound patterns are
    laid out for k = 64 (a multiple of NW) and k = 100 (not one) at the kernel's NW."""
    groups = [
        ("ascending", [1000, 777, 1200, 500], {}),
        ("descending", [1000, 777, 1200, 500], {}),
        ("equal", [1000, 777, 1200, 500], {}),
        ("needle", [1000, 600, 900, 333], {}),
        ("random", [1000, 777, 1200, 500], {}),
        ("plateau", [1000, 1000, 800, 700], {"leaders": 32}),
        ("plateau", [1000, 1000, 800, 700], {"leaders": 99}),
        ("bound", [1100, 900, 800], {"k": 64, "nw": nw}),
        ("bound", [1100, 900, 800], {"k": 100, "nw": nw}),
        ("few", [300, 200], {}),
    ]
    sizes = [s for _, g, _ in groups for s in g]
    D = Designed(sizes, M=M, dsub=dsub, distance=distance, initial_size=initial_size)
    rng = np.random.default_rng(M * 100 + dsub)
    rows, c0 = [], 0
    for name, g, kw in groups:
        cells = list(range(c0, c0 + len(g)))
        c0 += len(g)
        if name == "equal":
            D.st.is_empty[D.cell_slots(cells[2])[::7]] = 1                  # holes: partly live blocks
        if name == "needle":
            D.st.is_empty[D.cell_slots(cells[3])[-9:-1]] = 1                # the last block is partly live
        if name == "few":
            D.st.is_empty[D.cell_slots(cells[0])[::3]] = 1                  # 333 live slots: fewer than most k
        row = [cells[0], cells[1], cells[0], cells[2], cells[3]] if name == "random" else cells
        design(D, row, "random" if name == "few" else name, rng, **kw)
        rows.append(row)
    return D, rows


def batch(rows, nq):
    n_probe = max(len(r) for r in rows)
    cells = np.array([(rows[q % len(rows)] + [0] * n_probe)[:n_probe] for q in range(nq)], np.int64)
    npl = np.array([len(rows[q % len(rows)]) for q in range(nq)], np.int64)
    return cells, npl


# The kernels each index reaches (plan_scan, scan.cu): m_pad 32 takes 8 warps x 2 CTAs/SM; m_pad 64 takes 2 CTAs/SM from
# 2000 capacity blocks per CTA (initial_size 13000), else 3; d/M = 12 has no in-CTA LUT build, so lut_kernel stages it;
# m_pad 96 and 128 take 16 warps.
QM = {
    "m16": dict(M=16, dsub=4, want={"ivfpq_scan_kernel<32, 8, 2, 4, false>"}),
    "m64_3": dict(M=64, dsub=4, want={"ivfpq_scan_kernel<64, 8, 3, 4, false>"}),
    "m64_2": dict(M=64, dsub=4, initial_size=13000, want={"ivfpq_scan_kernel<64, 8, 2, 4, false>"}),
    "m64_staged": dict(M=64, dsub=12, want={"lut_kernel<0, 1>", "ivfpq_scan_kernel<64, 8, 3, 0, false>"}),
    "m96": dict(M=96, dsub=4, nw=16, want={"ivfpq_scan_kernel<96, 16, 1, 4, false>"}),
    "m128": dict(M=128, dsub=4, nw=16, want={"ivfpq_scan_kernel<128, 16, 1, 4, false>"}),
    "cosine_m8": dict(M=8, dsub=4, distance="cosine", want={"ivfpq_scan_kernel<32, 8, 2, 4, false>"}),
}


@pytest.mark.parametrize("cfg", list(QM))
def test_query_major(cuda_device, cfg):
    """Every pattern in one batch, every k: 1 and 31-33 (a 32-key list), 64/65, 100/128, 512/513 (both sides of the
    quick start's limit k <= 32 * 2 * NW at 8 warps), 1000/1024; the last group has fewer live slots than most k."""
    c = dict(QM[cfg])
    want = c.pop("want")
    D, rows = query_major_state(**c)
    ix = make_index(D.st)
    cells, npl = batch(rows, NQ)
    x, cg, ng = D.queries(NQ).cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()
    assert launched(lambda: ix.search_cells(x, cg, n_probe_list=ng, k=100)) == want | {"merge_topk_kernel"}
    for k in KS:
        assert_exact(D, ix.search_cells(x, cg, n_probe_list=ng, k=k, return_address=True), cells, npl, k)


def test_sliced_batches(cuda_device):
    """nq = 1 and 3: S = min(64, ceil(4 SMs / nq)) slices per query, merged by merge_topk_kernel.  One probe set has
    fewer blocks than slices (most slices return nothing), one holds its whole answer in a single slice."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    D = Designed([300, 2600, 2600, 2600, 1000, 1000], M=64, dsub=4)
    rng = np.random.default_rng(7)
    design(D, [0], "ascending", rng)
    one = [1, 2, 3]
    addr, blk, _ = visit_blocks(D, one)
    assert 4 * sm >= 64 * 3
    S = 64                                 # slices per query at nq = 1 and 3
    T = int(blk.max()) + 1
    j = S // 2 + 1
    lo, hi = T * j // S, T * (j + 1) // S
    inside = (blk >= lo) & (blk < hi)
    top = score_range("euclidean")[1]
    s = top - 5000 - rng.permutation(addr.shape[0])
    s[inside] = top - rng.permutation(int(inside.sum()))
    D.set_scores(addr, s)
    design(D, [4, 5], "plateau", rng, leaders=20)
    ix = make_index(D.st)
    rows = [[0], one, [4, 5], one[::-1]]
    for nq in (1, 3):
        for r0 in range(len(rows)):
            rr = rows[r0:] + rows[:r0]
            cells, npl = batch(rr, nq)
            x = D.queries(nq).cuda()
            for k in KS:
                out = ix.search_cells(x, torch.from_numpy(cells).cuda(), n_probe_list=torch.from_numpy(npl).cuda(),
                                      k=k, return_address=True)
                assert_exact(D, out, cells, npl, k)


def test_shards_with_the_answer_in_one(cuda_device):
    """Cell shards (cell c on shard c % world) merged by tpq_merge_topk: the whole answer lies in shard 1's cells, the
    other shards return only worse keys or none; bit-equal to the unsharded search and to the designed answer."""
    import torchpq_b200 as T
    D = Designed([800, 1100, 700, 500, 900, 650, 300, 1000, 420], M=16, dsub=4)
    rng = np.random.default_rng(11)
    top = score_range("euclidean")[1]
    mine = np.concatenate([D.cell_slots(c) for c in (1, 4, 7)])
    rest = np.concatenate([D.cell_slots(c) for c in (0, 2, 3, 5, 6, 8)])
    D.set_scores(mine, top - rng.permutation(mine.shape[0]))
    D.set_scores(rest, top - 10000 - rng.permutation(rest.shape[0]))
    ix = make_index(D.st)
    for nq in (3, NQ):
        rows = [list(range(9)), [1, 0, 4, 2, 7], [3, 5, 7], [8, 6, 4, 2, 0]]
        cells, npl = batch(rows, nq)
        x, cg, ng = D.queries(nq).cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()
        for k in (1, 33, 100, 1024):
            whole = ix.search_cells(x, cg, n_probe_list=ng, k=k, return_address=True)
            assert_exact(D, whole, cells, npl, k)
            parts = []
            for r in range(3):
                ix.set_shard(r, 3)
                parts.append(ix.search_cells(x, cg, n_probe_list=ng, k=k, return_keys=True)[2])
            ix.set_shard(0, 1)
            v, i, a = T.fn.merge_topk(torch.stack(parts).contiguous(), ix._address2id)
            assert torch.equal(v, whole[0]) and torch.equal(i, whole[1]) and torch.equal(a, whole[2])


def test_reference_layout_op(cuda_device):
    """fn.IVFPQTopk.topk (scan_ref.cu: warps take 32-slot chunks in a static stripe, no bootstrap, the threshold starts
    at 0, a final forced flush per warp) fed a designed LUT [M, nq, 256] of signed integers: entry (m, j) =
    (j - 128) 256^m on the three digit sub-quantizers, 0 elsewhere, so the scores are the designed cosine ones."""
    import torchpq_b200 as T
    D, rows = query_major_state(8, 4, distance="cosine")
    cells, npl = batch(rows, 200)
    M = D.M
    lut = np.zeros((M, 200, 256), np.float32)
    for m in range(3):
        lut[m] = (np.arange(256) - 128) * 256.0 ** m
    st = D.st
    args = [torch.from_numpy(a).cuda() for a in (st.storage, lut, st.cell_start[cells], st.cell_size[cells], st.is_empty,
                                                 npl)]
    op = T.fn.IVFPQTopk(M)
    for k in KS:
        v, a = op.topk(args[0], args[1], args[2], args[3], args[4], args[5], k=k)
        ev, ea, _ = D.expected(cells, npl, k)
        assert np.array_equal(v.cpu().numpy().view(np.uint32), ev.view(np.uint32)), k
        assert np.array_equal(a.cpu().numpy(), ea), k


# ----------------------------------------------------------------------------------------------- cell-major
S0_GAP = 100000


def cell_major_state():
    """Cell 0 (E0): every score s0.  A, B hold exactly 4096 slots above s0, C 4097, Z none; BIG is 336 full blocks
    (4 work items of 84 blocks), lanes 0-19 above s0.  Above s0, a lower lane scores higher and, within a lane, a later
    block higher, so the k best of a cell lie in every one of its blocks.  With E0 first, its k lowest addresses are
    the pass-1 list and the bound, and the survivors of a query are exactly its slots above s0."""
    sizes = {"E0": 1100, "A": 5000, "B": 5000, "C": 5000, "Z": 2000, "BIG": 336 * 32}
    names = list(sizes)
    D = Designed([sizes[n] for n in names], M=64, dsub=4)
    rng = np.random.default_rng(3)
    top = score_range("euclidean")[1]
    s0 = top - S0_GAP
    cell = {n: i for i, n in enumerate(names)}
    D.set_scores(D.cell_slots(cell["E0"]), np.full(sizes["E0"], s0))
    for n, above in (("A", 4096), ("B", 4096), ("C", 4097), ("Z", 0), ("BIG", 20 * 336)):
        a = D.cell_slots(cell[n])
        rel = np.arange(a.shape[0])
        order = np.lexsort((-(rel // 32), rel % 32))                       # lane ascending, block descending
        s = s0 - 1 - rng.permutation(a.shape[0])
        s[order[:above]] = s0 + above - np.arange(above)
        D.set_scores(a, s)
    return D, cell


def cell_major_rows(cell):
    E0, A, B, C, Z, BIG = (cell[n] for n in ("E0", "A", "B", "C", "Z", "BIG"))
    return [[E0, A, B],          # 8192 survivors: exactly the capacity
            [E0, A, C],          # 8193: overflow, re-run query-major
            [E0, A, Z, A],       # 8192 through A listed twice, apart
            [E0, BIG],           # 6720 survivors over BIG's 4 work items
            [E0, C, Z],
            [A, B],
            [C, BIG, Z]]


def cell_major(D):
    from test_cell_scan_gpu import cell_major_index
    return cell_major_index(D.st)


@pytest.mark.parametrize("k", [100, 1024])
def test_cell_major_survivor_capacity(cuda_device, k):
    D, cell = cell_major_state()
    ix = cell_major(D)
    cells, npl = batch(cell_major_rows(cell), NQ)
    x, cg, ng = D.queries(NQ).cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()
    assert "ivfpq_cell_scan_kernel<12, 7>" in launched(lambda: ix.search_cells(x, cg, n_probe_list=ng, k=k))
    assert_exact(D, ix.search_cells(x, cg, n_probe_list=ng, k=k, return_address=True), cells, npl, k)


@pytest.mark.parametrize("extra", [1, 600])
def test_cell_major_query_chunks(cuda_device, extra):
    """16 384 + extra queries: two launches of the cell-major stage, the last holding `extra` queries.  Rows cycle
    through 7 probe lists (16 384 % 7 != 0), so a buffer indexed by the global query where the chunk-local one is
    meant (or the reverse) reads another row's answer."""
    D, cell = cell_major_state()
    ix = cell_major(D)
    nq, k = 16384 + extra, 100
    cells, npl = batch(cell_major_rows(cell), nq)
    x, cg, ng = D.queries(nq).cuda(), torch.from_numpy(cells).cuda(), torch.from_numpy(npl).cuda()
    big = ix.search_cells(x, cg, n_probe_list=ng, k=k, return_address=True, return_keys=True)
    assert_exact(D, big, cells, npl, k)
    for s in range(16384 - 200, nq, 100):
        e = min(nq, s + 100)
        small = ix.search_cells(x[:, s:e].contiguous(), cg[s:e].contiguous(), n_probe_list=ng[s:e].contiguous(), k=k,
                                return_keys=True)
        assert torch.equal(big[3][s:e], small[2])
