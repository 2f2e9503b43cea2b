"""GPU: which kernels a search launches.  The scan's configuration (warps and CTAs per SM, in-CTA or staged LUT,
cell-major or query-major) changes speed, not results, so a wrong choice would pass every result test; this pins the
choice for each kind of index by the kernels a single search launches, as torch.profiler records them."""
import ctypes as C
import re
import time

import pytest
import torch

from oracle import build_state as B
from helpers import make_index

pytestmark = pytest.mark.gpu

NQ = 600          # > 4 x 132 SMs: an unsliced batch
SLICED = 100      # sliced into several CTAs per query
K = 10

CELL = {"cell_lut_kernel<2>", "ivfpq_scan_kernel<64, 8, 2, 0, false>", "ivfpq_cell_scan_kernel<12, 7>",
        "cell_pairs_count_kernel", "cell_plan_kernel", "cell_pairs_scatter_kernel", "cell_select_kernel",
        "merge_topk_kernel"}


def launched(fn, windows=3, max_windows=12):
    """names (namespace and parameter list stripped) of the scan, LUT, cell and merge kernels that fn() launches.
    The profiler keeps only the device events whose timestamps fall inside its window, and its device timestamps drift
    from its host clock as a process ages: late in a long pytest process it drops the first launches of a window, then
    every launch of it; and now and then a window loses its device events altogether.  So fn() runs between two marker
    kernels, with a pause on either side of them that doubles whenever a marker goes missing; a window counts when it
    recorded both markers (so nothing between them fell outside it), and the names seen in `windows` such windows are
    pooled (fn() launches the same kernels on every call, and a dropped event can only hide a name, never add one)."""
    fn()                                                                  # layout, module loads
    torch.cuda.synchronize()
    names, complete, pad = set(), 0, 0.05
    for _ in range(max_windows):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            time.sleep(pad)
            torch.cuda._sleep(1000)                                       # marker: spin_kernel
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            time.sleep(pad)
        markers = 0
        for e in prof.events():
            markers += e.device_type == torch.autograd.DeviceType.CUDA and "spin_kernel" in e.name
            n = re.sub(r"^void ", "", e.name).replace("tpq::", "").split("(")[0]
            if any(s in n for s in ("scan", "lut", "cell_", "merge")):
                names.add(n)
        if markers == 2:
            complete += 1
            if complete == windows:
                break
        else:
            pad = min(2 * pad, 3.2)
    return names


def make_residual_index(st):
    import torchpq_b200 as T
    ix = T.IVFPQIndex(st.d_vector, st.n_subvectors, st.n_cells, initial_size=1, device="cuda:0", pq_use_residual=True)
    return ix.load_state(st)


def index_of(d, M, n, n_probe, residual=False, distance="euclidean", initial_size=None, seed=0):
    st, queries = B.integer_state(d, M, 8, n, seed=seed, distance=distance, initial_size=initial_size)
    st.n_probe, st.use_smart_probing = n_probe, False
    ix = make_residual_index(st) if residual else make_index(st)
    return ix, queries


def searched(ix, queries, nq):
    x = queries(nq).cuda()
    return launched(lambda: ix.search(x, k=K))


def test_m64_long_lists(cuda_device):
    """at least 2000 capacity blocks per CTA: 2 CTAs/SM; fewer than 1536 live vectors per cell keeps it query-major"""
    ix, queries = index_of(128, 64, 6000, 8, initial_size=10000)
    lay = ix.layout()
    assert lay.n_blocks / 8 * 8 >= 2000 and lay.cindex.mean_cell_live < 1536
    assert searched(ix, queries, NQ) == {"ivfpq_scan_kernel<64, 8, 2, 2, false>", "merge_topk_kernel"}


def test_m64_short_lists(cuda_device):
    ix, queries = index_of(128, 64, 6000, 4)
    assert searched(ix, queries, NQ) == {"ivfpq_scan_kernel<64, 8, 3, 2, false>", "merge_topk_kernel"}


def test_m32(cuda_device):
    ix, queries = index_of(128, 32, 4000, 4)
    assert searched(ix, queries, NQ) == {"ivfpq_scan_kernel<32, 8, 2, 4, false>", "merge_topk_kernel"}


def test_m96_staged_lut(cuda_device):
    """d/M = 3 has no in-CTA LUT build: lut_kernel stages it"""
    ix, queries = index_of(288, 96, 3000, 4)
    assert searched(ix, queries, NQ) == {"lut_kernel<0, 1>", "ivfpq_scan_kernel<96, 16, 1, 0, false>", "merge_topk_kernel"}


def test_m120_cosine(cuda_device):
    ix, queries = index_of(960, 120, 2000, 4, distance="cosine")
    assert searched(ix, queries, NQ) == {"ivfpq_scan_kernel<128, 16, 1, 8, false>", "merge_topk_kernel"}


@pytest.mark.parametrize("d, M, want", [
    (128, 64, {"ivfpq_scan_kernel<64, 16, 1, 2, true>"}),
    (512, 64, {"lut_kernel<2, 1>", "ivfpq_scan_kernel<64, 16, 1, 0, true>"}),
    (192, 96, {"lut_kernel<2, 1>", "ivfpq_scan_kernel<96, 16, 1, 0, true>"}),
])
def test_residual(cuda_device, d, M, want):
    ix, queries = index_of(d, M, 3000, 4, residual=True)
    assert searched(ix, queries, NQ) == want | {"merge_topk_kernel"}


def cell_major_index():
    ix, queries = index_of(128, 64, 16000, 4, seed=21)
    assert ix.layout().cindex.mean_cell_live >= 1536
    return ix, queries


def test_cell_major(cuda_device):
    ix, queries = cell_major_index()
    assert searched(ix, queries, NQ) == CELL


def test_sliced_batch_of_a_cell_major_index(cuda_device):
    ix, queries = cell_major_index()
    assert searched(ix, queries, SLICED) == {"ivfpq_scan_kernel<64, 8, 3, 2, false>", "merge_topk_kernel"}


def test_scan_push_stays_query_major(cuda_device):
    ix, queries = cell_major_index()
    x = queries(NQ).cuda()
    buf = torch.zeros(NQ, K, dtype=torch.int64, device="cuda:0")
    ptrs = (C.c_void_p * 1)(buf.data_ptr())
    assert launched(lambda: ix.scan_push(x, K, ptrs, 1, 0)) == {"ivfpq_scan_kernel<64, 8, 3, 2, false>"}
    assert torch.count_nonzero(buf) > 0
