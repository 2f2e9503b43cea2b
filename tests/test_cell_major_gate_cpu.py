"""Which search takes the cell-major scan (scan.cu, plan_scan), pinned on hand-built index structs without a GPU.

tpq_search_workspace_bytes reads only the struct's scalar fields, and only the cell-major plan asks for the queries'
LUTs, their survivor lists and the per-SM survivor logs: its workspace exceeds that of the same index below the
live-vector threshold by at least those buffers, and every other plan's workspace does not depend on the threshold.
The cell-major scan must be taken exactly when every condition holds: a plain (not residual) index, m_pad == 64
(M = 36 .. 64), d/M in {1, 2, 4, 8}, an unsliced batch (at least 4 x SMs queries), an unsharded index with a scan
layout, and at least 1536 live vectors per cell on average.  Either metric qualifies."""
import ctypes as C
import itertools

import pytest

N_CELLS = 4096
N_PROBE = 16
K = 100
CELL_LOG = 256 * 12 * 7 * 32 * 8        # bytes of one CTA's survivor log (kCellWin x 12 warps x 7 blocks x 32 keys)


def sm_count():
    """what the library sizes its batches by: the device's SMs, 132 (H100 SXM) without one"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def index_struct(M, dsub, metric, residual, shard_world, n_blocks, mean_cell_live):
    import torchpq_b200 as T
    ix = T._lib.TpqIndex()
    ix.d_vector, ix.n_subvectors, ix.n_cells, ix.metric = M * dsub, M, N_CELLS, metric
    ix.capacity = N_CELLS * 2048
    ix.m_pad = (M + 31) // 32 * 32
    ix.shard_rank, ix.shard_world = 0, shard_world
    ix.n_blocks = n_blocks
    ix.mean_cell_live = mean_cell_live
    ix.residual = residual
    return ix


def ws_bytes(ix, nq, n_probe=N_PROBE, k=K):
    import torchpq_b200 as T
    return T._lib.lib.tpq_search_workspace_bytes(C.byref(ix), nq, n_probe, k)


def takes_cell_major(ix, nq, n_probe=N_PROBE, k=K):
    """The workspace rule: True when the plan carries the cell-major buffers, False when the workspace is that of the
    same index below the threshold; anything in between fails."""
    import torchpq_b200 as T
    below = T._lib.TpqIndex.from_buffer_copy(ix)
    below.mean_cell_live = 0
    extra = ws_bytes(ix, nq, n_probe, k) - ws_bytes(below, nq, n_probe, k)
    if extra == 0:
        return False
    chunk = min(nq, 16384)
    assert extra >= chunk * (65536 + max(8192, 8 * k) * 8) + sm_count() * CELL_LOG, extra
    return True


def expected(M, dsub, residual, shard_world, n_blocks, mean_cell_live, nq):
    return (not residual and 36 <= M <= 64 and dsub in (1, 2, 4, 8) and shard_world == 1 and n_blocks > 0
            and mean_cell_live >= 1536 and nq >= 4 * sm_count())


@pytest.mark.parametrize("M", [32, 36, 48, 64, 68])
def test_gate(M):
    sms = sm_count()
    taken = 0
    for dsub, metric, residual, shard_world, n_blocks, live, nq in itertools.product(
            (1, 2, 3, 4, 8, 16), (0, 1), (0, 1), (1, 2), (0, N_CELLS * 80), (1535, 1536), (4 * sms - 1, 4 * sms)):
        ix = index_struct(M, dsub, metric, residual, shard_world, n_blocks, live)
        want = expected(M, dsub, residual, shard_world, n_blocks, live, nq)
        cfg = dict(M=M, dsub=dsub, metric=metric, residual=residual, shard_world=shard_world, n_blocks=n_blocks,
                   mean_cell_live=live, nq=nq)
        assert takes_cell_major(ix, nq) == want, cfg
        taken += want
    assert taken == (4 * 2 if 36 <= M <= 64 else 0)                  # d/M x metric: every other condition fixed


@pytest.mark.parametrize("k", [1, 100, 1024])
@pytest.mark.parametrize("n_probe", [1, 2, 64])
def test_gate_ignores_k_and_n_probe(k, n_probe):
    """k and the probe count size the buffers, never the choice; the rule's survivor capacity follows k."""
    ix = index_struct(64, 2, 0, 0, 1, N_CELLS * 80, 1536)
    assert takes_cell_major(ix, 4 * sm_count(), n_probe, k)
    assert not takes_cell_major(ix, 4 * sm_count() - 1, n_probe, k)


def test_two_chunks_keep_the_cell_major_plan():
    """more than 16384 queries run in chunks of 16384 through the same plan"""
    ix = index_struct(64, 4, 1, 0, 1, N_CELLS * 80, 1536)
    assert takes_cell_major(ix, 16384 + 700, N_PROBE, 1024)
