"""Which scan a search takes, read off the workspace the library asks for (host-side, no GPU needed): the cell-major scan
needs the LUT and survivor buffers, the query-major kernel does not.  C3 shape: d = 128, M = 64, 4096 cells."""
import ctypes as C

import pytest


def c3_index(mean_cell_live=2441, shard_world=1, residual=0, d=128, M=64):
    import torchpq_b200 as T
    ix = T._lib.TpqIndex()
    ix.d_vector, ix.n_subvectors, ix.n_cells, ix.metric = d, M, 4096, 0
    ix.capacity = 4096 * 3200
    ix.m_pad = (M + 31) // 32 * 32
    ix.shard_rank, ix.shard_world = 0, shard_world
    ix.n_blocks = 4096 * 100 // shard_world
    ix.mean_cell_live = mean_cell_live
    ix.residual = residual
    return ix


def ws_bytes(ix, nq, n_probe=32, k=100):
    import torchpq_b200 as T
    return T._lib.lib.tpq_search_workspace_bytes(C.byref(ix), nq, n_probe, k)


def extra(nq, **kw):
    """workspace of the index as given minus that of the same index below the cell-major threshold"""
    return ws_bytes(c3_index(**kw), nq) - ws_bytes(c3_index(**dict(kw, mean_cell_live=0)), nq)


def test_c3_takes_the_cell_major_scan():
    nq = 10000
    assert extra(nq) >= nq * 65536 + nq * 8192 * 8                  # LUTs + survivors of every query of the chunk


@pytest.mark.parametrize("kw", [dict(mean_cell_live=1535), dict(shard_world=2), dict(shard_world=4), dict(M=120, d=960)])
def test_query_major_elsewhere(kw):
    """below 1536 live vectors per cell (C2: 977), on a cell shard (entry 0 is mostly another shard's empty cell, so the
    bound would be 0 and every query would overflow), and above M = 64 (C4)."""
    assert extra(10000, **kw) == 0


def test_sliced_batch_keeps_the_query_major_kernel():
    assert extra(100) == 0                                           # fewer than 4 x SMs queries: sliced


def test_cell_major_workspace_is_bounded_by_the_query_chunk():
    """The stage runs per chunk of 16384 queries, so its LUT and survivor buffers do not grow with the batch; only the
    8-byte pass-1 probe count per query does."""
    small, big = extra(16384), extra(1_000_000)
    assert big - small <= (1_000_000 - 16384) * 8 + 4096
    assert big < 3 * 1024 ** 3
