"""GPU parity of the build-side kernels (csrc/place.cu) against the oracle's restatement of CellContainer.add
(oracle/ivfpq_oracle.py: get_ioa / container_add, after kernels/cuda/get_ioa.cu, get_write_address_v2.cu and
container/CellContainer.py:249-367)."""
import numpy as np
import pytest
import torch

from oracle import ivfpq_oracle as O, build_state as B, ref_kernels as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,C", [(1, 4), (4095, 7), (4096, 300), (20_000, 50), (70_001, 5000)])
def test_get_ioa(cuda_device, n, C):
    import torchpq_b200 as T
    rng = np.random.default_rng(n)
    cells = rng.integers(0, C, n)
    cells[: min(n, 100)] = cells[0]                                   # a long run of one label across lanes
    ioa, counts = T.fn.get_ioa(torch.from_numpy(cells).cuda(), C)
    assert np.array_equal(ioa.cpu().numpy(), O.get_ioa(cells))
    assert np.array_equal(counts.cpu().numpy(), np.bincount(cells, minlength=C))
    if R.placement_available() and n <= 20_000:                       # the reference's own get_ioa kernel (O(n * n_unique))
        assert np.array_equal(R.get_ioa(torch.from_numpy(cells).cuda()).cpu().numpy(), ioa.cpu().numpy())


def test_empty_prefix_and_write_address_with_holes(cuda_device):
    import torchpq_b200 as T
    rng = np.random.default_rng(1)
    C, cap_cell = 37, 211
    cap = C * cap_cell
    is_empty = (rng.random(cap) < 0.4).astype(np.uint8)
    prefix = T.fn.empty_prefix(torch.from_numpy(is_empty).cuda()).cpu().numpy().astype(np.int64) % (1 << 32)
    expect = np.zeros(cap + 1, np.int64)
    expect[1:] = np.cumsum(is_empty, dtype=np.int64)
    assert np.array_equal(prefix, expect)
    start = np.arange(C, dtype=np.int64) * cap_cell
    free = np.array([int(is_empty[s:s + cap_cell].sum()) for s in start], dtype=np.int64)
    cells = np.repeat(np.arange(C), np.minimum(free, 20))
    rng.shuffle(cells)
    ioa = O.get_ioa(cells)
    g = lambda a: torch.as_tensor(a).cuda()
    w = T.fn.get_write_address(g(cells), g(ioa), g(start), g(np.zeros(C, np.int64)), g(np.zeros(C, np.int64) + cap_cell),
                               T.fn.empty_prefix(g(is_empty))).cpu().numpy()
    if R.placement_available():                                       # the reference's own get_write_address kernel
        rw = R.get_write_address(g(is_empty), g(start), g(np.zeros(C, np.int64) + cap_cell), g(cells), g(ioa)).cpu().numpy()
        assert np.array_equal(rw, w)
    for i in range(cells.shape[0]):                                   # the ioa-th empty slot of the cell, slot by slot
        s = start[cells[i]]
        assert w[i] == s + np.flatnonzero(is_empty[s:s + cap_cell])[ioa[i]]


def test_add_with_expansion_matches_oracle(cuda_device):
    """Three adds into a small container ('double' and 'step' growth): every buffer equals the oracle's afterwards."""
    from torchpq_b200 import build
    import torchpq_b200 as T
    for mode in ("double", "step"):
        rng = np.random.default_rng(4)
        st = O.empty_state(32, 8, 16, 8)
        ix = T.IVFPQIndex(32, 8, 16, initial_size=8, expand_mode=mode, expand_step_size=50, device="cuda:0")
        for n in (700, 300, 5000):
            codes = rng.integers(0, 256, (8, n)).astype(np.uint8)
            cells = rng.integers(0, 16, n)
            _, adr = O.container_add(st, codes, cells, expand_mode=mode, expand_step_size=50)
            _, gadr = build.container_add(ix, torch.from_numpy(codes).cuda(), torch.from_numpy(cells).cuda(), return_address=True)
            assert np.array_equal(gadr.cpu().numpy(), adr)
        for name, ref in (("_storage", st.storage), ("_is_empty", st.is_empty), ("_cell_start", st.cell_start),
                          ("_cell_size", st.cell_size), ("_cell_capacity", st.cell_capacity), ("_address2id", st.address2id)):
            assert np.array_equal(getattr(ix, name).cpu().numpy(), ref), (mode, name)


def test_add_updates_scan_layout_in_place(cuda_device):
    """An add that needs no expansion writes the new codes into the existing scan layout (no relayout): the layout object
    survives, holds the same bytes as a layout built afresh from the reference buffers (the two writers of the format,
    tpq_store_codes and tpq_relayout_codes, agree on every slot), and searches see the new items exactly as the fresh
    layout does.  Unsharded, and on shard 1 of 2, where only the shard's cells are written."""
    import torchpq_b200 as T
    torch.manual_seed(8)
    base = torch.randn(64, 30_000, device="cuda")
    x = torch.randn(64, 200, device="cuda")
    for rank, world in ((0, 1), (1, 2)):
        ix = T.IVFPQIndex(64, 16, 32, initial_size=2048, device="cuda:0")
        ix.train(base[:, :10_000].contiguous())
        ix.add(base[:, :12_000].contiguous())
        ix.set_shard(rank, world)
        ix.n_probe = 8
        ix.search(x, k=10)
        lay = ix._layout
        assert lay is not None and lay.shard == (rank, world)
        for s in (12_000, 18_000, 24_000):
            ix.add(base[:, s:s + 6000].contiguous())
            assert ix._layout is lay, "the add rebuilt the scan layout"
        v1, i1, a1 = ix.search(x, k=20, return_address=True)
        ix._state_changed()                                           # force a relayout from the reference buffers
        v2, i2, a2 = ix.search(x, k=20, return_address=True)
        fresh = ix._layout
        assert fresh is not lay and fresh.shard == (rank, world)
        assert fresh.n_blocks == lay.n_blocks > 0
        n_bytes = lay.n_blocks * lay.m_pad * 32
        assert torch.equal(lay.codes_scan[:n_bytes], fresh.codes_scan[:n_bytes]), (rank, world)
        assert torch.equal(lay.block_valid[:lay.n_blocks], fresh.block_valid[:fresh.n_blocks]), (rank, world)
        assert torch.equal(v1, v2) and torch.equal(i1, i2) and torch.equal(a1, a2)
        assert int((i1 >= 12_000).sum()) > 0                          # later adds are found
