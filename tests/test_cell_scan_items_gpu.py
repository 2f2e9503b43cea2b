"""GPU: cells probed by more pairs than the cell-major kernel's shared-memory record window holds (256).  The kernel
then walks an item's pairs window by window, draining the LUT ring in between; the result must stay bit-identical to
the query-major kernel's and to the oracle.  With 8 cells, n_probe = 4 and fixed probing, every query contributes three
pairs (entries 1..3), so NQ queries put about 3 NQ / 8 pairs on each cell."""
import numpy as np
import pytest
import torch

from oracle import ivfpq_oracle as O, build_state as B
from test_cell_scan_gpu import cell_major_index, in_small_batches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nq", [700, 1500, 3000])     # about 260, 560 and 1125 pairs per cell: 2, 3 and 5 windows
@pytest.mark.parametrize("k", [10, 100])
def test_cells_with_more_pairs_than_the_window(cuda_device, nq, k):
    st, queries = B.integer_state(128, 64, 8, 16000, seed=77 + k)
    st.n_probe, st.use_smart_probing = 4, False
    x = queries(nq)
    ix = cell_major_index(st)
    xd = x.cuda()
    big = ix.search(xd, k=k, return_address=True, return_keys=True)
    small = in_small_batches(lambda s, e: ix.search(xd[:, s:e].contiguous(), k=k, return_address=True,
                                                    return_keys=True), nq)
    for a, b in zip(big, small):
        assert torch.equal(a.cpu(), b.cpu())
    ov, oi, oa = O.search(st, x, k=k, return_address=True)
    assert np.array_equal(big[0].cpu().numpy(), ov)
    assert np.array_equal(big[2].cpu().numpy(), oa)
    assert np.array_equal(big[1].cpu().numpy(), oi)
