"""CPU: the workspace sizes of the fused GEMM searches (flat.cu, ivfflat.cu) pinned to exact values over a grid of
shapes.  A size is the plan's layout (QT, S, chunk and every offset), so a change to any plan decision shows here.
tests/golden/fused_plan_workspace.npz holds the values; S depends on the SM count, and they are for 132 SMs (H100
SXM, and what the library assumes without a device)."""
import itertools
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fused_plan_workspace.npz")
D = (8, 33, 128)
NQ = (1, 7, 100, 5000, 16384, 16385, 10 ** 6, 2 * 10 ** 7)
N = (0, 1, 1000, 10 ** 6, 10 ** 9)
N_CELLS = (0, 1, 100, 4096, 10 ** 6, 10 ** 9)
N_PROBE = (1, 32, 64, 1024)
K = (1, 10, 100, 512, 1024)


def workspace_sizes(L):
    """Every size over the grid, in the golden file's order."""
    return {
        "flat": [L.tpq_flat_workspace_bytes(*a) for a in itertools.product(D, NQ, N, K)],
        "flat_range": [L.tpq_flat_range_workspace_bytes(*a) for a in itertools.product(D, NQ, N)],
        "ivfflat": [L.tpq_ivfflat_workspace_bytes(*a) for a in itertools.product(D, NQ, N_CELLS, N_PROBE, K)],
        "ivfflat_range": [L.tpq_ivfflat_range_workspace_bytes(*a) for a in itertools.product(D, NQ, N_CELLS, N_PROBE)],
    }


@pytest.fixture(scope="module")
def lib():
    import torch
    import torchpq_b200 as T
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the pinned sizes are for 132 SMs")
    return T._lib.lib


@pytest.mark.parametrize("entry", ["flat", "flat_range", "ivfflat", "ivfflat_range"])
def test_workspace_sizes_pinned(lib, entry):
    want = np.load(GOLDEN)[entry]
    got = np.array(workspace_sizes(lib)[entry], dtype=np.uint64)
    assert got.shape == want.shape
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} sizes differ, first at grid index {bad[0]}: {got[bad[0]]} != {want[bad[0]]}"
