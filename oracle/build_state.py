"""Seeded builders of synthetic IVFPQ index states (TEST INFRASTRUCTURE, see oracle/__init__.py).

The reference trains with unseeded ``np.random.choice`` initial centroids
(clustering/MultiKMeans.py:277-283, clustering/KMeans.py:270-276), so parity is
defined on *identical trained state*: these builders produce one state, and the
oracle and the CUDA path are both fed that same state.

Assignment follows the reference's direct form ``argmax_j sum_i -(a_i - b_ij)^2``
(kernels/cuda/max_sim.cu:78-98); Lloyd updates follow compute_centroids.cu:9-86
(mean of members; an empty cluster becomes 0).
"""
from __future__ import annotations

import numpy as np
import torch

from . import ivfpq_oracle as O


def assign(data: torch.Tensor, centroids: torch.Tensor, chunk: int = 65536) -> torch.Tensor:
    """data [d, n], centroids [d, k] -> labels [n] (argmax of negative squared L2, lowest index on ties)."""
    out = torch.empty(data.shape[1], dtype=torch.long)
    c2 = (centroids ** 2).sum(0)
    for s in range(0, data.shape[1], chunk):
        a = data[:, s:s + chunk]
        sim = 2 * (a.T @ centroids) - (a ** 2).sum(0)[:, None] - c2[None, :]
        out[s:s + chunk] = sim.argmax(dim=1)
    return out


def lloyd(data: torch.Tensor, k: int, iters: int, gen: torch.Generator) -> torch.Tensor:
    """Seeded k-means: random distinct data points as initial centroids, `iters` Lloyd steps."""
    d, n = data.shape
    perm = torch.randperm(n, generator=gen)[:k]
    cent = data[:, perm].clone()
    if perm.shape[0] < k:                                   # fewer points than clusters
        cent = torch.cat([cent, torch.zeros(d, k - perm.shape[0])], dim=1)
    for _ in range(iters):
        lab = assign(data, cent)
        sums = torch.zeros(d, k).index_add_(1, lab, data)
        cnt = torch.zeros(k).index_add_(0, lab, torch.ones(n))
        cent = torch.where(cnt[None, :] > 0, sums / cnt.clamp(min=1)[None, :], torch.zeros(()))
    return cent


def train_codebooks(train: torch.Tensor, n_subvectors: int, n_cells: int, seed: int = 0,
                    vq_iters: int = 6, pq_iters: int = 6):
    """-> (vq_codebook [d, C], pq_codebook [M, dsub, 256]) fp32 numpy."""
    gen = torch.Generator().manual_seed(seed)
    d, n = train.shape
    M = n_subvectors
    dsub = d // M
    vq = lloyd(train, n_cells, vq_iters, gen)
    sub = train.reshape(M, dsub, n)
    pq = torch.stack([lloyd(sub[m], 256, pq_iters, gen) for m in range(M)], dim=0)
    return vq.numpy().astype(np.float32), pq.numpy().astype(np.float32)


def encode(x: torch.Tensor, vq: np.ndarray, pq: np.ndarray):
    """IVFPQIndex.add's two encodes (IVFPQIndex.py:351-356): coarse cell + PQ code.
    -> (cells [n] i64, codes [M, n] u8)."""
    M, dsub, _ = pq.shape
    cells = assign(x, torch.from_numpy(vq)).numpy()
    sub = x.reshape(M, dsub, x.shape[1])
    codes = np.stack([assign(sub[m], torch.from_numpy(pq[m])).numpy().astype(np.uint8) for m in range(M)], 0)
    return cells, codes


def build_state(base: torch.Tensor, n_subvectors: int, n_cells: int, distance: str = "euclidean",
                initial_size: int | None = None, seed: int = 0, n_train: int | None = None,
                add_batches: int = 1, vq_iters: int = 6, pq_iters: int = 6) -> O.IndexState:
    """Train on a prefix of `base`, then add all of `base` (ids = arange) the way
    IVFPQIndex.train / .add would (IVFPQIndex.py:234-260,316-364)."""
    d, n = base.shape
    x = O.normalize(base, 0) if distance == "cosine" else base
    n_train = n if n_train is None else min(n, n_train)
    vq, pq = train_codebooks(x[:, :n_train].contiguous(), n_subvectors, n_cells, seed, vq_iters, pq_iters)
    cells, codes = encode(x, vq, pq)
    if initial_size is None:
        initial_size = max(1, int(np.bincount(cells, minlength=n_cells).max()))
    st = O.empty_state(d, n_subvectors, n_cells, initial_size, distance, vq, pq)
    step = (n + add_batches - 1) // add_batches
    for s in range(0, n, step):
        O.container_add(st, codes[:, s:s + step], cells[s:s + step])
    return st


def integer_state(d: int, n_subvectors: int, n_cells: int, n: int, seed: int = 0,
                  distance: str = "euclidean", initial_size: int | None = None, lo: int = -3, hi: int = 4):
    """Known-answer state: small-integer codebooks and a random code/cell assignment, so that
    every coarse score, LUT entry and ADC sum is an exactly representable integer in fp32
    (and fp16).  -> (state, integer query generator)."""
    rng = np.random.default_rng(seed)
    M = n_subvectors
    vq = rng.integers(lo, hi, size=(d, n_cells)).astype(np.float32)
    pq = rng.integers(lo, hi, size=(M, d // M, 256)).astype(np.float32)
    cells = rng.integers(0, n_cells, size=n).astype(np.int64)
    codes = rng.integers(0, 256, size=(M, n)).astype(np.uint8)
    if initial_size is None:
        initial_size = max(1, int(np.bincount(cells, minlength=n_cells).max()))
    st = O.empty_state(d, M, n_cells, initial_size, distance, vq, pq)
    O.container_add(st, codes, cells)

    def queries(nq: int, qseed: int = 1):
        r = np.random.default_rng(qseed)
        return torch.from_numpy(r.integers(lo, hi, size=(d, nq)).astype(np.float32))

    return st, queries


def randn_state(d: int, n_subvectors: int, n_cells: int, n: int, seed: int = 0, distance: str = "euclidean",
                initial_size: int | None = None, scale: float = 1.0) -> O.IndexState:
    """Real-valued state without training: standard-normal codebooks (times `scale`), random codes and cells, so that
    LUT entries and scores are arbitrary fp32 values -- for the bit-exact restatements of oracle/fp32_exact.py, where
    what matters is the arithmetic, not the quality of the quantiser."""
    rng = np.random.default_rng(seed)
    M = n_subvectors
    vq = (rng.standard_normal((d, n_cells)) * scale).astype(np.float32)
    pq = (rng.standard_normal((M, d // M, 256)) * scale).astype(np.float32)
    cells = rng.integers(0, n_cells, size=n).astype(np.int64)
    codes = rng.integers(0, 256, size=(M, n)).astype(np.uint8)
    if initial_size is None:
        initial_size = max(1, int(np.bincount(cells, minlength=n_cells).max()))
    st = O.empty_state(d, M, n_cells, initial_size, distance, vq, pq)
    O.container_add(st, codes, cells)
    return st


def build_state_residual(base: torch.Tensor, n_subvectors: int, n_cells: int, seed: int = 0, n_train=None,
                         vq_iters: int = 4, pq_iters: int = 3) -> O.IndexState:
    """pq_use_residual=True: PQ is trained on and encodes x - vq_centroid(cell)
    (IVFPQIndex.train :248-256, IVFPQIndex.encode :281-284)."""
    d, n = base.shape
    M, dsub = n_subvectors, d // n_subvectors
    gen = torch.Generator().manual_seed(seed)
    n_train = n if n_train is None else min(n, n_train)
    tr = base[:, :n_train].contiguous()
    vq = lloyd(tr, n_cells, vq_iters, gen)
    res_tr = tr - vq[:, assign(tr, vq)]
    sub = res_tr.reshape(M, dsub, n_train)
    pq = torch.stack([lloyd(sub[m], 256, pq_iters, gen) for m in range(M)], 0)
    cells = assign(base, vq)
    res = (base - vq[:, cells]).reshape(M, dsub, n)
    codes = np.stack([assign(res[m], pq[m]).numpy().astype(np.uint8) for m in range(M)], 0)
    cells = cells.numpy()
    initial = max(1, int(np.bincount(cells, minlength=n_cells).max()))
    st = O.empty_state(d, M, n_cells, initial, "euclidean", vq.numpy().astype(np.float32), pq.numpy().astype(np.float32))
    O.container_add(st, codes, cells)
    return st
