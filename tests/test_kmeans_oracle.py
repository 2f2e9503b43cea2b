"""CPU: the two centroid-update oracles of oracle/kmeans_oracle.py agree with each other, and the sequential one takes
its sums in point order (the GPU update is pinned to it bit for bit in test_kmeans_gpu.py)."""
import numpy as np
import pytest

from oracle import kmeans_oracle as K


@pytest.mark.parametrize("l,d,n,k", [(2, 3, 1000, 7), (1, 17, 5000, 300), (3, 1, 50, 1), (1, 5, 2000, 4099)])
def test_sequential_centroids_match_float64_mean(l, d, n, k):
    rng = np.random.default_rng(n + k)
    data = rng.standard_normal((l, d, n)).astype(np.float32)
    labels = rng.integers(-2, k + 2, (l, n))
    labels[:, ::97] = 2 ** 40                                   # out of range: ignored by both
    seq = K.compute_centroids_seq(data, labels, k)
    ref = K.compute_centroids(data, labels, k)
    assert seq.dtype == np.float32 and seq.shape == (l, d, k)
    # sequential fp32 sum of c terms: error <= (c - 1) 2^-24 sum|x|; then two roundings of the mean
    abs_sum = K.compute_centroids(np.abs(data), labels, k).astype(np.float64)
    cnt = np.stack([np.bincount(lab[(lab >= 0) & (lab < k)], minlength=k) for lab in labels])[:, None, :]
    abs_sum *= cnt
    tol = 2.0 ** -24 * abs_sum + 2.0 ** -23 * np.abs(ref.astype(np.float64))
    assert (np.abs(seq.astype(np.float64) - ref.astype(np.float64)) <= tol).all()
    for li in range(l):
        assert (seq[li][:, cnt[li, 0] == 0] == 0).all()


def test_sequential_centroids_follow_point_order():
    """1e8 + 1 - 1e8 is 0 in fp32 taken in point order, 1 in any order that adds 1 last."""
    data = np.array([[[1e8, 1.0, -1e8, 5.0, 7.0]]], np.float32)
    labels = np.array([[0, 0, 0, -1, 2]])
    c = K.compute_centroids_seq(data, labels, 3)
    assert c[0, 0, 0] == np.float32(0.0)                     # (1e8 + 1) - 1e8, then / 3
    assert c[0, 0, 1] == 0 and c[0, 0, 2] == np.float32(7.0)  # empty cluster 0; label -1 ignored
    flipped = K.compute_centroids_seq(data[:, :, [0, 2, 1]], labels[:, [0, 2, 1]], 3)
    assert flipped[0, 0, 0] == np.float32(1.0) / np.float32(3.0)
    assert K.compute_centroids(data, labels, 3)[0, 0, 0] == np.float32(1.0 / 3.0)


def test_sequential_centroids_empty_input():
    c = K.compute_centroids_seq(np.zeros((2, 4, 0), np.float32), np.zeros((2, 0), np.int64), 5)
    assert c.shape == (2, 4, 5) and (c == 0).all()
