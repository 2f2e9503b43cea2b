"""CPU: the k-means assignment ABI (sizes, null pointers, metric, workspace size), the test-side restatements of the
manhattan metric, the distance-aware fit and k-means++ (tests/kmeans_ref.py), and the clustering classes' host-side
behaviour."""
import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as K
import kmeans_ref as R


def test_kmeans_assign_error_channel():
    import torchpq_b200 as T
    lib, P = T._lib.lib, 16  # any non-null value: the checks run before anything is dereferenced
    rc = lib.tpq_kmeans_assign(None, P, 1, 8, 100, 10, 0, 1, P, P, None, 0, None)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and "null pointer" in T._lib.last_error()
    rc = lib.tpq_kmeans_assign(P, P, 1, 0, 100, 10, 0, 1, P, P, None, 0, None)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and "bad sizes" in T._lib.last_error()
    rc = lib.tpq_kmeans_assign(P, P, 1, 8, -1, 10, 0, 1, P, P, None, 0, None)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and "bad sizes" in T._lib.last_error()
    rc = lib.tpq_kmeans_assign(P, P, 1, 8, 100, 10, 3, 1, P, P, None, 0, None)
    assert rc == T._lib.TPQ_ERR_BAD_ARG and "unsupported metric 3" in T._lib.last_error()
    with pytest.raises(AssertionError):
        T._lib.check(rc)
    assert lib.tpq_kmeans_assign(P, P, 1, 8, 0, 10, 0, 1, P, P, None, 0, None) == T._lib.TPQ_OK   # n = 0: nothing to do
    rc = lib.tpq_max_sim(P, P, 1, 8, 100, 10, 3, 1, P, P, None)
    assert rc == T._lib.TPQ_ERR_BAD_ARG


def test_manhattan_rejected_by_index_entry_points():
    import torchpq_b200 as T
    lib, P = T._lib.lib, 16
    assert T._lib.METRIC["manhattan"] == 2
    assert lib.tpq_build_lut(P, P, 16, 4, 1, 2, P, None) == T._lib.TPQ_ERR_BAD_ARG
    assert lib.tpq_relayout_codebook(P, 16, 4, 2, P, P, None) == T._lib.TPQ_ERR_BAD_ARG
    assert "unsupported metric 2" in T._lib.last_error()
    with pytest.raises(AssertionError):
        T.IVFPQIndex(32, 8, 4, initial_size=4, device="cpu", distance="manhattan")


@pytest.mark.parametrize("l,d,k,want", [(1, 128, 4096, 4096 * 136 * 4), (3, 72, 257, 3 * 384 * 80 * 4),
                                        (2, 256, 16384, 2 * 16384 * 264 * 4), (1, 264, 1000, 0), (1, 12, 1000, 0),
                                        (1, 64, 4, 0)])
def test_kmeans_assign_workspace_bytes(l, d, k, want):
    """One K-major row of d + 8 floats (features + bias block) per centroid, k padded to 128; 0 outside the
    streaming kernel's range (the exact kernel needs no workspace)."""
    import torchpq_b200 as T
    assert T._lib.lib.tpq_kmeans_assign_workspace_bytes(l, d, k) == want


def test_ref_manhattan_matches_direct_formula():
    rng = np.random.default_rng(0)
    data = rng.integers(-3, 4, (2, 6, 50)).astype(np.float32)
    cent = rng.integers(-3, 4, (2, 6, 30)).astype(np.float32)
    sims, labels = R.max_sim(data, cent, "manhattan")
    direct = -np.abs(data[:, :, :, None] - cent[:, :, None, :]).sum(axis=1)      # [l, n, k], exact for integers
    assert np.array_equal(sims, direct.max(axis=-1))
    assert np.array_equal(labels, direct.argmax(axis=-1))                       # numpy argmax: first maximum


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "manhattan"])
def test_ref_fit_distance(distance):
    """Two well separated blobs: one assignment splits them, the second changes nothing, so the loop stops at 2."""
    rng = np.random.default_rng(1)
    a = rng.normal(0, 0.1, (1, 4, 40)) + np.array([10, 0, 0, 0])[None, :, None]
    b = rng.normal(0, 0.1, (1, 4, 40)) + np.array([0, 10, 0, 0])[None, :, None]
    data = np.concatenate([a, b], axis=2).astype(np.float32)
    cent, labels, inertia, n_iter = R.fit(data, data[:, :, [0, 40]], 20, distance=distance)
    assert n_iter == 2 and (labels[0, :40] == 0).all() and (labels[0, 40:] == 1).all()
    assert np.allclose(cent[0, :, 0], data[0, :, :40].mean(1), atol=1e-5)
    assert np.array_equal(R.fit(data, data[:, :, [0, 40]], 20)[0], R.fit(data, data[:, :, [0, 40]], 20, distance="euclidean")[0])


@pytest.mark.parametrize("distance", ["euclidean", "manhattan", "inner"])
def test_ref_kmeanspp_is_farthest_first(distance):
    """The restated reference loop equals an incremental running-best version (what the GPU code does)."""
    rng = np.random.default_rng(2)
    data = rng.standard_normal((2, 5, 300)).astype(np.float32)
    k, first = 12, 17
    got = R.kmeanspp(data, k, first, distance)
    cent = np.zeros_like(got)
    cent[:, :, 0] = data[:, :, first]
    best = R.max_sim(data, cent[:, :, :1], distance)[0]
    for i in range(1, k):
        idx = best.argmin(-1)
        cent[:, :, i] = data[np.arange(2), :, idx]
        best = np.maximum(best, R.max_sim(data, cent[:, :, i:i + 1], distance)[0])
    assert np.array_equal(got, cent)
    assert (got[:, :, 0] == data[:, :, first]).all()


def test_clustering_constructor_and_state_dict():
    import torchpq_b200 as T
    with pytest.raises(AssertionError):
        T.KMeans(8, distance="inner")
    with pytest.raises(AssertionError):
        T.MultiKMeans(8, init_mode="kmeans||")
    km = T.KMeans(8, sm_size=123, seed=4)
    assert km.centroids is None and km.seed == 4
    with pytest.raises(AssertionError):
        km.predict(torch.zeros(4, 10))
    km.load_state_dict({"centroids": torch.arange(32.0).reshape(4, 8)})      # the reference's KMeans state_dict
    assert km.state_dict()["centroids"].shape == (4, 8)
    km2 = T.KMeans(8)
    km2.load_state_dict(km.state_dict())
    assert torch.equal(km2.centroids, km.centroids)
    with pytest.raises(AssertionError):
        km2.topk(torch.zeros(4, 10), k=9)                                       # more than n_clusters
    assert float(T.MultiKMeans.calculate_error(torch.ones(2, 3), torch.zeros(2, 3))) == 6.0
    assert float(T.KMeans.calculate_inertia(torch.tensor([-1.0, -3.0]))) == 2.0
