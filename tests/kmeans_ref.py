"""CPU restatements for the clustering tests, on top of oracle.kmeans_oracle (TEST INFRASTRUCTURE).

    max_sim    kmeans_oracle.max_sim plus the manhattan metric: acc - |a - b|, e ascending, fp32
               (kernels/cuda/max_sim.cu:100-120, thread_nmanhattan); lowest index among equal maxima
    fit        MultiKMeans.fit for one redo from given centroids, for every distance (clustering/MultiKMeans.py:431-441)
    kmeanspp   the reference's k-means++ loop (clustering/MultiKMeans.py:232-268), re-scoring every chosen centroid at
               each step: the check of the incremental GPU version
"""
import numpy as np

from oracle import kmeans_oracle as K


def max_sim(data, cent, distance="euclidean", chunk=4096):
    """data [l, d, n], cent [l, d, k] -> (maxsims [l, n] f32, labels [l, n] i64) for euclidean, inner ("cosine" on
    columns the caller has normalised) or manhattan."""
    if distance != "manhattan":
        return K.max_sim(data, cent, distance, chunk)
    data, cent = np.asarray(data, np.float32), np.asarray(cent, np.float32)
    l, d, n = data.shape
    k = cent.shape[2]
    sims = np.empty((l, n), np.float32)
    labels = np.empty((l, n), np.int64)
    for li in range(l):
        for s in range(0, n, chunk):
            x = data[li, :, s:s + chunk]
            acc = np.zeros((x.shape[1], k), np.float32)
            for e in range(d):
                acc = (acc - np.abs((x[e][:, None] - cent[li, e][None, :]).astype(np.float32))).astype(np.float32)
            labels[li, s:s + chunk] = acc.argmax(axis=1)                 # numpy: first maximum
            sims[li, s:s + chunk] = acc.max(axis=1)
    return sims, labels


def normalized(x):
    """x / (||x|| + 1e-8) per column (the reference's cosine normalisation), in fp32."""
    x = np.asarray(x, np.float32)
    nrm = np.sqrt((x.astype(np.float64) ** 2).sum(axis=-2, keepdims=True)).astype(np.float32)
    return (x / (nrm + np.float32(1e-8))).astype(np.float32)


def fit(data, centroids0, max_iter, tol=1e-4, distance="euclidean"):
    """One redo of MultiKMeans.fit from given initial centroids: labels = arg-max similarity (cosine: on normalised
    copies of data and centroids), new centroids = member means of the raw data, error = sum((new - old)^2), stop
    when error <= tol.  -> (centroids, labels of the last assignment, inertia = mean(-maxsims), iterations)."""
    cent = np.asarray(centroids0, np.float32)
    k = cent.shape[2]
    n_iter = 0
    for _ in range(max_iter):
        if distance == "cosine":
            sims, labels = max_sim(normalized(data), normalized(cent), "cosine")
        else:
            sims, labels = max_sim(data, cent, distance)
        new = K.compute_centroids(data, labels, k)
        diff = (new - cent).astype(np.float32)
        error = float((diff * diff).astype(np.float32).sum(dtype=np.float32))
        cent = new
        n_iter += 1
        if error <= tol:
            break
    return cent, labels, float((-sims).mean()), n_iter


def kmeanspp(data, k, first, distance="euclidean"):
    """Centroid 0 = column `first` (the same for every k-means); at each step i ALL chosen centroids are re-scored and
    the next centroid is the point with the lowest best similarity (first such point).  Cosine picks normalised
    points.  data [l, d, n] -> centroids [l, d, k]."""
    x = normalized(data) if distance == "cosine" else np.asarray(data, np.float32)
    l, d, n = x.shape
    cent = np.zeros((l, d, k), np.float32)
    cent[:, :, 0] = x[:, :, first]
    for i in range(1, k):
        sims, _ = max_sim(x, cent[:, :, :i], distance)
        cent[:, :, i] = x[np.arange(l), :, sims.argmin(axis=-1)]     # first minimum
    return cent
